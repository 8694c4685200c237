"""GPU: FusedBertAdam against tests/golden/ref_bert_adam.pt — outputs of the reference's OWN `BertAdam` class
(modules/optimization.py:66-168) run by oracle/make_golden.py with the drivers' four parameter groups
(main_task_retrieval.py:173-190) and the driver-side clip_grad_norm_(…, 1.0) (main_task_retrieval.py:347).

Tolerance: fp32 arithmetic on both sides; ours is compiled with --use_fast_math (approximate sqrt / division, ~2 ulp)
so parameters after k steps agree to |d| <= 2e-6 + 2e-5 * lr-scaled update (stated below as rtol 2e-5 / atol 2e-6 on
values of magnitude 0.5).
"""
import pytest
import torch

from oracle import synth
from tests.oracle_util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _groups(params, gold):
    named = list(params.items())
    no_decay = gold["no_decay"]
    dec = [(n, p) for n, p in named if not any(nd in n for nd in no_decay)]
    nod = [(n, p) for n, p in named if any(nd in n for nd in no_decay)]
    lr, coef = gold["lr"], gold["coef_lr"]
    return [{"params": [p for n, p in dec if "bert." in n], "weight_decay": 0.01, "lr": lr * coef},
            {"params": [p for n, p in dec if "bert." not in n], "weight_decay": 0.01},
            {"params": [p for n, p in nod if "bert." in n], "weight_decay": 0.0, "lr": lr * coef},
            {"params": [p for n, p in nod if "bert." not in n], "weight_decay": 0.0}]


def _make_opt(params, gold):
    from univl_b200.modules.optimization import BertAdam
    opt = BertAdam(_groups(params, gold), lr=gold["lr"], warmup=gold["warmup"], schedule="warmup_linear",
                   t_total=gold["t_total"], weight_decay=0.01, max_grad_norm=gold["max_grad_norm"])
    opt.global_clip_norm = gold["global_clip"]   # the driver's clip_grad_norm_, folded into the fused step
    return opt


def _check(t, want, what):
    t = t.detach().float().cpu()
    if isinstance(want, dict):    # long tensor: head / tail slices + moments
        f = t.flatten()
        torch.testing.assert_close(f[:256], want["head"], rtol=2e-5, atol=2e-6, msg=lambda m: what + " head: " + m)
        torch.testing.assert_close(f[-256:], want["tail"], rtol=2e-5, atol=2e-6, msg=lambda m: what + " tail: " + m)
        assert abs(float(f.double().sum()) - want["sum"]) <= 1e-4 * max(1.0, abs(want["sum"])) + 1e-3, what
        sq = float((f.double() ** 2).sum())
        assert abs(sq - want["sq_sum"]) <= 1e-4 * want["sq_sum"] + 1e-9, what
    else:
        torch.testing.assert_close(t, want, rtol=2e-5, atol=2e-6, msg=lambda m: what + ": " + m)


def test_bert_adam_matches_reference_class_over_driver_loop():
    """backward -> clip -> step -> zero_grad x 4, gradients ACCUMULATED into p.grad as autograd does (so a zero_grad
    that misses the per-parameter grads — the compat path the reference drivers use — shows up from step 2 on)."""
    gold = load_golden("bert_adam")
    names_shapes, init, grads, no_grad = synth.adam_case(len(gold["after"]))
    params = {n: torch.nn.Parameter(v.clone().to(DEV)) for n, v in init.items()}
    opt = _make_opt(params, gold)
    for t, after in enumerate(gold["after"]):
        for n, p in params.items():
            if n in no_grad:
                continue
            g = grads[t][n].to(DEV)
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.add_(g)
        opt.step()
        opt.zero_grad()
        for n, p in params.items():
            _check(p, after["params"][n], "step %d %s" % (t + 1, n))
        sd = opt.state_dict()
        order = [p for grp in opt.param_groups for p in grp["params"]]
        by_param = {id(p): sd["state"][i] for i, p in enumerate(order) if i in sd["state"]}
        for n, p in params.items():
            if n in after["next_m"]:
                st = by_param[id(p)]
                assert st["step"] == t + 1
                _check(st["next_m"], after["next_m"][n], "step %d next_m %s" % (t + 1, n))
                _check(st["next_v"], after["next_v"][n], "step %d next_v %s" % (t + 1, n))
    assert sorted(set(opt.get_lr()))  # the drivers log it (main_task_retrieval.py:357-360)


def test_bert_adam_resumes_from_reference_state_dict():
    """load the REFERENCE optimizer's state_dict (after step 3) and take step 4 (main_pretrain.py:270, :389)."""
    gold = load_golden("bert_adam")
    names_shapes, init, grads, no_grad = synth.adam_case(len(gold["after"]))
    after3, after4 = gold["after"][2], gold["after"][3]
    big = "decoder.classifier.cls.predictions.bias"
    # parameters as they were after step 3 (the long tensor is rebuilt by replaying 3 steps on the device)
    params = {n: torch.nn.Parameter(v.clone().to(DEV)) for n, v in init.items()}
    warm = _make_opt(params, gold)
    for t in range(3):
        for n, p in params.items():
            p.grad = grads[t][n].to(DEV).clone() if n not in no_grad else None
        warm.step()
    warm_sd = warm.state_dict()
    fresh = {n: torch.nn.Parameter(p.detach().clone()) for n, p in params.items()}
    for n, p in fresh.items():
        if n != big:
            p.data.copy_(after3["params"][n].to(DEV))
    sd = gold["state_dict_after3"]
    order = [n for grp in _groups({n: n for n in fresh}, gold) for n in grp["params"]]
    warm_order = [p for grp in warm.param_groups for p in grp["params"]]
    for i, st in sd["state"].items():       # the long tensor's moments were dropped from the fixture: take ours
        if st["next_m"] is None:
            assert order[i] == big
            st["next_m"] = warm_sd["state"][i]["next_m"].cpu()
            st["next_v"] = warm_sd["state"][i]["next_v"].cpu()
    assert len(warm_order) == len(order)
    opt = _make_opt(fresh, gold)
    opt.load_state_dict(sd)
    for n, p in fresh.items():
        p.grad = grads[3][n].to(DEV).clone() if n not in no_grad else None
    opt.step()
    for n, p in fresh.items():
        _check(p, after4["params"][n], "resumed step 4 %s" % n)
    assert int(opt.step_dev.item()) == 4


def test_param_group_lr_edit_is_honoured():
    from univl_b200.optim import FusedBertAdam
    p = torch.nn.Parameter(torch.ones(1000, device=DEV))
    opt = FusedBertAdam([p], lr=1e-2, weight_decay=0.0, max_grad_norm=-1.0)
    p.grad = torch.ones_like(p)
    opt.step()
    d1 = float((1.0 - p.detach()).mean())
    opt.param_groups[0]["lr"] = 1e-3
    before = p.detach().clone()
    opt.step()
    d2 = float((before - p.detach()).mean())
    assert d1 > 0 and 0.05 * d1 < d2 < 0.2 * d1, (d1, d2)   # 10x smaller lr -> ~10x smaller step (m/sqrt(v) drifts a bit)


def test_bf16_gradient_payload_equals_fp32_of_the_same_values():
    """the data-parallel loop hands the optimizer the summed bf16 all-reduce payload (univl_bert_adam_step_bf16grad):
    bit-identical to the fp32 path fed the same (bf16-representable) gradient values, clips included."""
    from univl_b200.optim import FusedBertAdam
    torch.manual_seed(0)
    shapes = [(300, 64), (77,), (1000, 3), (5,)]
    outs = []
    for use_payload in (False, True):
        torch.manual_seed(1)
        ps = [torch.nn.Parameter(torch.randn(s, device=DEV)) for s in shapes]
        opt = FusedBertAdam([{"params": ps[:2], "weight_decay": 0.01}, {"params": ps[2:], "weight_decay": 0.0}],
                            lr=1e-3, warmup=0.1, t_total=100, max_grad_norm=1.0, global_clip_norm=1.0, grad_scale=0.5)
        for t in range(3):
            gen = torch.Generator(device=DEV).manual_seed(10 + t)
            for i, p in enumerate(ps):
                g = torch.randn(p.shape, device=DEV, generator=gen).to(torch.bfloat16).float()
                p.grad = None if (i == 3 and t == 1) else g      # a tensor without gradient is skipped (sumsq == 0)
            if use_payload:
                if not opt._built:
                    opt._build()
                opt.g.zero_()                                      # (padding still holds the NaNs of the last round)
                opt._gather_grads()
                payload = opt.g.to(torch.bfloat16)
                assert torch.equal(payload.float(), opt.g)
                opt.g.fill_(float("nan"))                          # must not be read
                opt.grad_payload = payload
            opt.step()
            opt.grad_payload = None
        outs.append([p.detach().clone() for p in ps])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        opt.grad_payload = torch.zeros(3, device=DEV, dtype=torch.bfloat16)
        opt.step()


def test_fused_step_is_bitwise_repeatable_over_many_chunks():
    """the gradient norms (per-tensor and global clip) are per-chunk partial sums (adam_sumsq) added in chunk order
    (adam_tensor_sums): two optimizers on identical parameters and gradients end with identical bits in parameters and
    moments, over a flat buffer of 2.4M elements = 39 chunks of 64K, one tensor spanning 23 of them — also with SMs
    reserved for a concurrent collective"""
    from univl_b200 import runtime as rt
    from univl_b200.optim import FusedBertAdam
    shapes = [(1500, 1000), (300001,), (5, 7), (768, 768), (3,)]

    def run(reserve):
        torch.manual_seed(4)
        ps = [torch.nn.Parameter(torch.randn(s, device=DEV) * 0.1) for s in shapes]
        opt = FusedBertAdam([{"params": ps[:3], "weight_decay": 0.01}, {"params": ps[3:], "weight_decay": 0.0}],
                            lr=1e-3, warmup=0.1, t_total=100, max_grad_norm=1.0, global_clip_norm=1.0)
        rt.reserve_sms(reserve)
        try:
            for t in range(2):
                gen = torch.Generator(device=DEV).manual_seed(30 + t)
                for p in ps:
                    p.grad = torch.randn(p.shape, device=DEV, generator=gen) * (3.0 if t == 0 else 0.2)
                opt.step()
            torch.cuda.synchronize()
        finally:
            rt.reserve_sms(0)
        return [opt.p.clone(), opt.m.clone(), opt.v.clone()]
    base = run(0)
    assert base[0].numel() > 36 * 65536
    for reserve in (0, 40):
        for a, b in zip(base, run(reserve)):
            assert torch.equal(a, b), reserve
