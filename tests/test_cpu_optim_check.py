"""CPU: the fp64 reference of the fused BertAdam step (tests/optim_check.py) against the reference's own BertAdam class
(tests/golden/ref_bert_adam*.pt, four steps in the drivers' four parameter groups), a float32 emulation of
csrc/optim.cu within every bound, and each negative check's perturbation outside its bound."""
import numpy as np
import pytest
import torch

from oracle import synth
from tests import optim_check as oc
from tests.oracle_util import load_golden

f32 = np.float32
BIG = "decoder.classifier.cls.predictions.bias"


# ---------------------------------------------------------------------------------------------------------
# float32 emulation of csrc/optim.cu (the kernel's operation order; IEEE sqrt and division stand in for the
# approximate ones, which the bounds cover with room)
# ---------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _butterfly_block(acc):
    """256 per-thread values -> the block sum: warp_sum (xor butterfly) in each warp, then the 8 warps in order"""
    w = acc.reshape(8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, lanes ^ o]).astype(f32)
    t = f32(0)
    for k in range(8):
        t = f32(t + w[k, 0])
    return t


def _chunk_sumsq(x, gs):
    """adam_sumsq_kernel on one chunk: thread i takes elements 4i + 1024k in 4-term groups, squares scaled by gs twice"""
    n = x.size
    pad = np.zeros(-(-n // 1024) * 1024, f32)
    pad[:n] = x
    grp = pad.reshape(-1, 256, 4)
    s = (grp[..., 0] * grp[..., 0]).astype(f32)
    for j in (1, 2, 3):
        s = _fma(grp[..., j], grp[..., j], s)
    s = ((s * gs).astype(f32) * gs).astype(f32)
    acc = np.zeros(256, f32)
    for k in range(s.shape[0]):
        acc = (acc + s[k]).astype(f32)
    return _butterfly_block(acc)


def emulate32(ps, ms, vs, grads, groups, step, cfg, shadow_trunc=False):
    """-> (p', m', v', shadow') lists of float32 arrays and the scratch [n + 1] the kernel leaves"""
    gs = f32(cfg["grad_scale"])
    S = []
    for p, g in zip(ps, grads):
        g = np.zeros(p.size, f32) if g is None else g
        t = f32(0)
        for c0 in range(0, g.size, oc.CHUNK):
            t = f32(t + _chunk_sumsq(g[c0:c0 + oc.CHUNK], gs))
        S.append(t)
    S = np.array(S, f32)
    acc = np.zeros(256, f32)
    for i in range(len(S)):
        acc[i % 256] = f32(acc[i % 256] + S[i])
    T = _butterfly_block(acc)
    cg = f32(1)
    if cfg["global_clip_norm"] > 0:
        cg = min(f32(1), f32(f32(cfg["global_clip_norm"]) / f32(np.sqrt(T) + f32(oc.CLIP_EPS))))
    sched = f32(1)
    if cfg["t_total"] > 0:
        x, w = f32(step / cfg["t_total"]), f32(cfg["warmup"])
        sched = f32(x / w) if (w >= 0 and x < w) else max(f32(f32(x - 1) / f32(w - 1)), f32(0))
    b1, b2, eps = f32(cfg["b1"]), f32(cfg["b2"]), f32(cfg["eps"])
    outs = ([], [], [], [])
    for i, (p, m, v, g) in enumerate(zip(ps, ms, vs, grads)):
        lr_g, wd = f32(groups[i][0]), f32(groups[i][1])
        if g is None or not (g != 0).any():
            for o, x in zip(outs, (p, m, v, None)):
                o.append(x if x is not None else _bf16(p, shadow_trunc))
            continue
        ct = f32(1)
        if cfg["max_grad_norm"] > 0:
            ct = min(f32(1), f32(f32(cfg["max_grad_norm"]) / _fma(np.sqrt(S[i]), cg, f32(oc.CLIP_EPS))))
        gmul = f32(f32(gs * cg) * ct)
        lr = f32(lr_g * sched)
        gh = (g * gmul).astype(f32)
        m1 = _fma(b1, m, ((f32(1) - b1) * gh).astype(f32))
        v1 = _fma(b2, v, ((gh * (f32(1) - b2)).astype(f32) * gh).astype(f32))
        q = (m1 / (np.sqrt(v1) + eps).astype(f32)).astype(f32)
        u = _fma(wd, p, q)
        p1 = _fma(-lr, u, p)
        for o, x in zip(outs, (p1, m1, v1, _bf16(p1, shadow_trunc))):
            o.append(x)
    return outs + (np.concatenate([S, [T]]).astype(f32),)


def _bf16(p, trunc):
    """p -> bf16 bits as torch: round to nearest even (the kernel's pack_bf16x2 / __float2bfloat16), or toward zero"""
    t = torch.from_numpy(np.ascontiguousarray(p))
    if trunc:
        return ((t.view(torch.int32) >> 16) << 16).view(torch.float32).to(torch.bfloat16)
    return t.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------
SIZES = [1, 3, 7, 300, 4099, 65536 + 3]
GROUPS = [(1e-3, 0.01), (2e-4, 0.0), (5e-3, 0.1), (1e-3, 0.01), (2e-4, 0.0), (5e-3, 0.1)]


def _case(seed=0, gscale=(1.0,) * len(SIZES), bf16=False):
    """state after a few steps (nonzero moments) and one gradient per tensor; gscale sets each tensor's gradient size"""
    rng = np.random.default_rng(seed)
    ps = [(0.05 * rng.standard_normal(n)).astype(f32) for n in SIZES]
    ms = [(1e-2 * rng.standard_normal(n)).astype(f32) for n in SIZES]
    vs = [(1e-4 * rng.random(n) + 1e-6).astype(f32) for n in SIZES]
    gr = []
    for n, s in zip(SIZES, gscale):
        g = (s * rng.standard_normal(n)).astype(f32)
        if bf16:
            g = torch.from_numpy(g).to(torch.bfloat16).float().numpy()
        gr.append(g)
    groups = [(oc.f32(lr), oc.f32(wd)) for lr, wd in GROUPS]
    return ps, ms, vs, gr, groups


def _t(xs):
    return [None if x is None else torch.from_numpy(np.asarray(x)) for x in xs]


def _check_all(ps, ms, vs, grads, groups, step, cfg, got, eps_inside=False):
    p1, m1, v1, sh, scratch = got
    ref = oc.step64(_t(ps), _t(ms), _t(vs), _t(grads), groups, step, cfg, eps_inside=eps_inside)
    ratios = [oc.check_sums(torch.from_numpy(scratch), ref, "sums")]
    for i in range(len(ps)):
        ratios.append(oc.check_tensor(*_t([ps[i], p1[i], ms[i], m1[i], vs[i], v1[i]]), ref["t"][i], "t%d" % i))
        oc.check_shadow(sh[i], torch.from_numpy(p1[i]), "t%d shadow" % i)
    return ref, ratios


CFGS = {
    "clips": dict(global_clip_norm=1.0, max_grad_norm=0.5, warmup=0.1, t_total=100),
    "no_clip": dict(global_clip_norm=-1.0, max_grad_norm=0.0, warmup=0.1, t_total=100),
    "scaled": dict(global_clip_norm=1.0, max_grad_norm=1.0, warmup=0.1, t_total=100, grad_scale=0.37),
    "decay_w-1": dict(global_clip_norm=1.0, max_grad_norm=1.0, warmup=-1, t_total=20),
    "const_lr": dict(global_clip_norm=1.0, max_grad_norm=1.0, t_total=-1),
}


@pytest.mark.parametrize("name", sorted(CFGS))
@pytest.mark.parametrize("step", [0, 3, 10, 57, 100, 130])
def test_float32_emulation_is_within_bounds(name, step):
    cfg = oc.kernel_cfg(**CFGS[name])
    case = _case(seed=step, gscale=(0.02, 0.05, 3.0, 0.01, 0.02, 0.003))
    got = emulate32(*case, step, cfg)
    ref, ratios = _check_all(*case, step, cfg, got)
    # the sums and moments sit well inside their bounds; the update can reach 1 where p''s own rounding dominates it
    worst = max(max(r[:2]) for r in ratios)
    assert worst < 0.5, worst


def test_bf16_gradients_and_a_zero_gradient_tensor():
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=1.0, warmup=0.1, t_total=100, grad_scale=0.125)
    ps, ms, vs, gr, groups = _case(seed=5, bf16=True)
    gr[1] = np.zeros_like(gr[1])
    gr[3] = None
    got = emulate32(ps, ms, vs, gr, groups, 20, cfg)
    ref, _ = _check_all(ps, ms, vs, gr, groups, 20, cfg, got)
    assert ref["t"][1] is None and ref["t"][3] is None and ref["t"][0] is not None


def test_schedule_edges():
    s, _ = oc.warmup_linear64(0, 100, oc.f32(0.1))
    assert s == 0.0
    s, _ = oc.warmup_linear64(100, 100, oc.f32(0.1))
    assert s == 0.0
    s, _ = oc.warmup_linear64(150, 100, oc.f32(0.1))
    assert s == 0.0
    s, e = oc.warmup_linear64(10, 100, oc.f32(0.1))          # x = w (up to fp32(0.1)): the peak from either branch
    assert abs(s - 1) < 1e-7 and e < 1e-5
    s, _ = oc.warmup_linear64(5, 20, -1.0)
    assert s == pytest.approx((1 - 0.25) / 2)
    assert oc.warmup_linear64(12345, -1, 0.1) == (1.0, 0.0)


# ---------------------------------------------------------------------------------------------------------
# against the reference's own class
# ---------------------------------------------------------------------------------------------------------
def test_reference_matches_reference_class_golden():
    """each golden step from the previous golden state: the reference class's fp32 rounds the product b1 m on its own
    and multiplies the gradient by each clip factor in place, so it is held to twice the kernel's bound.  The long
    tensor is stored as head / tail slices: its update is elementwise once the norms (from its full gradient) are
    known."""
    gold = load_golden("bert_adam")
    names_shapes, init, grads, no_grad = synth.adam_case(len(gold["after"]))
    names = [n for n, _ in names_shapes]
    lr, coef = gold["lr"], gold["coef_lr"]
    groups = [(lr * coef if n.startswith("bert.") else lr,
               0.0 if any(nd in n for nd in gold["no_decay"]) else gold["weight_decay"]) for n in names]
    cfg = dict(b1=0.9, b2=0.999, eps=1e-6, max_grad_norm=gold["max_grad_norm"], global_clip_norm=gold["global_clip"],
               warmup=gold["warmup"], t_total=gold["t_total"], grad_scale=1.0)
    n_big = init[BIG].numel()
    slices = {n: {"all": slice(None)} for n in names}
    slices[BIG] = {"head": slice(0, 256), "tail": slice(n_big - 256, None)}
    state = {n: {k: (init[n].flatten()[sl], torch.zeros(init[n].numel())[sl], torch.zeros(init[n].numel())[sl])
                 for k, sl in slices[n].items()} for n in names}

    def part(x, k):
        return x[k] if isinstance(x, dict) else x.flatten()

    worst = 0.0
    for t, after in enumerate(gold["after"]):
        gr = [None if n in no_grad else grads[t][n].flatten() for n in names]
        S, b_S, T, b_T = oc.sums64(gr, 1.0, [init[n].numel() for n in names])
        gmul, d_gmul, _, _ = oc.clip64(S, b_S, T, b_T, cfg)
        sched, e_sched = oc.warmup_linear64(t, cfg["t_total"], cfg["warmup"])
        for i, n in enumerate(names):
            if n in no_grad:
                assert torch.equal(after["params"][n], init[n]) and n not in after["next_m"]
                continue
            for k, sl in slices[n].items():
                p0, m0, v0 = state[n][k]
                r = oc.update64(p0, m0, v0, gr[i][sl], float(gmul[i]), float(d_gmul[i]), groups[i][0], groups[i][1],
                                sched, e_sched, cfg)
                what = "step %d %s %s" % (t + 1, n, k)
                p1, m1, v1 = (part(after[key][n], k) for key in ("params", "next_m", "next_v"))
                worst = max(worst, oc.within(m1, r["m"], 2 * r["b_m"], what + " m"),
                            oc.within(v1, r["v"], 2 * r["b_v"], what + " v"),
                            oc.within(p0.double() - p1.double(), r["d"], 2 * r["b_d"], what + " update"))
                state[n][k] = (p1, m1, v1)
    assert worst < 1


# ---------------------------------------------------------------------------------------------------------
# negative checks: a kernel with each bug, emulated, falls outside the bounds
# ---------------------------------------------------------------------------------------------------------
def _rejected(fn):
    with pytest.raises(AssertionError):
        fn()


def _neg_case():
    # global clip inactive, the per-tensor clip active on tensor 2
    return oc.kernel_cfg(global_clip_norm=100.0, max_grad_norm=0.5, warmup=0.1, t_total=100), \
        _case(seed=9, gscale=(0.02, 0.05, 3.0, 0.01, 0.02, 0.003))


@pytest.mark.parametrize("step", [4, 60])
def test_schedule_one_step_off_is_rejected(step):
    cfg, case = _neg_case()
    got = emulate32(*case, step + 1, cfg)
    _rejected(lambda: _check_all(*case, step, cfg, got))


def test_swapped_betas_are_rejected():
    cfg, case = _neg_case()
    bad = dict(cfg, b1=cfg["b2"], b2=cfg["b1"])
    got = emulate32(*case, 30, bad)
    _rejected(lambda: _check_all(*case, 30, cfg, got))


def test_eps_inside_the_sqrt_is_rejected():
    """the kernel against a reference with eps inside the sqrt (the emulation cannot move eps without a flag)"""
    cfg, case = _neg_case()
    got = emulate32(*case, 30, cfg)
    _check_all(*case, 30, cfg, got)
    _rejected(lambda: _check_all(*case, 30, cfg, got, eps_inside=True))


def test_missing_per_tensor_clip_is_rejected():
    cfg, case = _neg_case()
    ref = oc.step64(*[_t(x) for x in case[:4]], case[4], 30, cfg)
    assert float(oc.clip64(ref["S"], ref["b_S"], ref["T"], ref["b_T"], cfg)[3][2]) < 0.5   # tensor 2 is clipped
    got = emulate32(*case, 30, dict(cfg, max_grad_norm=oc.f32(-1.0)))
    _rejected(lambda: _check_all(*case, 30, cfg, got))


def test_weight_decay_on_the_wrong_group_is_rejected():
    cfg, case = _neg_case()
    ps, ms, vs, gr, groups = case
    swapped = [(lr, groups[(i + 1) % len(groups)][1]) for i, (lr, _) in enumerate(groups)]
    got = emulate32(ps, ms, vs, gr, swapped, 30, cfg)
    _rejected(lambda: _check_all(ps, ms, vs, gr, groups, 30, cfg, got))


def test_shadow_rounded_toward_zero_is_rejected():
    cfg, case = _neg_case()
    got = emulate32(*case, 30, cfg, shadow_trunc=True)
    _rejected(lambda: _check_all(*case, 30, cfg, got))
