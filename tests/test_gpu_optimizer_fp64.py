"""GPU: the fused BertAdam step (csrc/optim.cu) against the fp64 reference of tests/optim_check.py, per element, one
step at a time from the kernel's own state: p, m and v are read back after each step and the next step is checked from
them, so errors do not compound.  Every step also checks the sums of squares left in `scratch`, that the bf16 weight
copy (the shadow the GEMMs read) equals p rounded to bf16 bit for bit, and that the padding between tensors in p, m, v
and the shadow keeps the NaN it was filled with.

Covered: the schedule over warmup, the peak, decay and the clamp (and t_total = -1, warmup = -1 and 0); each clip
just below and above its threshold and disabled; grad_scale on both gradient paths; tensors of 1-7, 65535-65537 and
2 * 65536 + 3 elements; tensors skipped for want of a gradient; gradients so small that their squares flush to zero;
the model's full parameter list (more than 256 tensors) in the drivers' four groups; a CUDA-graph replay of the step;
and a model trained through its shadow against a fresh model built from its state_dict.

The fused step keeps ONE device step counter, where the reference keeps a `step` per parameter that advances only when
the parameter has a gradient.  test_partial_gradients_are_scheduled_at_the_optimizer_step pins the fused rule."""
import struct

import pytest
import torch

from oracle import synth
from tests import optim_check as oc
from tests.model_util import bert_dir, build_model, to_device
from univl_b200.runtime import call

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
SIZES = [1, 2, 3, 4, 5, 6, 7, 65535, 65536, 65537, 2 * 65536 + 3, 300 * 64]
GROUPS = [(1e-3, 0.01), (1e-4, 0.0), (5e-3, 0.1)]     # (lr, weight_decay), cycled over the tensors


def _align(n):
    return -(-n // 64) * 64


class Flat:
    """tensors laid out in flat buffers at 64-element offsets, as FusedBertAdam lays them, driven through the C ABI.
    Every padding element of p, m, v, the shadow and both gradient buffers holds NaN."""

    def __init__(self, sizes, seed=0, groups=GROUPS):
        self.sizes = sizes
        self.offs, total = [], 0
        for n in sizes:
            self.offs.append(total)
            total += _align(n)
        self.groups = [tuple(oc.f32(x) for x in groups[i % len(groups)]) for i in range(len(sizes))]
        bufs = {k: torch.full((total,), NAN, device=DEV) for k in ("p", "m", "v", "g")}
        self.p, self.m, self.v, self.g = bufs["p"], bufs["m"], bufs["v"], bufs["g"]
        self.shadow = torch.full((total,), NAN, device=DEV, dtype=torch.bfloat16)
        self.payload = torch.full((total,), NAN, device=DEV, dtype=torch.bfloat16)
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.pad = torch.ones(total, dtype=torch.bool, device=DEV)
        for i, n in enumerate(sizes):
            self.pad[self.offs[i]:self.offs[i] + n] = False
            self.seg(self.p, i).copy_(0.05 * torch.randn(n, device=DEV, generator=gen))
            self.seg(self.m, i).zero_()
            self.seg(self.v, i).zero_()
            self.seg(self.shadow, i).copy_(self.seg(self.p, i))
        rows = []
        for i, n in enumerate(sizes):
            lr, wd = self.groups[i]
            for c0 in range(0, n, oc.CHUNK):
                rows.append(struct.pack("<qiiffff", self.offs[i] + c0, min(oc.CHUNK, n - c0), i, lr, wd, 0.0, 0.0))
        self.segs = torch.frombuffer(bytearray(b"".join(rows)), dtype=torch.uint8).to(DEV)
        self.n_chunks = len(rows)
        self.scratch = torch.zeros(len(sizes) + 1, device=DEV)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=DEV)

    def seg(self, buf, i):
        return buf[self.offs[i]:self.offs[i] + self.sizes[i]]

    def launch(self, cfg, payload=False):
        c = cfg
        call("univl_bert_adam_step_bf16grad" if payload else "univl_bert_adam_step", self.p.data_ptr(),
             (self.payload if payload else self.g).data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
             self.shadow.data_ptr(), self.segs.data_ptr(), self.n_chunks, len(self.sizes), self.scratch.data_ptr(),
             self.step_dev.data_ptr(), c["b1"], c["b2"], c["eps"], c["max_grad_norm"], c["global_clip_norm"],
             c["warmup"], c["t_total"], c["grad_scale"])

    def step(self, grads, cfg, payload=False, what=""):
        """set the gradients (None: zeros), run one step and check it -> worst ratio per output"""
        buf = self.payload if payload else self.g
        read = []
        for i, n in enumerate(self.sizes):
            g = torch.zeros(n, device=DEV) if grads[i] is None else grads[i]
            self.seg(buf, i).copy_(g)
            read.append(self.seg(buf, i).float())
        before = [tuple(self.seg(b, i).clone() for b in (self.p, self.m, self.v)) for i in range(len(self.sizes))]
        step = int(self.step_dev.item())
        self.launch(cfg, payload)
        torch.cuda.synchronize()
        assert int(self.step_dev.item()) == step + 1
        after = [tuple(self.seg(b, i) for b in (self.p, self.m, self.v)) for i in range(len(self.sizes))]
        worst = oc.check_step(before, after, read, self.groups, step, cfg, self.scratch, what)
        for i in range(len(self.sizes)):
            oc.check_shadow(self.seg(self.shadow, i), self.seg(self.p, i), "%s t%d shadow" % (what, i))
        for name, b in (("p", self.p), ("m", self.m), ("v", self.v), ("shadow", self.shadow)):
            assert bool(torch.isnan(b[self.pad].float()).all()), "%s: padding of %s was written" % (what, name)
        return worst


def _merge(acc, worst):
    for k, x in worst.items():
        acc[k] = max(acc.get(k, 0.0), x)
    return acc


def _report(what, acc):
    print("worst %-40s %s" % (what, " ".join("%s %.3e" % kv for kv in sorted(acc.items()))))


def _grads(sizes, scale, gen, bf16=False, boost=None):
    """per-tensor gradients with norm about `scale` each (randn / sqrt(n)); tensor `boost` (index, factor) larger"""
    out = []
    for i, n in enumerate(sizes):
        s = scale * (boost[1] if boost is not None and boost[0] == i else 1.0)
        g = torch.randn(n, device=DEV, generator=gen) * (s / n ** 0.5)
        out.append(g.to(torch.bfloat16).float() if bf16 else g)
    return out


@pytest.mark.parametrize("payload", [False, True], ids=["fp32", "bf16_payload"])
def test_steps_from_kernel_state(payload):
    """12 steps, t_total 10, warmup 0.2: step 0 (lr 0), warmup, x = warmup (step 2), decay, x = 1 (step 10, lr 0) and
    past it (clamped).  Steps alternate between tripping the global clip, tripping no clip, and tripping the
    per-tensor clip on one tensor.  The bf16 payload path reads bf16 gradients scaled by grad_scale = 1/8."""
    gs = 0.125 if payload else 1.0
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=0.5, warmup=0.2, t_total=10, grad_scale=gs)
    f = Flat(SIZES, seed=1)
    gen = torch.Generator(device=DEV).manual_seed(2)
    acc = {}
    for t in range(12):
        scale, boost = [(3.0, None), (0.02, None), (0.25, (t % len(SIZES), 8.0))][t % 3]
        grads = _grads(SIZES, scale / gs, gen, bf16=payload, boost=boost)
        _merge(acc, f.step(grads, cfg, payload, "step %d" % t))
    _report("steps " + ("bf16" if payload else "fp32"), acc)


def _norm_to(g, target):
    return (g.double() * (target / g.double().norm())).float()


@pytest.mark.parametrize("case", ["global_below", "global_above", "tensor_below", "tensor_above", "disabled",
                                  "scaled_fp32"])
def test_clip_edges(case):
    """each clip's factor min(1, C / (norm + 1e-6)) just below and just above 1 (norm = (C - 1e-6)(1 -+ 1e-4)), both
    clips disabled (<= 0) under large gradients, and grad_scale 0.37 on the fp32 path"""
    sizes = [7, 4099, 65537, 300]
    gen = torch.Generator(device=DEV).manual_seed(3)
    grads = _grads(sizes, 0.2, gen)
    kw = dict(global_clip_norm=1.0, max_grad_norm=1.0, warmup=0.2, t_total=10)
    if case.startswith("global"):
        kw["max_grad_norm"] = -1.0
        target = (1.0 - 1e-6) * (1 + (1e-4 if case == "global_above" else -1e-4))
        total = torch.cat([g.double() for g in grads]).norm()
        grads = [_norm_to(g, float(g.double().norm() / total) * target) for g in grads]
    elif case.startswith("tensor"):
        kw["global_clip_norm"] = -1.0
        grads[2] = _norm_to(grads[2], (1.0 - 1e-6) * (1 + (1e-4 if case == "tensor_above" else -1e-4)))
    elif case == "disabled":
        kw.update(global_clip_norm=-1.0, max_grad_norm=0.0)
        grads = [g * 250.0 for g in grads]
    else:
        kw["grad_scale"] = 0.37
        grads = [g * 20.0 for g in grads]
    cfg = oc.kernel_cfg(**kw)
    f = Flat(sizes, seed=4)
    acc = {}
    for t in range(3):
        f.step_dev.fill_(4 + t)
        _merge(acc, f.step(grads, cfg, what="%s step %d" % (case, t)))
    _report("clip " + case, acc)


@pytest.mark.parametrize("warmup,t_total,steps", [
    (0.1, 100, [0, 1, 9, 10, 11, 99, 100, 101, 250]),
    (-1.0, 20, [0, 7, 19, 20, 25]),
    (0.0, 50, [0, 1, 49, 50]),
    (0.1, -1, [0, 3, 1000]),
], ids=["warmup0.1", "warmup-1", "warmup0", "t_total-1"])
def test_schedule_edges(warmup, t_total, steps):
    """the device step counter set to each edge of warmup_linear: step 0 (lr 0), x = warmup, x >= 1 (clamped to 0),
    the reference's (1 - x) / 2 rule for warmup = -1, and a constant lr for t_total = -1"""
    sizes = [5, 1000, 65537]
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=1.0, warmup=warmup, t_total=t_total)
    f = Flat(sizes, seed=5)
    gen = torch.Generator(device=DEV).manual_seed(6)
    acc = {}
    for s in steps:
        f.step_dev.fill_(s)
        p0 = f.p[~f.pad].clone()
        _merge(acc, f.step(_grads(sizes, 0.3, gen), cfg, what="step %d" % s))
        if oc.warmup_linear64(s, t_total, cfg["warmup"])[0] == 0.0:
            assert torch.equal(f.p[~f.pad], p0), "lr 0 moved p at step %d" % s
    _report("schedule w=%g T=%d" % (warmup, t_total), acc)


@pytest.mark.parametrize("payload", [False, True], ids=["fp32", "bf16_payload"])
def test_tiny_gradient_is_a_gradient(payload):
    """gradients of about 1e-20 square to below 2^-126 and flush to zero under fast math, so their sum of squares is 0:
    the tensor must still be updated (its moments move and weight decay applies, which dominates its update) while a
    tensor whose gradient is exactly zero is skipped, as the reference skips a parameter without a gradient"""
    gs = 0.125 if payload else 1.0
    sizes = [1000, 1000, 4099]
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=1.0, warmup=0.1, t_total=100, grad_scale=gs)
    f = Flat(sizes, seed=7, groups=[(1e-3, 0.01)])
    gen = torch.Generator(device=DEV).manual_seed(8)
    for t in range(2):
        f.step_dev.fill_(20 + t)
        tiny = torch.randn(1000, device=DEV, generator=gen) * 1e-20
        normal = torch.randn(4099, device=DEV, generator=gen) * 0.01
        if payload:
            tiny, normal = tiny.to(torch.bfloat16).float(), normal.to(torch.bfloat16).float()
        p0 = [f.seg(f.p, i).clone() for i in range(3)]
        m0 = f.seg(f.m, 0).clone()
        f.step([tiny, None, normal], cfg, payload, "tiny step %d" % t)
        assert float(f.scratch[0]) == 0.0                       # the squares did flush
        assert not torch.equal(f.seg(f.p, 0), p0[0]), "tiny-gradient tensor was skipped"
        assert torch.equal(f.seg(f.p, 1), p0[1])
        assert not torch.equal(f.seg(f.m, 0), m0)
        lr, wd = f.groups[0]
        lr = lr * oc.warmup_linear64(20 + t, 100, cfg["warmup"])[0]
        decay = lr * wd * p0[0].double()
        d = p0[0].double() - f.seg(f.p, 0).double()
        assert bool(((d - decay).abs() <= 1e-3 * decay.abs() + 2 * oc.U * p0[0].double().abs()).all())


def test_partial_gradients_are_scheduled_at_the_optimizer_step():
    """a tensor with gradients on steps 0, 1 and 3 only: it is skipped on step 2, and on step 3 the fused step
    schedules it at the optimizer's count (3), where the reference's per-parameter count would be 2.  This pins the
    documented difference: the check at step 2 rejects the kernel's update."""
    sizes = [1000, 1000]
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=1.0, warmup=0.5, t_total=10)
    f = Flat(sizes, seed=9, groups=[(1e-3, 0.01)])
    gen = torch.Generator(device=DEV).manual_seed(10)
    for t in range(3):
        grads = _grads(sizes, 0.3, gen)
        if t == 2:
            grads[1] = None
        f.step(grads, cfg, what="partial step %d" % t)
    grads = _grads(sizes, 0.3, gen)
    for i in range(2):
        f.seg(f.g, i).copy_(grads[i])
    before = [tuple(f.seg(b, i).clone() for b in (f.p, f.m, f.v)) for i in range(2)]
    f.launch(cfg)
    torch.cuda.synchronize()
    after = [tuple(f.seg(b, i) for b in (f.p, f.m, f.v)) for i in range(2)]
    oc.check_step(before, after, grads, f.groups, 3, cfg, f.scratch, "optimizer count")
    S, b_S, T, b_T = oc.sums64(grads, 1.0, sizes)
    gmul, d_gmul, _, _ = oc.clip64(S, b_S, T, b_T, cfg)
    sched, e_sched = oc.warmup_linear64(2, cfg["t_total"], cfg["warmup"])
    own = oc.update64(*before[1], grads[1], float(gmul[1]), float(d_gmul[1]), *f.groups[1], sched, e_sched, cfg)
    (p0, m0, v0), (p1, m1, v1) = before[1], after[1]
    with pytest.raises(AssertionError, match="update"):
        oc.check_tensor(p0, p1, m0, m1, v0, v1, own, "t1 at its own step count")


def test_graph_replay_matches_eager_steps():
    """one captured step replayed 5 times equals 5 eager steps bit for bit: the device step counter drives the
    schedule through warmup (t_total 10, warmup 0.3) inside the graph"""
    sizes = [3, 4099, 65537]
    cfg = oc.kernel_cfg(global_clip_norm=1.0, max_grad_norm=0.5, warmup=0.3, t_total=10)
    gen = torch.Generator(device=DEV).manual_seed(11)
    grads = _grads(sizes, 2.0, gen)
    eager, graphed = Flat(sizes, seed=12), Flat(sizes, seed=12)
    for f in (eager, graphed):
        for i in range(len(sizes)):
            f.seg(f.g, i).copy_(grads[i])
    for _ in range(5):
        eager.launch(cfg)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.launch(cfg)
    assert int(graphed.step_dev.item()) == 0
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert int(graphed.step_dev.item()) == 5
    for name in ("p", "m", "v", "shadow", "scratch"):
        a, b = getattr(eager, name), getattr(graphed, name)
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32)), name


def _driver_groups(model):
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    dec = [(n, p) for n, p in named if not any(nd in n for nd in no_decay)]
    nod = [(n, p) for n, p in named if any(nd in n for nd in no_decay)]
    lr, coef = 3e-5, 0.1
    return [{"params": [p for n, p in dec if "bert." in n], "weight_decay": 0.01, "lr": lr * coef},
            {"params": [p for n, p in dec if "bert." not in n], "weight_decay": 0.01},
            {"params": [p for n, p in nod if "bert." in n], "weight_decay": 0.0, "lr": lr * coef},
            {"params": [p for n, p in nod if "bert." not in n], "weight_decay": 0.0}]


def test_model_trained_through_its_shadow_equals_a_fresh_model():
    """an FT-Align model (dropout 0) trained 3 steps by FusedBertAdam(model=...) runs its forward GEMMs on the shadow
    the update kernel wrote; a fresh model built from its state_dict casts its arena from the same fp32 values.  Their
    next step's loss and every gradient agree bit for bit."""
    from univl_b200.optim import FusedBertAdam
    cfg = synth.task_config(mode="ft_align", batch_size=4, text_layers=2, visual_layers=1, cross_layers=1,
                            max_words=16, max_frames=12)
    batch = to_device(synth.make_batch(cfg, seed=13))
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=14), dropout=0.0)
    opt = FusedBertAdam(_driver_groups(model), lr=1e-3, warmup=0.1, t_total=20, max_grad_norm=1.0,
                        global_clip_norm=1.0, model=model)
    for _ in range(3):
        opt.zero_grad()
        model(**batch).backward()
        opt.step()
    torch.cuda.synchronize()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    fresh = build_model(cfg, sd=sd, dropout=0.0)
    opt2 = FusedBertAdam(_driver_groups(fresh), lr=1e-3, warmup=0.1, t_total=20, max_grad_norm=1.0,
                         global_clip_norm=1.0, model=fresh)
    opt2._build()
    assert torch.equal(opt.p, opt2.p)
    assert torch.equal(opt.shadow.view(torch.int16), opt2.shadow.view(torch.int16))
    losses = []
    for m, o in ((model, opt), (fresh, opt2)):
        o.zero_grad()
        loss = m(**batch)
        loss.backward()
        losses.append(loss.detach().clone())
    torch.cuda.synchronize()
    assert torch.equal(losses[0], losses[1])
    assert float(opt.g.abs().max()) > 0
    assert torch.equal(opt.g, opt2.g)


def test_full_parameter_list():
    """the BASELINE configuration's parameters, flattened through model= in the drivers' four groups: more than 256
    tensors, so adam_tensor_sums runs more than one block and adam_total's strided loop takes several tensors per
    thread.  The sums in scratch and every element of every tensor are checked, at a warmup and a decay step."""
    from univl_b200.modules.modeling import UniVL
    from univl_b200.optim import FusedBertAdam
    cfg = synth.task_config(mode="ft_align", batch_size=32, max_words=48, max_frames=48)
    torch.manual_seed(0)
    model = UniVL.from_pretrained(bert_dir(), "visual-base", "cross-base", "decoder-base", task_config=cfg).to(DEV)
    opt = FusedBertAdam(_driver_groups(model), lr=3e-5, warmup=0.1, t_total=100000, max_grad_norm=1.0,
                        global_clip_norm=1.0, model=model)
    opt._build()
    assert opt.n_tensors > 256, opt.n_tensors
    ckw = dict(b1=0.9, b2=0.999, eps=1e-6, max_grad_norm=1.0, global_clip_norm=1.0, warmup=0.1, t_total=100000)
    kcfg = oc.kernel_cfg(**ckw)
    segs, groups = [], []
    for grp in opt.param_groups:
        for p in grp["params"]:
            off, n, _ = opt._lookup[id(p)]
            segs.append((off, n))
            groups.append((oc.f32(grp["lr"]), oc.f32(grp["weight_decay"])))
    gen = torch.Generator(device=DEV).manual_seed(15)
    acc = {}
    for t, step in enumerate((7000, 60000)):
        opt.zero_grad()
        for i, (off, n) in enumerate(segs):
            if i % 97 != 5:                       # a few tensors without a gradient
                opt.g[off:off + n].copy_(torch.randn(n, device=DEV, generator=gen) * (0.05 / n ** 0.5))
        opt.step_dev.fill_(step)
        before = [(opt.p[o:o + n].clone(), opt.m[o:o + n].clone(), opt.v[o:o + n].clone()) for o, n in segs]
        opt.step()
        torch.cuda.synchronize()
        after = [(opt.p[o:o + n], opt.m[o:o + n], opt.v[o:o + n]) for o, n in segs]
        grads = [opt.g[o:o + n] for o, n in segs]
        _merge(acc, oc.check_step(before, after, grads, groups, step, kcfg, opt.scratch, "model step %d" % t))
        for i, (o, n) in enumerate(segs):
            oc.check_shadow(opt.shadow[o:o + n], opt.p[o:o + n], "model t%d shadow" % i)
        del before, after
    _report("full parameter list (%d tensors)" % opt.n_tensors, acc)
