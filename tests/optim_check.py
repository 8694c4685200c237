"""fp64 reference and per-element bounds of the fused BertAdam step (csrc/optim.cu): the driver's global clip, the
per-tensor clip, grad_scale, the moments without bias correction, eps outside the sqrt, decoupled weight decay,
warmup_linear at the device step and the skip rule.  Shared by tests/test_gpu_optimizer_fp64.py and validated on CPU
by tests/test_cpu_optim_check.py, which also holds the float32 emulation of the kernel used there.

Bounds are derived from the kernel's fp32 --use_fast_math arithmetic in the style of tests/row_check.py: U = 2^-24 per
rounding; sqrtf is MUFU.SQRT (sqrt.approx.f32, relative error 2^-23 in the PTX ISA; SQRT_REL leaves a factor 2) and
a / b is a reciprocal approximation times a (div.approx.f32, 2 ulp: DIV_REL); contraction into FMAs only removes
roundings; fp32 results below 2^-126 may flush to zero (FTZ_ABS).  The functions take and return torch tensors on any
device; all work is in fp64.

The reference keeps a `step` per parameter and advances it only for parameters that have a gradient; the fused step
keeps one device counter for all tensors.  `step64` takes that one counter: a tensor that receives gradients on only
some steps is scheduled at the optimizer's step count (tests/test_gpu_optimizer_fp64.py pins this)."""
import math

import numpy as np
import torch

from tests.gemm_check import U, within  # noqa: F401  (within: re-exported for the tests)
from tests.row_check import DIV_REL, FTZ_ABS

SQRT_REL = 4 * U
CLIP_EPS = float(np.float32(1e-6))   # the clip denominators' 1e-6f
CHUNK = 65536                        # elements per chunk (one CTA of adam_sumsq / adam_update)
THREADS = 256


def f32(x):
    return float(np.float32(x))


def kernel_cfg(b1=0.9, b2=0.999, eps=1e-6, max_grad_norm=1.0, global_clip_norm=-1.0, warmup=-1.0, t_total=-1,
               grad_scale=1.0):
    """the hyperparameters as univl_bert_adam_step receives them (floats rounded to fp32)"""
    return dict(b1=f32(b1), b2=f32(b2), eps=f32(eps), max_grad_norm=f32(max_grad_norm),
                global_clip_norm=f32(global_clip_norm), warmup=f32(warmup), t_total=int(t_total),
                grad_scale=f32(grad_scale))


def _gamma(k):
    return k * U / (1 - k * U)


# ---------------------------------------------------------------------------------------------------------
# schedule
# ---------------------------------------------------------------------------------------------------------
def warmup_linear64(step, t_total, warmup):
    """(schedule factor, its bound) at device step `step`.  warmup_linear(x, w) = x / w if x < w else
    max((x - 1) / (w - 1), 0), x = step / t_total; 1 when t_total <= 0 (the reference's t_total = -1).  warmup < 0 never
    takes the first branch, so w = -1 gives the reference's (1 - x) / 2.
    The kernel rounds x to float (U x) and evaluates either branch with a rounded subtraction or two and one division.
    The function is continuous (both branches are 1 at x = w, and 0 at x = 1 under the clamp), so the rounding of x
    moves it by at most its steepest slope times U x, whichever branch the float x falls in."""
    if t_total <= 0:
        return 1.0, 0.0
    x = step / t_total
    w = warmup
    s = x / w if (w >= 0 and x < w) else max((x - 1) / (w - 1), 0.0)
    slope = 1 / abs(w - 1)
    if w > 0:
        slope = max(slope, 1 / w)
    return s, slope * U * x + (3 * U + DIV_REL) * s


# ---------------------------------------------------------------------------------------------------------
# gradient norms (adam_sumsq_kernel -> adam_tensor_sums_kernel -> adam_total_kernel)
# ---------------------------------------------------------------------------------------------------------
def sum_depth(n):
    """roundings on the path of one element's square into its tensor's sum: the 4-term group (one product and three
    FMAs), two multiplies by grad_scale, up to 64 groups per thread, the 5-level warp butterfly, 8 warps, then the
    tensor's chunks in order"""
    per_thread = -(-min(n, CHUNK) // (4 * THREADS))
    return 4 + 2 + per_thread + 5 + 8 + -(-n // CHUNK)


def sums64(grads, grad_scale, counts):
    """per-tensor sums of squares of the scaled gradients and their total, with bounds.  grads: list of 1-D tensors
    (None: no gradient, counted as zeros); counts: elements per tensor.
    Returns S [n], b_S [n], T, b_T (fp64 tensors on the gradients' device).
    Every term is nonnegative, so a sum taken in a fixed order of depth k errs by at most gamma(k) of its value; each
    flushed square or partial loses under 2^-126 (8 per element covers the group's intermediates)."""
    dev = next((g.device for g in grads if g is not None), torch.device("cpu"))
    S = torch.zeros(len(grads), dtype=torch.float64, device=dev)
    for i, g in enumerate(grads):
        if g is not None:
            S[i] = ((g.double() * grad_scale) ** 2).sum()
    counts = torch.tensor(counts, dtype=torch.float64, device=dev)
    depth = torch.tensor([sum_depth(int(n)) for n in counts.tolist()], dtype=torch.float64, device=dev)
    b_S = _gamma(depth) * S + 8 * counts * FTZ_ABS
    T = S.sum()
    k_tot = float(depth.max()) + -(-len(grads) // THREADS) + 5 + 8
    b_T = _gamma(k_tot) * T + 8 * counts.sum() * FTZ_ABS
    return S, b_S, T, b_T


# ---------------------------------------------------------------------------------------------------------
# clip factors
# ---------------------------------------------------------------------------------------------------------
def _sqrt_err(x, e):
    """bound of |sqrt.approx(x~) - sqrt(x)| for |x~ - x| <= e (x, e >= 0)"""
    lo = (x - e).clamp_min(0.0) if torch.is_tensor(x) else max(x - e, 0.0)
    sq = torch.sqrt if torch.is_tensor(x) else math.sqrt
    return (sq(x) - sq(lo)) + SQRT_REL * sq(x + e)


def clip64(S, b_S, T, b_T, cfg):
    """gradient multipliers grad_scale * cg * ct per tensor and their relative bounds.
    cg = min(1, C / (sqrt(T) + 1e-6)) (C = global_clip_norm > 0, else 1); ct = min(1, M / (cg sqrt(S_t) + 1e-6))
    (M = max_grad_norm > 0, else 1): the per-tensor clip sees the globally clipped gradient, as the reference's
    per-parameter clip_grad_norm_ runs after the driver's.  min(1, r) moves by no more than r's relative error, so a
    factor near its threshold is bounded the same on either side."""
    T = torch.as_tensor(T, dtype=torch.float64)
    cg, d_cg = torch.ones_like(T), torch.zeros_like(T)
    if cfg["global_clip_norm"] > 0:
        den = torch.sqrt(T) + CLIP_EPS
        e_den = _sqrt_err(T, b_T) + U * den * (1 + U)
        cg = torch.clamp(cfg["global_clip_norm"] / den, max=1.0)
        d_cg = e_den / (den - e_den) * (1 + DIV_REL) + DIV_REL
    ct, d_ct = torch.ones_like(S), torch.zeros_like(S)
    if cfg["max_grad_norm"] > 0:
        rt = torch.sqrt(S)
        den = cg * rt + CLIP_EPS                       # one FMA
        e_den = cg * (_sqrt_err(S, b_S) + d_cg * (rt + _sqrt_err(S, b_S))) + U * den * (1 + 4 * U)
        ct = torch.clamp(cfg["max_grad_norm"] / den, max=1.0)
        d_ct = e_den / (den - e_den) * (1 + DIV_REL) + DIV_REL
    gmul = cfg["grad_scale"] * cg * ct
    d_gmul = (1 + d_cg) * (1 + d_ct) * (1 + U) ** 2 - 1   # two roundings: grad_scale * cg * ct
    return gmul, d_gmul, cg, ct


# ---------------------------------------------------------------------------------------------------------
# one fused step
# ---------------------------------------------------------------------------------------------------------
def update64(p, m, v, g, gmul, d_gmul, lr, wd, sched, e_sched, cfg, eps_inside=False):
    """fp64 element update of one tensor (any slice of it) and the bound of every output.
    p, m, v: the kernel's state before the step; g: the gradient values it reads (fp32 or bf16).
    Returns dict m, b_m, v, b_v, d, b_d with d = p - p' the update p received: lr sched (m' / (sqrt v' + eps) + wd p).
    eps_inside: m' / sqrt(v' + eps) (a perturbation for the negative checks, not the kernel's statement).

    Kernel, per element: g~ = g gmul~ (U); m' = fma(b1, m, round((1 - b1) g~)); v' = fma(b2, v, round(round(g~ (1 - b2))
    g~)); q = m' rcp(sqrt(v') + eps); p' = p - lr~ (q + wd p) with lr~ = round(lr sched~), at most two roundings for
    the last line.  The bounds also allow b1 m and b2 v to be rounded on their own (no contraction).  d is checked instead of p', with p''s own rounding U |p'| in the bound, so an update far below
    ulp(p) is still held to its own relative accuracy."""
    p, m, v, g = p.double(), m.double(), v.double(), g.double()
    b1, b2, eps = cfg["b1"], cfg["b2"], cfg["eps"]
    c1, c2 = 1 - b1, 1 - b2                           # the kernel's 1.f - b: exact for b in [0.5, 1], else U
    gh = g * gmul
    e_gh = gh.abs() * (d_gmul + U) + FTZ_ABS
    m1 = b1 * m + c1 * gh
    e_m = c1 * e_gh + 3 * U * c1 * gh.abs() + U * (b1 * m.abs() + m1.abs() + c1 * e_gh) + FTZ_ABS
    v1 = b2 * v + c2 * gh * gh
    e_v = c2 * (2 * gh.abs() * e_gh + e_gh * e_gh) + 4 * U * c2 * gh * gh + U * (b2 * v + v1) + 2 * FTZ_ABS
    if eps_inside:
        den = torch.sqrt(v1 + eps)
    else:
        den = torch.sqrt(v1) + eps
    e_den = _sqrt_err(v1, e_v) + U * (den + _sqrt_err(v1, e_v))
    den_lo = den - e_den
    q = m1 / den
    e_q = (e_m + q.abs() * e_den) / den_lo + DIV_REL * (m1.abs() + e_m) / den_lo + FTZ_ABS
    u = q + wd * p
    e_u = e_q + U * (wd * p).abs() + U * (u.abs() + e_q)
    lr_eff = lr * sched
    d = lr_eff * u
    b_d = (lr_eff * e_u + lr * e_sched * (u.abs() + e_u) + 3 * U * (d.abs() + lr_eff * e_u)
           + U * (p.abs() + d.abs()) + FTZ_ABS)
    return {"m": m1, "b_m": e_m, "v": v1, "b_v": e_v, "d": d, "b_d": b_d}


def skipped(g):
    """the skip rule: a tensor without a nonzero gradient element (the reference's `p.grad is None`, which the flat
    gradient buffer holds as zeros) keeps p, m and v; any nonzero element, however small, takes the whole update"""
    return g is None or not bool((g != 0).any())


def step64(ps, ms, vs, grads, groups, step, cfg, eps_inside=False):
    """one fused step over a list of tensors.  ps, ms, vs: 1-D state tensors; grads: 1-D gradients (None or all zero:
    skipped); groups: (lr, weight_decay) per tensor as fp32 values; step: the device step counter before the step.
    Returns dict S, b_S, T, b_T, sched, and "t": per tensor None (skipped: p, m, v keep their bits) or update64's
    dict."""
    counts = [p.numel() for p in ps]
    S, b_S, T, b_T = sums64(grads, cfg["grad_scale"], counts)
    gmul, d_gmul, _, _ = clip64(S, b_S, T, b_T, cfg)
    sched, e_sched = warmup_linear64(step, cfg["t_total"], cfg["warmup"])
    out = []
    for i, (p, m, v, g) in enumerate(zip(ps, ms, vs, grads)):
        if skipped(g):
            out.append(None)
            continue
        lr, wd = groups[i]
        out.append(update64(p, m, v, g, float(gmul[i]), float(d_gmul[i]), lr, wd, sched, e_sched, cfg,
                            eps_inside=eps_inside))
    return {"S": S, "b_S": b_S, "T": T, "b_T": b_T, "sched": sched, "t": out}


def check_tensor(p_old, p, m_old, m, v_old, v, ref, what):
    """the kernel's state after the step against one entry of step64()["t"] -> worst (m, v, d) ratios"""
    if ref is None:
        assert torch.equal(p, p_old) and torch.equal(m, m_old) and torch.equal(v, v_old), what + ": skipped tensor moved"
        return 0.0, 0.0, 0.0
    d = p_old.double() - p.double()                    # exact: two fp32 values within a factor 2^29 of each other
    return (within(m, ref["m"], ref["b_m"], what + " m"), within(v, ref["v"], ref["b_v"], what + " v"),
            within(d, ref["d"], ref["b_d"], what + " update"))


def check_step(before, after, grads, groups, step, cfg, scratch, what):
    """one kernel step over a list of tensors, checked per element from the kernel's own state before it (so errors do
    not compound over steps) and one tensor at a time (the fp64 temporaries of a whole model need not coexist).
    before / after: (p, m, v) 1-D tensors per tensor; grads: the gradient values the kernel read; scratch: its sums.
    Returns the worst error-to-bound ratio per output."""
    S, b_S, T, b_T = sums64(grads, cfg["grad_scale"], [b[0].numel() for b in before])
    worst = dict(zip(("sumsq", "total"), check_sums(scratch, {"S": S, "b_S": b_S, "T": T, "b_T": b_T}, what)))
    gmul, d_gmul, _, _ = clip64(S, b_S, T, b_T, cfg)
    sched, e_sched = warmup_linear64(step, cfg["t_total"], cfg["warmup"])
    for i, ((p0, m0, v0), (p1, m1, v1), g) in enumerate(zip(before, after, grads)):
        ref = None if skipped(g) else update64(p0, m0, v0, g, float(gmul[i]), float(d_gmul[i]), groups[i][0],
                                                 groups[i][1], sched, e_sched, cfg)
        r = check_tensor(p0, p1, m0, m1, v0, v1, ref, "%s t%d" % (what, i))
        for k, x in zip(("m", "v", "update"), r):
            worst[k] = max(worst.get(k, 0.0), x)
    return worst


def check_sums(scratch, ref, what):
    """scratch [n + 1] (per-tensor sums of squares, then the total) against step64()'s -> worst (S, T) ratios"""
    n = ref["S"].numel()
    return (within(scratch[:n], ref["S"], ref["b_S"], what + " sumsq"),
            within(scratch[n:], ref["T"].reshape(1), ref["b_T"].reshape(1), what + " total"))


def check_shadow(shadow, p, what):
    """the bf16 weight copy is p rounded to nearest even, bit for bit"""
    want = p.to(torch.bfloat16)
    same = shadow.view(torch.int16) == want.view(torch.int16)
    if not bool(same.all()):
        i = int((~same).nonzero()[0])
        raise AssertionError("%s: shadow differs from p in %d of %d elements; first %d: %r vs %r"
                             % (what, int((~same).sum()), same.numel(), i, float(shadow[i]), float(want[i])))
