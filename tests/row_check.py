"""fp64 references and per-element bounds of the row-wise kernels: LayerNorm (csrc/layernorm.cu) and the embedding
LayerNorm (csrc/embed.cu ln_row_fwd), the elementwise GELU / tanh kernels and the casts (csrc/misc.cu), mean pooling,
the similarity losses and the softmax cross-entropy (csrc/loss.cu).  Shared by tests/test_gpu_rowwise_fp64.py and
validated on CPU by tests/test_cpu_row_check.py.

Every bound is derived from the kernel's fp32 arithmetic in the style of tests/gemm_check.py: U = 2^-24 per rounding,
n U sum|terms| for a sum taken in a fixed order of n steps, and BF16_ROUND |ref| (plus the fp32 error carried through
it) for a bf16 store.  The functions take and return torch tensors on any device; all work is in fp64."""
import math

import numpy as np
import torch

from tests.attn_check import EXP_ARG, EXP_REL, LOG_ABS
from tests.gemm_check import BF16_ROUND, U, within  # noqa: F401  (within: re-exported for the tests)

EPS32 = float(np.float32(1e-12))   # the LayerNorm eps as the kernels receive it (a float)
BF16_MAX = float(torch.finfo(torch.bfloat16).max)
# 1.0f / sqrtf(v) under --use_fast_math: rsqrt.approx, or sqrt.approx then an approximate reciprocal.  Each is within
# 2 ulp (2^-22 relative); 8U leaves a factor 2 for the composition.
RSQRT_REL = 8 * U
# a / b under --use_fast_math is div.approx (2 ulp): 4U relative
DIV_REL = 4 * U
# MUFU.TANH (tanhf under --use_fast_math): relative error below 2^-10.9, plus an absolute floor near 0
# (the bound of test_gpu_kernels.py::test_pooler_sim_bwd_param_grads_fp64_and_repeatable)
TANH_REL = 2.0 ** -10
TANH_ABS = 2.0 ** -20
# GELU: common.cuh gelu_erf evaluates w = 1 - Phi(|x|) with Abramowitz & Stegun 7.1.26.  Over every finite bf16 input
# its absolute error in w is at most 7.0e-8 (tests/test_cpu_row_check.py evaluates it), so gelu = max(x, 0) - |x| w
# errs by up to 7.0e-8 |x| absolute.  For x <= -5.25, where gelu(x) is about 1e-6, that is up to 16% of the value: the
# formula's tail, not a bug.  (The reference's own fp32 x * 0.5 * (1 + erf(x / sqrt 2)) is worse there: 1 + erf
# cancels to 0.)  GELU_ABS = 2^-23 > 7.0e-8 is the absolute term per unit |x|; the fp32 operations on top of it
# (rcp.approx on t, ex2.approx on exp(-x^2/2) and the rounding of its argument, the Horner fmas) are GELU_REL
# relative to w plus EXP_ARG U |arg| from the argument.
GELU_ABS = 2.0 ** -23
GELU_REL = EXP_REL + 16 * U
# --use_fast_math flushes fp32 denormals to zero: an elementwise result below 2^-126 may come out as 0
FTZ_ABS = 2.0 ** -126


def bf16_store(err, ref):
    """bound of a bf16 store of an fp32 value within `err` of `ref`: the fp32 error (grown by the rounding) plus half a
    bf16 ulp of the value (BF16_ROUND |ref|, a ratio near 1 at the bottom of a binade is expected)"""
    return err * (1 + BF16_ROUND) + BF16_ROUND * ref.abs()


# ---------------------------------------------------------------------------------------------------------
# LayerNorm forward (layernorm.cu layernorm_fwd_kernel, embed.cu ln_row_fwd / embed_src_fwd_kernel)
# ---------------------------------------------------------------------------------------------------------
def ln_fwd(z, gamma, beta, ez=None, drop=None, unbiased=False):
    """fp64 LayerNorm of the pre-LN rows z [R, C] (the exact values the kernel should see) and the bound of every
    output.  ez: per-element bound of the kernel's fp32 z against z (0 where z is exact: fp32 or bf16 input).  drop:
    (keep bool [R, C], scale) applied to the output (drop mode 2).  unbiased: divide the variance by C - 1 (a
    perturbation for the negative checks, not the kernel's statement).
    Returns dict mean, b_mean, rstd, b_rstd [R]; y, b_y [R, C].

    The kernel, per row: each lane adds its C / 32 elements in order, a 5-level warp tree adds the lanes, and one
    multiply by 1/C (itself rounded) gives the mean: e_mean = (C/32 + 7) U mean|z| + mean(ez).  The variance is the
    same sum of d^2, d = z - mean, over the kernel's mean.  With sum d = 0 exactly in fp64, a shift of the mean moves
    the sum of squares only at second order, so the error of the centred sum is 2 sum|d| ed + sum (ed + e_mean)^2
    (ed: the rounding of d and ez) plus (C/32 + 7) U on the sum of the squares, then U for eps.  rstd is bounded by
    evaluating 1/sqrt at the low end of that interval, plus RSQRT_REL.  y = gamma ((z - mean) rstd) + beta: the stats'
    errors through xhat, two roundings per product and sum, and the bf16 store."""
    z = z.double()
    R, C = z.shape
    ez = torch.zeros_like(z) if ez is None else ez.double()
    nsum = C / 32 + 7
    mean = z.mean(1, keepdim=True)
    d = z - mean
    n_var = C - 1 if unbiased else C
    var = (d * d).sum(1, keepdim=True) / n_var
    rstd = 1.0 / torch.sqrt(var + EPS32)
    e_mean = nsum * U * z.abs().mean(1, keepdim=True) + ez.mean(1, keepdim=True)
    ed = ez + U * (d.abs() + ez + e_mean)
    sq = ((d.abs() + ed + e_mean) ** 2).sum(1, keepdim=True)
    e_q = 2 * (d.abs() * ed).sum(1, keepdim=True) + ((ed + e_mean) ** 2).sum(1, keepdim=True) + (nsum + 1) * U * sq
    e_var = e_q / C + 2 * U * var + U * (var + EPS32)
    lo = (var + EPS32 - e_var).clamp_min(EPS32 * 0.5)
    b_rstd = (1.0 / torch.sqrt(lo) - rstd) + RSQRT_REL / torch.sqrt(lo)
    xhat = d * rstd
    e_d = ed + e_mean
    e_xhat = ((d.abs() + e_d) * b_rstd + rstd * e_d) * (1 + 4 * U) + 2 * U * xhat.abs()
    g, b = gamma.double(), beta.double()
    o = g * xhat + b
    e_o = g.abs() * e_xhat + 2 * U * ((g * xhat).abs() + b.abs())
    if drop is not None:
        keep, scale = drop
        k = keep.to(z.device).double() * scale
        o = o * k
        e_o = e_o * k + U * o.abs()
    return {"mean": mean[:, 0], "b_mean": e_mean[:, 0], "rstd": rstd[:, 0], "b_rstd": b_rstd[:, 0], "y": o,
            "b_y": bf16_store(e_o, o)}


def ln_bwd64(z, d, gamma):
    """fp64 LayerNorm backward of rows z [R, C] for upstream d: (xhat, dz, e_xhat, e_dz) where e_* bound the fp32
    kernels' per-element error (C-term row sums for the mean, variance and the two backward row sums)"""
    C = z.shape[1]
    mean = z.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(1, keepdim=True) + 1e-12)
    xhat = (z - mean) * rstd
    g = d * gamma.double()
    gx = (g * xhat).mean(1, keepdim=True)
    dz = rstd * (g - g.mean(1, keepdim=True) - xhat * gx)
    k = (C + 16) * U
    e_xhat = k * (rstd * (z.abs().mean(1, keepdim=True) + z.abs()) + xhat.abs())
    e_dz = 2 * k * (rstd * (g.abs() + g.abs().mean(1, keepdim=True) + (1 + xhat.abs()) * (g * xhat).abs().mean(1, keepdim=True))
                    + dz.abs()) + rstd * (g * xhat).abs().mean(1, keepdim=True) * e_xhat
    return xhat, dz, e_xhat, e_dz


def check_ln(y, mean, rstd, ref, what):
    """kernel outputs against an ln_fwd() dict -> worst (mean, rstd, y) ratios"""
    return (within(mean, ref["mean"], ref["b_mean"], what + " mean"),
            within(rstd, ref["rstd"], ref["b_rstd"], what + " rstd"),
            within(y, ref["y"], ref["b_y"], what + " y"))


# ---------------------------------------------------------------------------------------------------------
# elementwise (misc.cu eltwise_bf16_kernel)
# ---------------------------------------------------------------------------------------------------------
def _w64(x):
    """1 - Phi(|x|) in fp64"""
    from scipy.special import erfc
    return torch.from_numpy(0.5 * erfc(np.abs(x.cpu().numpy()) / math.sqrt(2.0))).to(x.device)


def gelu64(x):
    """x Phi(x) = max(x, 0) - |x| (1 - Phi(|x|)), evaluated without cancellation in the tail"""
    x = x.double()
    return torch.clamp(x, min=0.0) - x.abs() * _w64(x)


def gelu_grad64(x):
    x = x.double()
    w = _w64(x)
    cdf = torch.where(x >= 0, 1.0 - w, w)
    return cdf + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def gelu_bound(x):
    """|gelu_erf(x) - gelu(x)| in fp32, before the store"""
    x = x.double()
    arg = 0.5 * x * x / math.log(2.0)
    return x.abs() * (GELU_ABS + _w64(x) * (GELU_REL + EXP_ARG * U * arg)) + U * gelu64(x).abs()


def gelu_grad_bound(x):
    """|gelu_erf_grad(x) - gelu'(x)| in fp32: the w term (absolute, as for gelu) and the Gaussian term's exponential"""
    x = x.double()
    arg = 0.5 * x * x / math.log(2.0)
    phi_x = (x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)).abs()
    return GELU_ABS + _w64(x) * (GELU_REL + EXP_ARG * U * arg) + phi_x * (EXP_REL + EXP_ARG * U * arg + 4 * U) \
        + U * gelu_grad64(x).abs()


def eltwise_ref(kind, x, dy=None):
    """(fp64 value, bound of the kernel's bf16 output) of one elementwise kernel on bf16 x (and dy)"""
    xd = x.double()
    if kind == "gelu":
        ref, e = gelu64(xd), gelu_bound(xd)
    elif kind == "gelu_bwd":
        gd = gelu_grad64(xd)
        ref = dy.double() * gd
        e = dy.double().abs() * gelu_grad_bound(xd) + U * ref.abs()
    elif kind == "tanh":
        ref = torch.tanh(xd)
        e = TANH_REL * ref.abs() + TANH_ABS
    else:  # tanh_bwd: dy (1 - y^2) with y = x; y^2 and 1 - y^2 are exact in fp32 for bf16 y, one rounding each besides
        ref = dy.double() * (1.0 - xd * xd)
        e = 3 * U * (dy.double().abs() * (1.0 + xd * xd))
    return ref, bf16_store(e + FTZ_ABS, ref)


# ---------------------------------------------------------------------------------------------------------
# mean pooling (loss.cu meanpool_fwd_kernel / meanpool_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------
def meanpool_on(mask, skip_first):
    on = mask != 0
    if skip_first:
        on = on.clone()
        on[:, 0] = False
    return on


def meanpool_ref(x, mask, N, S, skip_first, guard_zero, l2norm, dy=None, count_first=False):
    """fp64 autograd of the masked mean over S tokens (position 0 excluded under skip_first, an all-padded row's
    denominator 1 under guard_zero) and F.normalize, and the bounds of the forward (out) and backward (dx).
    count_first: a denominator that still counts position 0 under skip_first (a perturbation for the negative checks).

    Forward: u = (sum over S tokens, in order) / den: S U sum|x| / den + DIV_REL |u|.  With l2norm: the block's sum of
    u^2 (<= 4 per thread, then 5 warp levels and 8 warps in order), sqrtf (sqrt.approx, 4U) and u / n (DIV_REL).
    Backward: du = (dy - y dot) / n with the kernel's own y and n, dot = sum y dy: the forward bounds of y and n
    carried through, the sum and the two divisions, then the bf16 store."""
    x3 = x.double().view(N, S, -1).clone().requires_grad_(dy is not None)
    H = x3.shape[2]
    on = meanpool_on(mask, skip_first).double()
    den = (meanpool_on(mask, False) if count_first else on).double().sum(1, keepdim=True)
    if guard_zero:
        den = torch.where(den == 0, torch.ones_like(den), den)
    u = (x3 * on[:, :, None]).sum(1) / den
    out = torch.nn.functional.normalize(u, dim=-1) if l2norm else u
    with torch.no_grad():
        ud = u.detach()
        e_u = S * U * (x3.detach().abs() * on[:, :, None]).sum(1) / den + DIV_REL * ud.abs()
        if l2norm:
            n = ud.norm(dim=1, keepdim=True).clamp_min(1e-12)
            e_sq = 2 * (ud.abs() * e_u).sum(1, keepdim=True) + (H / 256 + 16) * U * (ud * ud).sum(1, keepdim=True)
            e_n = e_sq / (2 * n) * (1 + 1e-3) + 4 * U * n
            o = out.detach()
            e_out = (e_u + o.abs() * e_n) / n + DIV_REL * o.abs()
        else:
            e_out = e_u
    res = {"out": out.detach(), "b_out": e_out}
    if dy is None:
        return res
    out.backward(dy.double())
    with torch.no_grad():
        dyd = dy.double()
        dx = x3.grad.reshape(N * S, H)
        if l2norm:
            y = out.detach()
            dot = (y * dyd).sum(1, keepdim=True)
            e_dot = (dyd.abs() * e_out).sum(1, keepdim=True) + (H / 256 + 16) * U * (y * dyd).abs().sum(1, keepdim=True)
            num = dyd - y * dot
            e_num = dot.abs() * e_out + y.abs() * e_dot + 2 * U * (dyd.abs() + (y * dot).abs())
            du = num / n
            e_du = (e_num + du.abs() * e_n) / n * (1 + 1e-3) + DIV_REL * du.abs()
        else:
            du, e_du = dyd, torch.zeros_like(dyd)
        e_g = (e_du / den + DIV_REL * (du / den).abs())[:, None, :] * on[:, :, None]
        res["dx"] = dx
        res["b_dx"] = bf16_store(e_g.reshape(N * S, H), dx)
    return res


# ---------------------------------------------------------------------------------------------------------
# similarity matrix and losses (loss.cu sim_fwd / sim_bwd, maxmargin / crossen / milnce kernels)
# ---------------------------------------------------------------------------------------------------------
def pooler_sim_ref(u, w, b):
    """(ref, bound) of univl_pooler_sim_fwd (PoolerSimFn): logit = tanh(u) . w + b per row, u bf16 [N, H], w [H] (or
    [1, H]), b [1]; MUFU.TANH per element, then an fp32 dot product in H / 32 lane steps and a warp tree"""
    H = u.shape[1]
    th = torch.tanh(u.double())
    wd = w.double().reshape(-1).to(th.device)
    bd = float(b.double().reshape(-1)[0])
    ref = th @ wd + bd
    terms = (th.abs() * wd.abs()).sum(1)
    bound = ((TANH_REL * th.abs() + TANH_ABS) * wd.abs()).sum(1) + (H / 32 + 8) * U * (terms + abs(bd))
    return ref, bound


def sim_ref(t, v):
    """sim = t v^T: each lane adds H / 32 products in order, then 5 warp levels"""
    H = t.shape[1]
    td, vd = t.double(), v.double()
    return td @ vd.t(), (H / 32 + 7) * U * (td.abs() @ vd.abs().t())


def sim_bwd_ref(dsim, b_dsim, t, v):
    """dt = dsim v, dv = dsim^T t from the kernel's fp32 dsim (reference: the fp64 dsim, whose bound b_dsim is carried
    through), each a sum over B terms in order"""
    Bt, Bv = dsim.shape
    ds = dsim.double()
    td, vd = t.double(), v.double()
    return (ds @ vd, (Bv + 2) * U * (ds.abs() @ vd.abs()) + b_dsim @ vd.abs(),
            ds.t() @ td, (Bt + 2) * U * (ds.abs().t() @ td.abs()) + b_dsim.t() @ td.abs())


def _lse_terms(x, n_lane):
    """logsumexp of the rows of x (fp64, -inf allowed) and its bound when a kernel takes the max, adds expf(x - m)
    over n_lane terms per lane plus 5 warp levels (more for a CTA: the caller's n_lane covers it) and adds logf:
    each exponential errs by EXP_REL + EXP_ARG U |x - m| relative (weighted by its share p of the sum), the sum by
    (n_lane + 6) U, the log by LOG_ABS, and the final add by U |lse|"""
    m = x.amax(1, keepdim=True)
    lse = torch.logsumexp(x, 1, keepdim=True)
    p = torch.exp(x - lse)
    arg = torch.where(p > 0, (x - m).abs(), torch.zeros_like(x))
    rel = (p * (EXP_REL + (EXP_ARG + 1) * U * arg)).sum(1, keepdim=True) + (n_lane + 6) * U
    return lse, rel * (1 + 2 * rel) + LOG_ABS + U * lse.abs()


def crossen_ref(sim):
    """-mean_i log_softmax(sim)[i, i] and d/dsim; one warp per row, lanes over columns"""
    s = sim.double().clone().requires_grad_()
    B = s.shape[0]
    loss = -torch.diagonal(torch.log_softmax(s, 1)).mean()
    loss.backward()
    with torch.no_grad():
        sd = s.detach()
        lse, e_lse = _lse_terms(sd, B / 32)
        nll = lse[:, 0] - torch.diagonal(sd)
        b_loss = (e_lse.sum() + (B / 8 + 16) * U * nll.abs().sum()) / B + DIV_REL * loss.abs()
        p = torch.exp(sd - lse)
        e_p = p * (EXP_REL + (EXP_ARG + 1) * U * (sd - lse).abs() + e_lse)
        b_dsim = (e_p + U * (p - torch.eye(B, dtype=p.dtype, device=p.device)).abs()) / B + DIV_REL * s.grad.abs()
    return loss.detach(), b_loss, s.grad, b_dsim


def maxmargin_weights(bs, n_pair, hard_negative_rate):
    """(w_same, w_diff) of the reference's hard-negative weighting (oracle max_margin_loss), as the floats the kernel
    receives"""
    easy = 1 - hard_negative_rate
    alpha = easy / ((bs - 1) * (1 - easy))
    scale = bs * (1 - easy)
    return float(np.float32(scale)), float(np.float32(alpha * scale))


def maxmargin_ref(sim, margin, n_pair, w_same, w_diff, drop_diag=None):
    """mean_ij w_ij (relu(m + s_ij - s_ii) + relu(m + s_ij - s_jj)) and d/dsim.  The hinge decisions are fp64's; the
    tests keep every |m + s_ij - s_kk| far above its fp32 rounding (U |m + s_ij| + U |a|).  drop_diag: leave one hinge
    term out of dsim[k, k] (a perturbation for the negative checks)."""
    s = sim.double()
    B = s.shape[0]
    idx = torch.arange(B, device=s.device)
    same = (idx[:, None] // n_pair) == (idx[None, :] // n_pair) if n_pair > 0 else torch.ones(B, B, dtype=torch.bool,
                                                                                              device=s.device)
    w = torch.where(same, w_same, w_diff) if n_pair > 0 else torch.ones(B, B, dtype=s.dtype, device=s.device)
    m = float(np.float32(margin))
    diag = torch.diagonal(s)
    a = m + s - diag[:, None]
    c = m + s - diag[None, :]
    ha, hc = (a > 0).double(), (c > 0).double()
    inv = 1.0 / (B * B)
    loss = (w * (a * ha + c * hc)).sum() * inv
    g = w * (ha + hc) * inv
    gd = -(w * ha).sum(1) * inv - (w * hc).sum(0) * inv
    if drop_diag is not None:
        k = drop_diag
        j = int(torch.nonzero(ha[k])[0])
        gd[k] += w[k, j] * inv
    dsim = g + torch.diag(gd)
    e_a = U * (m + s).abs() + 2 * U * a.abs()
    e_c = U * (m + s).abs() + 2 * U * c.abs()
    terms = (w * (a.abs() * ha + c.abs() * hc))
    b_loss = inv * ((w * (e_a * ha + e_c * hc)).sum() + (B * B / 256 + 20) * U * terms.sum()) + 2 * U * loss.abs()
    b_dsim = 2 * U * g + torch.diag((2 * B + 4) * U * (g.sum(1) + g.sum(0)))
    return loss, b_loss, dsim, b_dsim, (a, c, e_a, e_c)


def milnce_ref(sim, bs, P, pick_offset=None):
    """the oracle's MIL-NCE (until_module.py:193-221) and d/dsim in fp64, and the bounds: per picked row, the
    logsumexp of 2N values and of its positives (one warp, 2N / 32 per lane), the loss over bs rows, the gradient's
    two exponentials, and one more rounding for the second of a cell's two atomic addends.  pick_offset: the picked
    row within a block (the reference's P // 2; other values are perturbations for the negative checks)."""
    s = sim.double().clone().requires_grad_()
    N = bs * P
    dev = s.device
    mask = torch.kron(torch.eye(bs, dtype=torch.float64, device=dev), torch.ones(P, P, dtype=torch.float64, device=dev))
    new = torch.cat([s.t(), s + mask * -1e12], 1)
    logpt = torch.log_softmax(new, 1)
    mask2 = torch.cat([mask, torch.zeros_like(mask)], 1)
    new_logpt = -torch.logsumexp(logpt + (1.0 - mask2) * -1e12, 1)
    pick = torch.arange(bs, device=dev) * P + (P // 2 if pick_offset is None else pick_offset)
    loss = new_logpt[pick].mean()
    loss.backward()
    with torch.no_grad():
        x = new.detach()[pick]
        lse, e_lse = _lse_terms(x, 2 * N / 32)
        xp = torch.where(mask2[pick] > 0, x, torch.full_like(x, -math.inf))
        lsep, e_lsep = _lse_terms(xp, 2 * N / 32)
        nl = (lse - lsep)[:, 0]
        b_loss = ((e_lse + e_lsep).sum() + (bs / 8 + 16) * U * nl.abs().sum()) / bs + DIV_REL * loss.abs()
        p = torch.exp(x - lse)
        pp = torch.where(mask2[pick] > 0, torch.exp(xp - lsep), torch.zeros_like(x))
        ex = lambda q, l, e: q * (EXP_REL + (EXP_ARG + 1) * U * torch.where(q > 0, (x - l).abs(), 0 * x) + e)
        e_gr = (ex(p, lse, e_lse) + ex(pp, lsep, e_lsep) + U * (p - pp).abs()) / bs + DIV_REL * (p - pp).abs() / bs
        b = torch.zeros(N, N, dtype=torch.float64, device=dev)
        b[:, pick] += e_gr[:, :N].t()
        b[pick, :] += e_gr[:, N:]
        b_dsim = b + 2 * U * s.grad.abs()
    return loss.detach(), b_loss, s.grad, b_dsim


# ---------------------------------------------------------------------------------------------------------
# softmax cross-entropy (loss.cu xent_fwd_kernel / xent_sum_kernel / xent_bwd_kernel)
# ---------------------------------------------------------------------------------------------------------
def xent_ref(logits, labels, V, target_mode, groups, pair_mask=None, gscale=1.0, drop_row=None):
    """fp64 lse per row, the loss (mean over groups of each group's mean over its scored rows) and dlogits [T, V], with
    bounds.  logits: fp32 [T, >= V] (columns >= V unread).  pair_mask: MFM's vm [T]: logit += (1 - vm_r vm_c) * -1e8
    over the row's group's columns.  drop_row: leave this scored row out of the loss (a perturbation for the negative
    checks).  lse: one CTA of 256 threads per row, V / 256 terms per thread then the block's 13 levels.  Loss: the
    group's rows in order per thread (R / 256 each), 13 more levels, the division by the count and the mean over
    groups.  dlogits: (expf(x - lse) - onehot) (gscale / G) / count: the exponential, lse's bound, two divisions and
    the bf16 store."""
    T = logits.shape[0]
    R = T // groups
    dev = logits.device
    x = logits[:, :V].double()
    rows = torch.arange(T, device=dev)
    grp = rows // R
    if pair_mask is not None:
        vm = (pair_mask != 0).double()
        cols = (grp * R if target_mode == 1 else torch.zeros_like(grp))[:, None] + torch.arange(V, device=dev)[None, :]
        x = x + (1.0 - vm[:, None] * vm[cols]) * -1e8
    tgt = labels.clone() if target_mode == 0 else rows - grp * R
    scored = labels != -1
    lse, e_lse = _lse_terms(x, V / 256 + 8)
    lse, e_lse = lse[:, 0], e_lse[:, 0]
    xt = x.gather(1, tgt.clamp(0, V - 1)[:, None])[:, 0]
    term = torch.where(scored, lse - xt, torch.zeros_like(lse))
    use = scored.clone()
    if drop_row is not None:
        use[drop_row] = False
    cnt = torch.zeros(groups, dtype=torch.float64, device=dev).index_add_(0, grp, scored.double())
    s = torch.zeros(groups, dtype=torch.float64, device=dev).index_add_(0, grp, torch.where(use, term, 0 * term))
    e_term = torch.where(scored, e_lse + U * term.abs(), 0 * term)
    es = torch.zeros_like(s).index_add_(0, grp, e_term)
    mag = torch.zeros_like(s).index_add_(0, grp, term.abs())
    Lg = s / cnt
    loss = Lg.mean()
    b_loss = ((es + (R / 256 + 16) * U * mag) / cnt + DIV_REL * Lg.abs()).mean() + (groups + 2) * U * abs(float(loss))
    p = torch.exp(x - lse[:, None])
    onehot = torch.zeros_like(p)
    onehot[rows, tgt.clamp(0, V - 1)] = 1.0
    gr = (gscale / groups) / cnt[grp]
    d = torch.where(scored[:, None], (p - onehot) * gr[:, None], 0 * p)
    e_p = p * (EXP_REL + (EXP_ARG + 1) * U * torch.where(p > 0, (x - lse[:, None]).abs(), 0 * p) + e_lse[:, None])
    e_d = torch.where(scored[:, None], (e_p + U * (p - onehot).abs()) * gr[:, None] + 3 * DIV_REL * d.abs(), 0 * p)
    return {"lse": torch.where(scored, lse, 0 * lse), "b_lse": torch.where(scored, e_lse, 0 * lse), "loss": loss,
            "b_loss": b_loss, "count": cnt, "sum": s, "dl": d, "b_dl": bf16_store(e_d, d)}
