"""GPU: the row-wise kernels against fp64 under per-element bounds (tests/row_check.py): LayerNorm at every width and the
NormalizeVideo LayerNorm, the embedding forwards, the elementwise GELU / tanh kernels over every bf16 bit pattern, the
casts, mean pooling, the pooler similarity, the similarity matrix and its three losses at production batch sizes, and
the softmax cross-entropy called directly.  Each check prints its worst err / bound as "ratio"; the negative checks
perturb the reference and show the bound rejects it."""
import numpy as np
import pytest
import torch

from tests import attn_check as ac
from tests import row_check as rc
from tests.gemm_check import U, within
from tests.test_gpu_kernels import _same_bits
from univl_b200 import ops
from univl_b200.runtime import call, ptr

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
SEED, EPOCH = 123, 2


def _rng():
    return torch.tensor([SEED, EPOCH], dtype=torch.int64, device=DEV)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rejects(got, ref, bound, what):
    with pytest.raises(AssertionError):
        within(got, ref, bound, what + " (perturbed reference)")


# ---------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------
def _special_rows(x, cols, g):
    """rows 0-2 constant (rstd = 1/sqrt(eps), y = beta), rows 3-5 offset 64 with std 1e-2 (where E[z^2] - E[z]^2 would
    cancel), row 6 spanning a wide dynamic range (+-2^50 next to +-2^-60).  The fp32 statistics hold up to |z| of about
    2^59 at C = 768; beyond it the sum of squares overflows (rstd 0, y = beta), as in any fp32 LayerNorm, so the bf16
    extremes near 3.4e38 are outside what this kernel (or the reference's fp32 LayerNorm) computes."""
    n = x.shape[0]
    for r, c in zip(range(min(3, n)), (1.0, -2.5, 0.375)):
        x[r] = c
    for r in range(3, min(6, n)):
        x[r] = (64.0 + 1e-2 * torch.randn(cols, device=DEV, generator=g)).to(BF16)
    if n > 6:
        sgn = torch.where(torch.rand(cols, device=DEV, generator=g) < 0.5, -1.0, 1.0)
        mag = torch.where(torch.rand(cols, device=DEV, generator=g) < 0.5, 2.0 ** 50, 2.0 ** -60)
        x[6] = (sgn * mag).to(BF16)
    return x


LN_CASES = [(rows, cols, True, 0) for cols in (256, 512, 768, 1024) for rows in (1, 7, 37)] + \
    [(37, 768, False, 0), (37, 768, True, 1), (37, 768, True, 2), (37, 1024, False, 2), (98304, 768, True, 0),
     (98304, 768, False, 0)]


@pytest.mark.parametrize("rows,cols,with_res,mode", LN_CASES)
def test_layernorm_fwd(rows, cols, with_res, mode):
    g = _gen(rows * 7 + cols + mode)
    x = (1.5 * torch.randn(rows, cols, device=DEV, generator=g) + 0.3).to(BF16)
    res = (torch.randn(rows, cols, device=DEV, generator=g)).to(BF16) if with_res else None
    if not with_res:
        x = _special_rows(x, cols, g)
    gamma = 1 + 0.1 * torch.randn(cols, device=DEV, generator=g)
    beta = 0.1 * torch.randn(cols, device=DEV, generator=g)
    p = 0.1 if mode else 0.0
    rng = _rng()
    y, mean, rstd = ops.layernorm_fwd(x, res, gamma, beta, p=p, mode=mode, seed=rng.data_ptr(), stream=9)
    torch.cuda.synchronize()
    scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if mode else 1.0
    keep = ac.keep_elem(SEED, ac.kernel_stream(9, EPOCH), p, rows, cols).to(DEV) if mode else None
    z = x.double() * (keep.double() * scale if mode == 1 else 1.0)
    if with_res:
        z = z + res.double()
    ez = U * (x.double().abs() * (scale if mode == 1 else 1.0) + z.abs()) * 1.01 if (with_res or mode == 1) else None
    ref = rc.ln_fwd(z, gamma, beta, ez=ez, drop=(keep, scale) if mode == 2 else None)
    rc.check_ln(y, mean, rstd, ref, "layernorm %dx%d res=%d mode=%d" % (rows, cols, with_res, mode))
    if not with_res and rows >= 3:
        for r, c in zip(range(3), (1.0, -2.5, 0.375)):
            assert float(mean[r]) == c
            assert abs(float(rstd[r]) - 1.0 / np.sqrt(rc.EPS32)) <= rc.RSQRT_REL / np.sqrt(rc.EPS32)
            assert torch.equal(y[r], beta.to(BF16)) or mode == 2
    if rows == 37 and cols == 768 and mode == 0:
        _rejects(rstd, rc.ln_fwd(z, gamma, beta, ez=ez, unbiased=True)["rstd"], ref["b_rstd"], "unbiased variance")


@pytest.mark.parametrize("rows", [32 * 48, 98304])
def test_normalize_video_fwd_bwd(rows):
    """NormalizeVideo: fp32 rows that are not bf16-exact, every 5th frame all zero; stats and y against fp64, dgamma /
    dbeta against fp64 with the same bits on repeat and with 40 SMs reserved"""
    cols = 1024
    g = _gen(rows)
    x = 0.7 * torch.randn(rows, cols, device=DEV, generator=g) + 0.2
    x[::5] = 0.0
    gamma = 1 + 0.1 * torch.randn(cols, device=DEV, generator=g)
    beta = 0.1 * torch.randn(cols, device=DEV, generator=g)
    y = torch.empty(rows, cols, dtype=BF16, device=DEV)
    mean = torch.empty(rows, device=DEV)
    rstd = torch.empty(rows, device=DEV)
    call("univl_layernorm_f32_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(),
         rstd.data_ptr(), rows, cols, ops.LN_EPS)
    torch.cuda.synchronize()
    rc.check_ln(y, mean, rstd, rc.ln_fwd(x.double(), gamma, beta), "normalize_video %d" % rows)
    assert bool((y[::5] == beta.to(BF16)).all())
    dy = torch.randn(rows, cols, device=DEV, generator=g).to(BF16)

    def run():
        dgamma, dbeta = torch.zeros(cols, device=DEV), torch.zeros(cols, device=DEV)
        call("univl_layernorm_f32_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(),
             rstd.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), rows, cols)
        return [dgamma, dbeta]
    dgamma, dbeta = _same_bits(run)
    d = dy.double()
    xhat, _, e_xhat, _ = rc.ln_bwd64(x.double(), d, gamma)
    n = rows + 2
    within(dbeta, d.sum(0), n * U * d.abs().sum(0) + 1e-30, "normalize_video dbeta")
    within(dgamma, (d * xhat).sum(0), n * U * (d * xhat).abs().sum(0) + (d.abs() * e_xhat).sum(0),
           "normalize_video dgamma")


# ---------------------------------------------------------------------------------------------------------
# embeddings
# ---------------------------------------------------------------------------------------------------------
def _tables(g, H=768):
    return (0.05 * torch.randn(512, H, device=DEV, generator=g), 0.05 * torch.randn(2, H, device=DEV, generator=g),
            1 + 0.1 * torch.randn(H, device=DEV, generator=g), 0.1 * torch.randn(H, device=DEV, generator=g))


@pytest.mark.parametrize("with_type", [True, False])
def test_embed_text_fwd(with_type):
    n, S, H, V = 32, 48, 768, 30522
    g = _gen(31 + with_type)
    word = 0.05 * torch.randn(V, H, device=DEV, generator=g)
    pos, typ, gamma, beta = _tables(g)
    ids = torch.randint(1000, 3000, (n, S), device=DEV, generator=g)
    ids[:, 0] = 101                                   # [CLS]
    ids[:, 30] = 102                                  # [SEP]
    ids[:, 31:] = 0                                   # [PAD]
    tids = torch.zeros(n, S, dtype=torch.long, device=DEV)
    tids[:, S // 2:] = 1
    y = torch.empty(n * S, H, dtype=BF16, device=DEV)
    mean, rstd = torch.empty(n * S, device=DEV), torch.empty(n * S, device=DEV)
    call("univl_embed_text_fwd", ids.data_ptr(), tids.data_ptr() if with_type else None, word.data_ptr(),
         pos.data_ptr(), typ.data_ptr() if with_type else None, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
         mean.data_ptr(), rstd.data_ptr(), n, S, H, V, ops.LN_EPS, 0.0, None, 0)
    torch.cuda.synchronize()
    parts = [word.double()[ids.reshape(-1)], pos.double()[torch.arange(S, device=DEV).repeat(n)]]
    if with_type:
        parts.append(typ.double()[tids.reshape(-1)])
    z = sum(parts)
    ez = 2 * U * sum(t.abs() for t in parts)
    rc.check_ln(y, mean, rstd, rc.ln_fwd(z, gamma, beta, ez=ez), "embed_text type=%d" % with_type)


# (Na, Wa, Nb, Fb, all_pairs): visual-only, aligned, all-pairs G = 1, grouped G = 2 and 3
SRC_CASES = [(32, 48, 0, 0, 0), (32, 24, 32, 24, 0), (8, 48, 8, 48, 1), (12, 20, 6, 28, 2), (9, 16, 6, 12, 3)]


@pytest.mark.parametrize("Na,Wa,Nb,Fb,G", SRC_CASES)
def test_embed_src_fwd(Na, Wa, Nb, Fb, G):
    """y, mean and rstd on every output row, every fan-out copy of a source row included"""
    H = 768
    g = _gen(Na * 100 + Nb + G)
    a = torch.randn(Na * Wa, H, device=DEV, generator=g).to(BF16)
    b = torch.randn(Nb * Fb, H, device=DEV, generator=g).to(BF16) if Fb else None
    pos, typ, gamma, beta = _tables(g)
    n_seq = Na * Nb // G if (G and Fb) else Na
    S = Wa + Fb
    y = torch.full((n_seq * S, H), float("nan"), dtype=BF16, device=DEV)
    mean = torch.full((n_seq * S,), float("nan"), device=DEV)
    rstd = torch.full((n_seq * S,), float("nan"), device=DEV)
    call("univl_embed_src_fwd", a.data_ptr(), ptr(b), pos.data_ptr(), typ.data_ptr(), gamma.data_ptr(),
         beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), Na, Wa, Nb, Fb, G, H, ops.LN_EPS, 0.0, None,
         0)
    torch.cuda.synchronize()
    p = torch.arange(n_seq)
    if not Fb:
        src = a.double().view(Na, Wa, H)
    else:
        if G == 0:
            i = j = p
        else:
            Gv, per = Nb // G, n_seq // G
            grp = p // per
            r = p - grp * per
            i, j = grp * (Na // G) + r // Gv, grp * Gv + r % Gv
        src = torch.cat([a.double().view(Na, Wa, H)[i.to(DEV)], b.double().view(Nb, Fb, H)[j.to(DEV)]], 1)
    types = torch.cat([torch.zeros(Wa, dtype=torch.long), torch.ones(Fb, dtype=torch.long)]).to(DEV)
    add = pos.double()[:S] + typ.double()[types]
    z = (src + add).reshape(-1, H)
    ez = (2 * U * (src.abs() + pos.double()[:S].abs() + typ.double()[types].abs())).reshape(-1, H)
    rc.check_ln(y, mean, rstd, rc.ln_fwd(z, gamma, beta, ez=ez), "embed_src %s" % ((Na, Wa, Nb, Fb, G),))


# ---------------------------------------------------------------------------------------------------------
# elementwise kernels, every bf16 bit pattern
# ---------------------------------------------------------------------------------------------------------
ELTWISE = {"gelu": "univl_gelu_fwd_bf16", "tanh": "univl_tanh_fwd_bf16", "gelu_bwd": "univl_gelu_bwd_bf16",
           "tanh_bwd": "univl_tanh_bwd_bf16"}


def _eltwise(kind, x, dy):
    out = torch.empty_like(x)
    if kind in ("gelu", "tanh"):
        call(ELTWISE[kind], x.data_ptr(), out.data_ptr(), x.numel())
    else:
        call(ELTWISE[kind], dy.data_ptr(), x.data_ptr(), out.data_ptr(), x.numel())
    return out


def _all_bf16():
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(BF16).to(DEV)


@pytest.mark.parametrize("kind", list(ELTWISE))
def test_eltwise_every_bf16_input(kind):
    x = _all_bf16()
    dy = torch.randn(65536, device=DEV, generator=_gen(5)).to(BF16)
    got = _eltwise(kind, x, dy)
    torch.cuda.synchronize()
    fin = torch.isfinite(x)
    ref, bound = rc.eltwise_ref(kind, x[fin], dy[fin])
    # the backward kernels' products can leave the bf16 range: from the top bf16 binade on inf is allowed, and past it
    # required.  gelu(x) = x there and tanh is bounded, so the forwards are checked exactly over every finite input.
    big = ref.abs() >= 2.0 ** 127 if kind in ("gelu_bwd", "tanh_bwd") else torch.zeros_like(ref, dtype=torch.bool)
    gf = got[fin]
    if kind == "tanh_bwd":                        # y^2 past the fp32 range: 1 - y^2 is -inf in fp32, the limit
        sq = x[fin].double() ** 2 >= 2.0 ** 128
        d = dy[fin].double()
        assert torch.equal(gf[sq & (d != 0)].double(), -torch.sign(d[sq & (d != 0)]) * float("inf"))
        big = big | sq
    ok = ~big
    within(gf[ok], ref[ok], bound[ok], kind + " finite inputs")
    over = ref.abs() >= rc.BF16_MAX * (1 + 2.0 ** -9)
    assert bool((torch.isinf(gf[over]) & (torch.sign(gf[over].double()) == torch.sign(ref[over]))).all()), kind
    top = big & ~over
    assert bool(((gf[top].double() - ref[top]).abs() <= bound[top]).logical_or(torch.isinf(gf[top])).all()), kind
    nan = torch.isnan(x)
    assert bool(torch.isnan(got[nan]).all()), kind + ": NaN in, NaN out"
    pinf, ninf = x == float("inf"), x == float("-inf")
    d_p, d_n = dy[pinf].float(), dy[ninf].float()
    want = {"gelu": (float("inf"), 0.0), "tanh": (1.0, -1.0)}
    if kind in want:
        assert float(got[pinf]) == want[kind][0] and float(got[ninf]) == want[kind][1], (kind, got[pinf], got[ninf])
    elif kind == "gelu_bwd":
        assert torch.equal(got[pinf].float(), d_p) and float(got[ninf]) == 0.0, (got[pinf], d_p, got[ninf])
    else:
        assert torch.equal(got[pinf].float(), -torch.sign(d_p) * float("inf"))
        assert torch.equal(got[ninf].float(), -torch.sign(d_n) * float("inf"))
    if kind in ("gelu", "tanh"):
        zero = got[x.view(torch.int16) == -32768]             # -0
        assert float(zero) == 0.0 and bool(torch.signbit(zero).all()), kind + ": -0 must keep its sign"


@pytest.mark.parametrize("kind", list(ELTWISE))
@pytest.mark.parametrize("n", [1, 7, 8 * 132 * 512 * 2 + 3])
def test_eltwise_lengths(kind, n):
    """n = 1, an odd tail, and more elements than the grid-stride cap covers in one pass"""
    g = _gen(n)
    x = (2 * torch.randn(n, device=DEV, generator=g)).to(BF16)
    dy = torch.randn(n, device=DEV, generator=g).to(BF16)
    if kind == "tanh_bwd":
        x = torch.tanh(x.float()).to(BF16)
    buf = torch.full((n + 1,), -77.0, dtype=BF16, device=DEV)
    out = buf[:n]
    if kind in ("gelu", "tanh"):
        call(ELTWISE[kind], x.data_ptr(), out.data_ptr(), n)
    else:
        call(ELTWISE[kind], dy.data_ptr(), x.data_ptr(), out.data_ptr(), n)
    torch.cuda.synchronize()
    ref, bound = rc.eltwise_ref(kind, x, dy)
    within(out, ref, bound, "%s n=%d" % (kind, n))
    assert float(buf[n]) == -77.0, "wrote past n"


# ---------------------------------------------------------------------------------------------------------
# casts
# ---------------------------------------------------------------------------------------------------------
def _cast_inputs(n, g):
    x = torch.randn(n, device=DEV, generator=g) * torch.exp2(torch.randint(-130, 128, (n,), device=DEV, generator=g)
                                                             .float())
    special = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8,
                            -(1.0 + 2.0 ** -8), 3.3961e38, -3.3961e38, 3.4e38, 1e-40, -1e-40, 2.0 ** -133,
                            1.0 + 2.0 ** -8 + 2.0 ** -20], device=DEV)
    k = min(n, special.numel())
    x[:k] = special[:k]
    if n > 64:  # ties: 8 significant bits plus exactly half an ulp, both parities
        t = torch.randint(-(2 ** 15), 2 ** 15, (n // 4,), device=DEV, generator=g).to(torch.int32)
        x[k:k + n // 4] = ((t << 16) | 0x8000).view(torch.float32)
    return x


def _same_cast(got, want):
    nan = torch.isnan(want)
    assert bool((torch.isnan(got) == nan).all())
    assert torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16))


@pytest.mark.parametrize("n", [1, 7, 8, 9, 8 * 132 * 2048 + 13])
def test_cast_f32_to_bf16_bit_exact(n):
    g = _gen(n + 1)
    src = _cast_inputs(n + 1, g)
    want = src.to(BF16)
    outs = []
    for off in (0, 1):          # vector path (16-byte aligned) and the scalar path (src and dst one element in)
        dst = torch.empty(n + 1, dtype=BF16, device=DEV)
        call("univl_cast_f32_to_bf16", src[off:].data_ptr(), dst[off:].data_ptr(), n)
        torch.cuda.synchronize()
        _same_cast(dst[off:off + n], want[off:off + n])
        outs.append(dst[off:off + n])
    # the two paths on the same values: src shifted by one element into the aligned buffer
    shifted = src[1:n + 1].clone()
    dst = torch.empty(n, dtype=BF16, device=DEV)
    call("univl_cast_f32_to_bf16", shifted.data_ptr(), dst.data_ptr(), n)
    torch.cuda.synchronize()
    assert torch.equal(dst.view(torch.int16), outs[1].view(torch.int16))


@pytest.mark.parametrize("n", [1, 7, 8, 9, 8 * 132 * 2048 + 13])
def test_cast_bf16_to_f32_exact(n):
    g = _gen(n + 2)
    src = _cast_inputs(n, g).to(BF16)
    dst = torch.full((n + 4,), -7777.0, device=DEV)
    call("univl_cast_bf16_to_f32", src.data_ptr(), dst.data_ptr(), n)
    torch.cuda.synchronize()
    want = src.float()
    nan = torch.isnan(want)
    assert bool((torch.isnan(dst[:n]) == nan).all())
    assert torch.equal(dst[:n][~nan].view(torch.int32), want[~nan].view(torch.int32))
    assert bool((dst[n:] == -7777.0).all())
    with pytest.raises(RuntimeError):
        call("univl_cast_bf16_to_f32", src[1:].data_ptr(), dst.data_ptr(), n - 1)


def test_multi_cast_table():
    g = _gen(77)
    lens = [1, 7, 9, 4097, 768 * 3 + 5, 250001]
    # each length twice: 16-byte aligned src and dst (the vector path, as the runtime's 128-byte arena slots give it)
    # and both one element in (the scalar path)
    srcs = [_cast_inputs(n + 1, g)[off:off + n] for off in (0, 1) for n in lens]
    dsts = [torch.empty(n + 1, dtype=BF16, device=DEV)[off:off + n] for off in (0, 1) for n in lens]
    lens = lens + lens
    table = torch.tensor([[s.data_ptr(), d.data_ptr(), n] for s, d, n in zip(srcs, dsts, lens)], dtype=torch.int64,
                         device=DEV)
    call("univl_multi_cast_f32_to_bf16", table.data_ptr(), len(lens), 16)
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        _same_cast(d, s.to(BF16))


# ---------------------------------------------------------------------------------------------------------
# mean pooling
# ---------------------------------------------------------------------------------------------------------
# modeling.py:352-353 and retrieval.py:38-39: text (skip_first, no guard), video (no skip, guarded)
POOL_FLAGS = {"text": (True, False), "video": (False, True)}


@pytest.mark.parametrize("which", ["text", "video"])
@pytest.mark.parametrize("N,S,H", [(32, 48, 768), (5, 12, 1024), (7, 1, 768), (1024, 12, 768)])
@pytest.mark.parametrize("l2norm", [True, False])
def test_meanpool_fwd_bwd(which, N, S, H, l2norm):
    skip_first, guard = POOL_FLAGS[which]
    if which == "text" and S == 1:
        pytest.skip("a text row is [CLS] plus at least one token")
    g = _gen(N + S + H + l2norm)
    x = torch.randn(N * S, H, device=DEV, generator=g).to(BF16)
    lens = torch.randint(1, S + 1, (N,), device=DEV, generator=g)
    if which == "text":
        lens = lens.clamp_min(2)
    mask = (torch.arange(S, device=DEV)[None, :] < lens[:, None]).long()
    if which == "video" and N > 2:
        mask[1] = 0                                     # a fully padded video: the guarded denominator
    dy = torch.randn(N, H, device=DEV, generator=g)
    xg = x.clone().requires_grad_()
    out = ops.MeanPoolFn.apply(xg, mask, N, S, skip_first, guard, l2norm)
    out.backward(dy)
    torch.cuda.synchronize()
    out = out.detach()
    ref = rc.meanpool_ref(x, mask, N, S, skip_first, guard, l2norm, dy=dy)
    what = "meanpool %s N=%d S=%d H=%d l2=%d" % (which, N, S, H, l2norm)
    within(out, ref["out"], ref["b_out"], what + " out")
    within(xg.grad, ref["dx"], ref["b_dx"], what + " dx")
    if which == "text" and N == 32 and not l2norm:     # the L2 normalisation cancels the denominator
        bad = rc.meanpool_ref(x, mask, N, S, skip_first, guard, l2norm, count_first=True)
        _rejects(out, bad["out"], ref["b_out"], "meanpool denominator counting position 0")


# ---------------------------------------------------------------------------------------------------------
# pooler similarity forward
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1024, 37])
def test_pooler_sim_fwd(N):
    H = 768
    g = _gen(N + 5)
    u = (2 * torch.randn(N, H, device=DEV, generator=g)).to(BF16)
    w = 0.05 * torch.randn(H, device=DEV, generator=g)
    b = torch.randn(1, device=DEV, generator=g)
    out = torch.empty(N, device=DEV)
    call("univl_pooler_sim_fwd", u.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, H)
    torch.cuda.synchronize()
    ref, bound = rc.pooler_sim_ref(u, w, b)
    within(out, ref, bound, "pooler_sim_fwd N=%d" % N)


# ---------------------------------------------------------------------------------------------------------
# similarity matrix and losses
# ---------------------------------------------------------------------------------------------------------
def _sim_inputs(B, H, g, peaked=True):
    t = torch.nn.functional.normalize(torch.randn(B, H, device=DEV, generator=g), dim=-1) * 4
    v = torch.nn.functional.normalize(torch.randn(B, H, device=DEV, generator=g), dim=-1) * 4
    if peaked:    # rows whose exponentials saturate: |s| about 30
        t[: B // 8] *= 1.4
        v[: B // 8] = t[: B // 8] * 0.95
    return t, v


def _call_loss(kind, sim, G, args):
    B = sim.shape[-1]
    loss = torch.empty((), device=DEV)
    dsim = torch.empty_like(sim)
    if kind == "maxmargin":
        margin, n_pair, ws, wd = args
        call("univl_maxmargin_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), B, float(margin), n_pair,
             float(ws), float(wd), G)
    elif kind == "crossen":
        call("univl_crossen_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), B, G)
    else:
        call("univl_milnce_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), args[0], args[1], G)
    return loss, dsim


@pytest.mark.parametrize("B", [32, 256])
def test_sim_matmul_and_crossen(B):
    H = 768
    g = _gen(B)
    t, v = _sim_inputs(B, H, g)
    sim = torch.empty(B, B, device=DEV)
    call("univl_sim_matmul_fwd", t.data_ptr(), v.data_ptr(), sim.data_ptr(), B, B, H, 1)
    torch.cuda.synchronize()
    s_ref, b_s = rc.sim_ref(t, v)
    within(sim, s_ref, b_s, "sim_matmul_fwd B=%d" % B)
    assert float(sim.abs().max()) > 25
    loss, dsim = _call_loss("crossen", sim, 1, None)
    torch.cuda.synchronize()
    l_ref, b_l, d_ref, b_d = rc.crossen_ref(sim)
    within(loss.view(1), l_ref.view(1), b_l.view(1), "crossen loss B=%d" % B)
    within(dsim, d_ref, b_d, "crossen dsim B=%d" % B)
    dt, dv = torch.empty_like(t), torch.empty_like(v)
    call("univl_sim_matmul_bwd", dsim.data_ptr(), t.data_ptr(), v.data_ptr(), dt.data_ptr(), dv.data_ptr(), B, B, H, 1)
    torch.cuda.synchronize()
    rdt, bdt, rdv, bdv = rc.sim_bwd_ref(d_ref, b_d, t, v)
    within(dt, rdt, bdt, "sim_matmul_bwd dt B=%d" % B)
    within(dv, rdv, bdv, "sim_matmul_bwd dv B=%d" % B)


@pytest.mark.parametrize("B,n_pair", [(32, 1), (256, 1), (96, 3), (255, 3)])
def test_maxmargin_loss(B, n_pair):
    g = _gen(B + n_pair)
    # multiples of 2^-6 keep every hinge argument at least 0.1 - 6/64 from 0: fp32 and fp64 take the same decisions
    sim = torch.round(torch.randn(B, B, device=DEV, generator=g) * 64 * 4) / 64
    sim[: B // 8] *= 7                                                  # peaked rows
    ws, wd = rc.maxmargin_weights(B // n_pair, n_pair, 0.5) if n_pair > 1 else (1.0, 1.0)
    np_arg = n_pair if n_pair > 1 else 0
    loss, dsim = _call_loss("maxmargin", sim, 1, (0.1, np_arg, ws, wd))
    torch.cuda.synchronize()
    l_ref, b_l, d_ref, b_d, _ = rc.maxmargin_ref(sim, 0.1, np_arg, ws, wd)
    within(loss.view(1), l_ref.view(1), b_l.view(1), "maxmargin loss B=%d P=%d" % (B, n_pair))
    within(dsim, d_ref, b_d, "maxmargin dsim B=%d P=%d" % (B, n_pair))
    _, _, d_bad, _, _ = rc.maxmargin_ref(sim, 0.1, np_arg, ws, wd, drop_diag=B // 2)
    _rejects(dsim, d_bad, b_d, "maxmargin dsim without one diagonal term")


@pytest.mark.parametrize("bs,P", [(32, 1), (256, 1), (32, 3), (85, 3)])
def test_milnce_loss(bs, P):
    N = bs * P
    g = _gen(N + P)
    t, v = _sim_inputs(N, 768, g)
    sim = (t @ v.t()).contiguous()
    torch.cuda.synchronize()

    def run():
        return list(_call_loss("milnce", sim, 1, (bs, P)))
    loss, dsim = _same_bits(run, launches=3)
    l_ref, b_l, d_ref, b_d = rc.milnce_ref(sim, bs, P)
    within(loss.view(1), l_ref.view(1), b_l.view(1), "milnce loss bs=%d P=%d" % (bs, P))
    within(dsim, d_ref, b_d, "milnce dsim bs=%d P=%d" % (bs, P))
    if P == 3:
        l_bad, _, _, _ = rc.milnce_ref(sim, bs, P, pick_offset=0)
        _rejects(loss.view(1), l_bad.view(1), b_l.view(1), "milnce picking row k P")


def test_grouped_losses():
    """G = 2 stacks: each group's loss, the mean over groups, dsim scaled by 1/G"""
    G, B = 2, 32
    g = _gen(99)
    sims = torch.stack([_sim_inputs(B, 768, g)[0] @ _sim_inputs(B, 768, g)[1].t() for _ in range(G)]).contiguous()
    for kind in ("crossen", "milnce"):
        loss, dsim = _call_loss(kind, sims, G, (B, 1))
        torch.cuda.synchronize()
        refs = [rc.crossen_ref(sims[k]) if kind == "crossen" else rc.milnce_ref(sims[k], B, 1) for k in range(G)]
        l_ref = sum(r[0] for r in refs) / G
        b_l = sum(r[1] for r in refs) / G + (G + 2) * U * l_ref.abs()
        within(loss.view(1), l_ref.view(1), b_l.view(1), kind + " G=2 loss")
        within(dsim, torch.stack([r[2] for r in refs]) / G, torch.stack([r[3] for r in refs]) / G * (1 + 2 * U)
               + U * torch.stack([r[2] for r in refs]).abs() / G, kind + " G=2 dsim")


# ---------------------------------------------------------------------------------------------------------
# softmax cross-entropy
# ---------------------------------------------------------------------------------------------------------
def _xent(logits, labels, V, target_mode, groups, vm=None, gscale=1.0, ld_d=None):
    T, ld = logits.shape[0], logits.stride(0)
    lse = torch.empty(T, device=DEV)
    sc = torch.empty(2 * groups, device=DEV)
    loss = torch.empty((), device=DEV)
    call("univl_softmax_xent_fwd", logits.data_ptr(), ld, labels.data_ptr(), ptr(vm), lse.data_ptr(), sc.data_ptr(),
         loss.data_ptr(), T, V, target_mode, -1, groups)
    ld_d = ld_d or V
    dl = torch.full((T, ld_d), 5.0, dtype=BF16, device=DEV)
    gs = torch.tensor([gscale], device=DEV)
    call("univl_softmax_xent_bwd", logits.data_ptr(), ld, labels.data_ptr(), ptr(vm), lse.data_ptr(), sc.data_ptr(),
         gs.data_ptr(), dl.data_ptr(), ld_d, T, V, target_mode, -1, groups)
    torch.cuda.synchronize()
    return loss, lse, sc, dl


XENT_CASES = [(0, 1, 1.0), (0, 3, 0.37), (1, 1, 1.0), (1, 3, 2.5)]


@pytest.mark.parametrize("target_mode,G,gscale", XENT_CASES)
def test_softmax_xent(target_mode, G, gscale):
    g = _gen(target_mode * 10 + G)
    if target_mode == 0:     # MLM / caption: vocabulary rows, ld = 30528
        T, V, ld = 96 * G, 30522, 30528
        logits = (3 * torch.randn(T, ld, device=DEV, generator=g))[:, :V]
        labels = torch.randint(0, V, (T,), device=DEV, generator=g)
        labels[torch.rand(T, device=DEV, generator=g) < 0.4] = -1
        labels[0], labels[1], labels[T - 1] = 0, V - 1, V - 1
        logits[2, 17] = 40.0                                           # a peaked row
        vm = None
    else:                    # MFM NCE: each group's rows against its own R frames, pair-masked
        R = 48
        T, V = R * G, R
        logits = (3 * torch.randn(T, 64, device=DEV, generator=g))[:, :V]
        vm = (torch.rand(T, device=DEV, generator=g) < 0.8).long()
        labels = torch.where(torch.rand(T, device=DEV, generator=g) < 0.7, 1, -1).to(torch.long)
        labels[vm == 0] = -1
        for k in range(G):
            vm[k * R] = 1
            labels[k * R] = 1
    loss, lse, sc, dl = _xent(logits, labels, V, target_mode, G, vm, gscale, ld_d=-(-V // 64) * 64)
    gscale = float(np.float32(gscale))
    ref = rc.xent_ref(logits, labels, V, target_mode, G, pair_mask=vm, gscale=gscale)
    what = "softmax_xent mode=%d G=%d" % (target_mode, G)
    within(lse, ref["lse"], ref["b_lse"], what + " lse")
    within(loss.view(1), ref["loss"].view(1), ref["b_loss"].view(1), what + " loss")
    assert torch.equal(sc[G:].double(), ref["count"])
    within(dl[:, :V], ref["dl"], ref["b_dl"], what + " dlogits")
    assert bool((dl[:, V:] == 0).all()), "columns [V, ld_d) must be zero"
    first = int(torch.nonzero(labels != -1)[0])
    bad = rc.xent_ref(logits, labels, V, target_mode, G, pair_mask=vm, gscale=gscale, drop_row=first)
    _rejects(loss.view(1), bad["loss"].view(1), ref["b_loss"].view(1), "xent loss without one scored row")
    again = _xent(logits, labels, V, target_mode, G, vm, gscale, ld_d=-(-V // 64) * 64)
    assert torch.equal(again[0], loss) and torch.equal(again[2], sc), "the loss sums its rows in a fixed order"


def test_cast_truncation_is_rejected():
    """round-to-nearest-even against truncation on the tie and round-up inputs: the perturbed cast differs"""
    g = _gen(3)
    src = _cast_inputs(4096, g)
    dst = torch.empty(4096, dtype=BF16, device=DEV)
    call("univl_cast_f32_to_bf16", src.data_ptr(), dst.data_ptr(), 4096)
    torch.cuda.synchronize()
    trunc = (src.view(torch.int32) >> 16).to(torch.int16)
    fin = torch.isfinite(src)
    assert not torch.equal(dst.view(torch.int16)[fin], trunc[fin])
