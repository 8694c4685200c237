"""GPU: each C-ABI kernel against a plain PyTorch fp32 statement of the same op on the same (bf16-rounded) inputs,
plus the reference's semantic edge cases (SURVEY.md §4): -10000 additive mask on fully masked rows, causal mask
applied once, zero frames, guarded denominators, eps inside the sqrt, ragged / non-multiple-of-tile shapes."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import attn_check as ac  # noqa: E402
from tests import gemm_check as gc  # noqa: E402
from tests.layer_check import colsum_bound  # noqa: E402
from tests.row_check import ln_bwd64 as _ln_bwd64  # noqa: E402
from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402

DEV = "cuda"
# device-resident dropout RNG state {seed, epoch} (the kernels' `rng_state` argument)
RNG = torch.tensor([123, 0], dtype=torch.int64, device=DEV) if torch.cuda.is_available() else None


def _bf(t):
    return t.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------
# GEMM: the automatic plan and every epilogue, per element against fp64 (tests/gemm_check.py; the template instances,
# split-K, scalar path and production shapes are in tests/test_gpu_gemm.py)
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("shape", [(128, 64, 64), (300, 200, 136), (1536, 768, 768), (520, 30522, 768)])
def test_gemm_all_operand_majors(a_mn, b_mn, shape):
    """automatic plan (tile width and split-K chosen by the library); MN-major extents that are not multiples of 8 are
    stored with the leading dimension padded to 64, as the vocab projection stores them"""
    M, N, K = shape
    g = torch.Generator(device=DEV).manual_seed(1)
    A, B = gc.bf_randn((M, K), 0.5, g), gc.bf_randn((N, K), 0.5, g)
    As, Bs = gc.store(A, a_mn, 64), gc.store(B, b_mn, 64)
    gc.run_epi(ops.EPI_F32, A, B, As, Bs, a_mn, b_mn, g=g, what="auto %s a_mn%d b_mn%d F32" % (shape, a_mn, b_mn))
    gc.run_epi(ops.EPI_ATOMIC, A, B, As, Bs, a_mn, b_mn, g=g,
               what="auto %s a_mn%d b_mn%d ATOMIC" % (shape, a_mn, b_mn))


def test_reserved_sms_shrink_persistent_grids_not_results():
    """univl_set_reserved_sms: persistent kernels launched while a collective holds SMs use fewer CTAs (each walks more
    tiles); every output is unchanged — GEMM (several tile widths) and the fused attention forward / backward."""
    g = torch.Generator(device=DEV).manual_seed(4)
    cases = [(1536, 768, 768), (2560, 3072, 768), (300, 200, 136)]
    mats = [(_bf(torch.randn(M, K, device=DEV, generator=g) * 0.5), _bf(torch.randn(N, K, device=DEV, generator=g) * 0.5))
            for M, N, K in cases]
    x, w, b, mask = _fused_inputs(40, 96, 11)
    spec = ops.MaskSpec(mask, causal=False)

    def run():
        outs = []
        for (M, N, K), (A, B) in zip(cases, mats):
            out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
            outs.append(ops.gemm(A, B, M, N, K, out, epi=ops.EPI_BIAS))
        o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, 40, 96, spec)
        dqkv = torch.empty_like(qkv)
        ops.fused_attention_bwd(qkv, o, lse, o, dqkv, 40, 96, spec, p=0.0, seed=RNG.data_ptr(), stream=7)
        torch.cuda.synchronize()
        return outs + [o, lse, dqkv]
    base = run()
    try:
        for n in (16, 40):
            rt.reserve_sms(n)
            for a, c in zip(base, run()):
                assert torch.equal(a, c), n
    finally:
        rt.reserve_sms(0)
    with pytest.raises(RuntimeError):
        rt.reserve_sms(-1)


# ---------------------------------------------------------------------------------------------------------
def test_gemm_fused_epilogues():
    """each of the six epilogues on a tail shape with strided out / aux_in / aux_out (ld > N, sentinel padding, rows
    past M untouched), with alpha = 1 and a bias, then alpha != 1 and bias=None (GELU and GELU-backward keep alpha = 1:
    their callers never scale).  The GELU epilogues run at the FFN's scale (pre-activations of order 1, where gelu' is
    far from 0 and 1)."""
    M, N, K = 300, 520, 760                         # 300 % 128 = 44, 520 % 256 = 8, 760 % 64 = 56
    for epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_GELU_BWD, ops.EPI_ADD, ops.EPI_F32, ops.EPI_ATOMIC):
        for alpha, with_bias in ((1.0, True), (-0.75, False)):
            if epi in (ops.EPI_GELU, ops.EPI_GELU_BWD):
                alpha = 1.0
            g = torch.Generator(device=DEV).manual_seed(2 + epi)
            A, B = gc.bf_randn((M, K), 0.3, g), gc.bf_randn((N, K), 0.05, g)
            for a_mn, b_mn in ((0, 0), (0, 1), (1, 1)):
                gc.run_epi(epi, A, B, gc.store(A, a_mn, 8), gc.store(B, b_mn, 8), a_mn, b_mn, alpha=alpha,
                           with_bias=with_bias, ldo=N + 8, ld_aux=N + 24, g=g,
                           what="epi%d alpha%g bias%d a_mn%d b_mn%d" % (epi, alpha, with_bias, a_mn, b_mn))


# ---------------------------------------------------------------------------------------------------------
def _ln_ref(z, g, b):
    u = z.mean(-1, keepdim=True)
    s = (z - u).pow(2).mean(-1, keepdim=True)
    return g * ((z - u) / torch.sqrt(s + 1e-12)) + b


@pytest.mark.parametrize("rows,cols", [(1, 768), (37, 768), (1536, 768), (100, 1024)])
def test_layernorm_residual_fwd_bwd(rows, cols):
    g = torch.Generator(device=DEV).manual_seed(3)
    x = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    res = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    gamma = (1 + 0.1 * torch.randn(cols, device=DEV, generator=g)).requires_grad_()
    beta = (0.1 * torch.randn(cols, device=DEV, generator=g)).requires_grad_()
    y, mean, rstd = ops.layernorm_fwd(x, res, gamma.detach(), beta.detach())
    xf, rf = x.float().requires_grad_(), res.float().requires_grad_()
    ref = _ln_ref(xf + rf, gamma, beta)
    assert (y.float() - ref).abs().max() <= 2e-2
    dy = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    dy2 = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    ref.backward(dy.float() + dy2.float())
    dx, dxd, dgamma, dbeta, dbias = ops.layernorm_bwd(dy, dy2, x, res, gamma.detach(), mean, rstd)
    assert dxd is dx
    assert (dx.float() - xf.grad).abs().max() <= 3e-2 * max(1.0, float(xf.grad.abs().max()))
    torch.testing.assert_close(dgamma, gamma.grad, rtol=2e-2, atol=2e-2 * float(gamma.grad.abs().max()))
    torch.testing.assert_close(dbeta, beta.grad, rtol=2e-2, atol=2e-2 * float(beta.grad.abs().max()))
    torch.testing.assert_close(dbias, xf.grad.sum(0), rtol=3e-2, atol=3e-2 * float(xf.grad.sum(0).abs().max()) + 1e-3)


def test_layernorm_zero_rows_return_beta():
    """all-zero (masked) frames: (x - u) = 0 so NormalizeVideo returns `bias` exactly (SURVEY.md §4)."""
    cols = 1024
    x = torch.zeros(5, cols, device=DEV)
    gamma = torch.full((cols,), 1.3, device=DEV)
    beta = torch.linspace(-1, 1, cols, device=DEV)
    y = ops.VideoNormFn.apply(x.view(1, 5, cols), gamma, beta)
    assert torch.equal(y.view(5, cols), beta.to(torch.bfloat16).expand(5, cols))


def test_dropout_statistics_and_backward_mask_consistency():
    rows, cols, p = 2048, 768, 0.1
    x = torch.ones(rows, cols, device=DEV, dtype=torch.bfloat16)
    gamma, beta = torch.ones(cols, device=DEV), torch.zeros(cols, device=DEV)
    # mode 2 (dropout after LN) on a row pattern whose LN output is known: use x with two values
    x[:, ::2] = -1
    y, mean, rstd = ops.layernorm_fwd(x, None, gamma, beta, p=p, mode=2, seed=RNG.data_ptr(), stream=7)
    kept = (y != 0).float().mean().item()
    assert abs(kept - (1 - p)) < 5e-3
    vals = y[y != 0].float().abs()
    assert (vals - 1 / (1 - p)).abs().max() < 2e-2            # inverted-dropout scaling
    y2, _, _ = ops.layernorm_fwd(x, None, gamma, beta, p=p, mode=2, seed=RNG.data_ptr(), stream=7)
    assert torch.equal(y, y2)                                  # same (seed, stream) -> same mask
    y3, _, _ = ops.layernorm_fwd(x, None, gamma, beta, p=p, mode=2, seed=RNG.data_ptr(), stream=8)
    assert not torch.equal(y, y3)                              # independent streams differ
    from univl_b200.runtime import call
    call("univl_rng_advance", RNG.data_ptr())                  # next epoch: same launch arguments, fresh mask
    y4, _, _ = ops.layernorm_fwd(x, None, gamma, beta, p=p, mode=2, seed=RNG.data_ptr(), stream=7)
    assert not torch.equal(y, y4) and abs((y4 != 0).float().mean().item() - (1 - p)) < 5e-3
    RNG[1] -= 1
    # backward must regenerate the same mask: gradient is zero exactly where the output was dropped
    dy = torch.ones_like(x)
    dx, _, _, dbeta, _ = ops.layernorm_bwd(dy, None, x, None, gamma, mean, rstd, p=p, mode=2, seed=RNG.data_ptr(), stream=7,
                                           want_dbias=False)
    assert abs(float(dbeta.sum()) - float((y != 0).sum()) / (1 - p)) <= 1e-3 * rows * cols


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_seq,Sq,Sk,causal", [(3, 48, 48, False), (2, 96, 96, False), (2, 20, 52, False),
                                                 (2, 128, 128, True), (1, 224, 224, False), (2, 33, 33, True),
                                                 (3, 1, 96, False),   # Sq = 1: first-token-only last cross layer
                                                 (1024, 96, 96, False), (1024, 1, 96, False)])  # all-pairs cross encoder
def test_attention_fwd_bwd(n_seq, Sq, Sk, causal):
    H = 768
    g = torch.Generator(device=DEV).manual_seed(Sq + Sk)
    q = _bf(torch.randn(n_seq * Sq, H, device=DEV, generator=g))
    kv = _bf(torch.randn(n_seq * Sk, 2 * H, device=DEV, generator=g))
    k, v = kv[:, :H], kv[:, H:]
    lens = torch.randint(1, Sk + 1, (n_seq,), generator=torch.Generator().manual_seed(1)).to(DEV)
    mask = (torch.arange(Sk, device=DEV).unsqueeze(0) < lens.unsqueeze(1)).long()
    if n_seq > 1:
        mask[0] = 0  # a fully masked sequence: softmax of the raw scores, NOT NaN / uniform (SURVEY.md §4)
    spec = ops.MaskSpec(mask, causal=causal)
    o, lse = ops.attention_fwd(q, k, v, n_seq, Sq, Sk, spec)
    d_o = _bf(torch.randn(n_seq * Sq, H, device=DEV, generator=g))
    dq = torch.empty_like(q)
    dkv = torch.empty_like(kv)
    dbias = torch.ones(3, H, device=DEV)  # accumulated into: starts at 1
    ops.attention_bwd(q, k, v, o, lse, d_o, dq, dkv[:, :H], dkv[:, H:], n_seq, Sq, Sk, spec,
                      dbias=(dbias[0], dbias[1], dbias[2]))
    torch.cuda.synchronize()
    # every output element against fp64 (tests/attn_check.py)
    what = "attention n%d Sq%d Sk%d causal%d" % (n_seq, Sq, Sk, causal)
    ref = ac.reference(q, k, v, n_seq, Sq, Sk, mask, causal, d_o=d_o, o_kernel=o)
    ac.check_fwd(o, lse, ref, what)
    ac.check_bwd(dq, dkv[:, :H], dkv[:, H:], ref, what)
    for n, got in enumerate((dq, dkv[:, :H], dkv[:, H:])):
        # fused projection-bias gradient = column sums of the same gradient (fp32 accumulators, before the bf16
        # rounding of the stored tile): equal to the column sums of what was stored up to that rounding, 2^-9 per
        # element.  (The sums themselves may cancel to ~0 — dK columns do, exactly, in exact arithmetic — so the bound
        # is relative to the summed magnitudes, not to the sum.)
        tol = got.float().abs().sum(0) * 2.0 ** -8 + 1e-3
        assert bool(((dbias[n] - 1.0 - got.float().sum(0)).abs() <= tol).all())
    # the bias gradients are per-sequence partial rows added in order: the same bits on every launch
    def again():
        dq_, dkv_ = torch.empty_like(q), torch.empty_like(kv)
        db_ = torch.ones(3, H, device=DEV)
        ops.attention_bwd(q, k, v, o, lse, d_o, dq_, dkv_[:, :H], dkv_[:, H:], n_seq, Sq, Sk, spec,
                          dbias=(db_[0], db_[1], db_[2]))
        return [dq_, dkv_, db_]
    for a, b in zip((dq, dkv, dbias), _same_bits(again, launches=2)):
        assert torch.equal(a, b)
    # the same launch without the bias pointers leaves everything else unchanged
    dq2, dkv2 = torch.empty_like(q), torch.empty_like(kv)
    ops.attention_bwd(q, k, v, o, lse, d_o, dq2, dkv2[:, :H], dkv2[:, H:], n_seq, Sq, Sk, spec)
    assert torch.equal(dq2, dq) and torch.equal(dkv2, dkv)


def test_attention_all_pairs_mask_indexing():
    """pair p = (i, j) = (p / Nb, p % Nb) takes text mask i and video mask j (reference modeling.py:355-367)."""
    Na, Nb, W, F, H = 2, 3, 16, 16, 768
    g = torch.Generator(device=DEV).manual_seed(5)
    S = W + F
    x = _bf(torch.randn(Na * Nb * S, 3 * H, device=DEV, generator=g))
    ma = (torch.arange(W, device=DEV).unsqueeze(0) < torch.tensor([5, 16], device=DEV).unsqueeze(1)).long()
    mb = (torch.arange(F, device=DEV).unsqueeze(0) < torch.tensor([3, 16, 9], device=DEV).unsqueeze(1)).long()
    o, _ = ops.attention_fwd(x[:, :H], x[:, H:2 * H], x[:, 2 * H:], Na * Nb, S, S, ops.MaskSpec(ma, mb, all_pairs=True))
    full = torch.cat([ma.unsqueeze(1).expand(Na, Nb, W), mb.unsqueeze(0).expand(Na, Nb, F)], -1).reshape(Na * Nb, S)
    o2, _ = ops.attention_fwd(x[:, :H], x[:, H:2 * H], x[:, 2 * H:], Na * Nb, S, S, ops.MaskSpec(full))
    assert torch.equal(o, o2)


def test_attention_dropout_forward_backward_consistent():
    n_seq, S, H, p = 2, 48, 768, 0.25
    g = torch.Generator(device=DEV).manual_seed(6)
    qkv = _bf(torch.randn(n_seq * S, 3 * H, device=DEV, generator=g))
    spec = ops.MaskSpec(torch.ones(n_seq, S, dtype=torch.long, device=DEV))
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    o0, _ = ops.attention_fwd(q, k, v, n_seq, S, S, spec)
    o1, lse = ops.attention_fwd(q, k, v, n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    o2, _ = ops.attention_fwd(q, k, v, n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    assert torch.equal(o1, o2) and not torch.equal(o0, o1)
    # E[dropout(P) V] = P V: averaged over many streams the output approaches the p=0 one
    acc = torch.zeros_like(o0, dtype=torch.float32)
    n = 64
    for s in range(n):
        acc += ops.attention_fwd(q, k, v, n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=100 + s)[0].float()
    assert (acc / n - o0.float()).abs().mean() <= 3e-2
    # directional derivative check of the dropped function: <dO, O(q + e dq) - O(q)> / e ~ <dq_grad, dq>
    d_o = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    dqkv = torch.empty_like(qkv)
    ops.attention_bwd(q, k, v, o1, lse, d_o, dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:], n_seq, S, S, spec, p=p,
                      seed=RNG.data_ptr(), stream=3)
    v_dir = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    eps = 0.25
    vp = _bf(v.float() + eps * v_dir.float())
    op, _ = ops.attention_fwd(q, k, vp, n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    lhs = ((op.float() - o1.float()) * d_o.float()).sum() / eps     # O is linear in V: exact up to bf16 rounding
    rhs = (dqkv[:, 2 * H:].float() * v_dir.float()).sum()
    assert abs(float(lhs - rhs)) <= 3e-2 * abs(float(rhs)) + 1.0


# ---------------------------------------------------------------------------------------------------------
def _fused_inputs(n_seq, S, seed):
    H = 768
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    w = _bf(torch.randn(3 * H, H, device=DEV, generator=g) * 0.04)
    b = torch.randn(3 * H, device=DEV, generator=g) * 0.2
    lens = torch.randint(1, S + 1, (n_seq,), generator=torch.Generator().manual_seed(seed)).to(DEV)
    mask = (torch.arange(S, device=DEV).unsqueeze(0) < lens.unsqueeze(1)).long()
    if n_seq > 1:
        mask[0] = 0   # fully masked sequence: softmax of the raw scores (SURVEY.md §4)
    return x, w, b, mask


@pytest.mark.parametrize("n_seq,S,causal", [(3, 48, False), (2, 96, False), (5, 48, False), (2, 128, True), (3, 16, False),
                                            (9, 16, True), (4, 32, False), (3, 64, False), (2, 80, False), (1, 112, False),
                                            (40, 96, False), (301, 48, False)])
def test_fused_qkv_attention_fwd_matches_unfused_and_fp32(n_seq, S, causal):
    """ONE wgmma kernel (projection + softmax(QK^T)V) and the QKV-GEMM + attention-core pair on its q/k/v, both per
    element against fp64 (tests/attn_check.py); packed sequences (S = 16 ... 64), partial last row block, several items
    per CTA."""
    H = 768
    assert ops.fused_attention_supported(n_seq, S, H)
    x, w, b, mask = _fused_inputs(n_seq, S, S + n_seq)
    spec = ops.MaskSpec(mask, causal=causal)
    o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec)
    torch.cuda.synchronize()
    what = "fused n%d S%d causal%d" % (n_seq, S, causal)
    # the saved q/k/v per element (tests/gemm_check.py), then the attention on them against fp64 (tests/attn_check.py)
    acc, mag = gc.mm64(x, w)
    qkv_ref = acc + b.double()
    gc.within(qkv, qkv_ref, gc.elem_bound(mag, H, b.double().abs(), qkv_ref), what + " qkv")
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    ref = ac.reference(q, k, v, n_seq, S, S, mask, causal, kind="fused")
    ac.check_fwd(o, lse, ref, what)
    # the unfused pair on the kernel's own q/k/v
    o2, lse2 = ops.attention_fwd(q, k, v, n_seq, S, S, spec)
    ac.check_fwd(o2, lse2, ref, what + " unfused")
    # no q/k/v copy requested: same context
    o3, _, none = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, save_qkv=False)
    assert none is None and torch.equal(o3, o)


@pytest.mark.parametrize("n_seq,S,causal,p", [(3, 48, False, 0.0), (2, 96, False, 0.0), (2, 128, True, 0.0),
                                              (5, 32, False, 0.0), (9, 16, True, 0.0), (1, 112, False, 0.0),
                                              (40, 96, False, 0.0), (3, 48, False, 0.25), (2, 128, False, 0.25),
                                              (301, 48, False, 0.1), (1024, 96, False, 0.0), (1024, 96, False, 0.1)])
def test_fused_attention_bwd_matches_fp32_and_unfused_backward(n_seq, S, causal, p):
    """wgmma attention backward and the mma.sync backward regenerating the same row-major dropout mask, both against
    fp64 under that mask (tests/attn_check.py); bias-gradient column sums included."""
    H = 768
    x, w, b, mask = _fused_inputs(n_seq, S, 100 + S + n_seq)
    spec = ops.MaskSpec(mask, causal=causal)
    o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=7)
    g = torch.Generator(device=DEV).manual_seed(9)
    d_o = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    dqkv = torch.empty_like(qkv)
    dbias = torch.ones(3 * H, device=DEV)
    ops.fused_attention_bwd(qkv, o, lse, d_o, dqkv, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=7, dbias=dbias)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    # (a) the mma.sync backward on the same saved tensors and the same dropout layout
    dq2 = torch.empty_like(qkv)
    db2 = torch.ones(3, H, device=DEV)
    ops.attention_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], o, lse, d_o, dq2[:, :H], dq2[:, H:2 * H],
                      dq2[:, 2 * H:], n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=7,
                      dbias=(db2[0], db2[1], db2[2]), rng_layout=1)
    torch.cuda.synchronize()
    what = "fused bwd n%d S%d causal%d p%g" % (n_seq, S, causal, p)
    rng = [int(t) for t in RNG.cpu()]
    keep = ac.keep_rowmajor(rng[0], ac.kernel_stream(7, rng[1]), p, n_seq * 12, S) if p > 0 else None
    ref = ac.reference(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], n_seq, S, S, mask, causal, keep, p, d_o=d_o,
                       o_kernel=o, kind="fused")
    ac.check_fwd(o, lse, ref, what)
    ac.check_bwd(dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:], ref, what)
    ac.check_bwd(dq2[:, :H], dq2[:, H:2 * H], dq2[:, 2 * H:], ref, what + " mma.sync")
    tol = dqkv.float().abs().sum(0) * 2.0 ** -7 + 2e-3
    assert bool(((dbias - 1.0 - dqkv.float().sum(0)).abs() <= tol).all())

    def again():
        dq_, db_ = torch.empty_like(qkv), torch.ones(3 * H, device=DEV)
        ops.fused_attention_bwd(qkv, o, lse, d_o, dq_, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=7, dbias=db_)
        return [dq_, db_]
    for a, b in zip((dqkv, dbias), _same_bits(again, launches=2)):
        assert torch.equal(a, b)


def _all_pairs_fused_case(Na, Nb, W, F):
    H = 768
    S = W + F
    x, w, b, _ = _fused_inputs(Na * Nb, S, 11)
    g = torch.Generator().manual_seed(Na + W)
    ma = (torch.arange(W).unsqueeze(0) < torch.randint(1, W + 1, (Na,), generator=g).unsqueeze(1)).long().to(DEV)
    mb = (torch.arange(F).unsqueeze(0) < torch.randint(1, F + 1, (Nb,), generator=g).unsqueeze(1)).long().to(DEV)
    full = torch.cat([ma.unsqueeze(1).expand(Na, Nb, W), mb.unsqueeze(0).expand(Na, Nb, F)], -1).reshape(Na * Nb, S)
    d_o = _bf(torch.randn(Na * Nb * S, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)))
    outs = []
    for spec in (ops.MaskSpec(ma, mb, all_pairs=True), ops.MaskSpec(full)):
        o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, Na * Nb, S, spec)
        dqkv = torch.empty_like(qkv)
        dbias = torch.zeros(3 * H, device=DEV)
        ops.fused_attention_bwd(qkv, o, lse, d_o, dqkv, Na * Nb, S, spec, dbias=dbias)
        outs.append((o, lse, dqkv, dbias))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


def test_fused_qkv_attention_all_pairs_masks():
    """all-pairs masks (text mask i, video mask j for pair (i, j)) give the bits of the same masks expanded to one full
    mask, forward and backward (bias gradient included); also at the cross encoder's 32 x 32 pairs of 48 + 48 tokens"""
    _all_pairs_fused_case(3, 4, 16, 32)
    _all_pairs_fused_case(32, 32, 48, 48)


@pytest.mark.parametrize("n_seq,S", [(3, 48), (2, 96), (2, 128)])
def test_fused_qkv_attention_dropout_pairs_with_backward(n_seq, S):
    """dropout masks drawn by the fused forward (row-major layout) are regenerated by attention_bwd(rng_layout=1)"""
    H, p = 768, 0.25
    x, w, b, mask = _fused_inputs(n_seq, S, 21)
    mask[:] = 1
    spec = ops.MaskSpec(mask)
    o0, _, _ = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec)
    o1, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    o2, _, _ = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    assert torch.equal(o1, o2) and not torch.equal(o0, o1)
    acc = torch.zeros_like(o0, dtype=torch.float32)
    n = 48
    for s in range(n):
        acc += ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=100 + s)[0].float()
    assert (acc / n - o0.float()).abs().mean() <= 3e-2
    # O is linear in V = x Wv^T + bv: a step along a bias direction d moves every V row by d, so
    # <dO, O(bv + e d) - O(bv)> / e = <colsum(dV), d>, exact up to bf16 rounding — IF backward regenerates the same mask
    g = torch.Generator(device=DEV).manual_seed(5)
    d_o = _bf(torch.randn(n_seq * S, H, device=DEV, generator=g))
    dqkv = torch.empty_like(qkv)
    ops.attention_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], o1, lse, d_o, dqkv[:, :H], dqkv[:, H:2 * H],
                      dqkv[:, 2 * H:], n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=3, rng_layout=1)
    d = torch.randn(H, device=DEV, generator=g)
    eps = 0.5
    b2 = b.clone()
    b2[2 * H:] += eps * d
    op, _, _ = ops.fused_qkv_attention_fwd(x, w, b2, n_seq, S, spec, p=p, seed=RNG.data_ptr(), stream=3)
    lhs = ((op.float() - o1.float()) * d_o.float()).sum() / eps
    rhs = (dqkv[:, 2 * H:].float().sum(0) * d).sum()
    assert abs(float(lhs - rhs)) <= 3e-2 * abs(float(rhs)) + 1.0
    # and the wrong layout must NOT satisfy it (guards against the test passing vacuously)
    dq_bad = torch.empty_like(qkv)
    ops.attention_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], o1, lse, d_o, dq_bad[:, :H], dq_bad[:, H:2 * H],
                      dq_bad[:, 2 * H:], n_seq, S, S, spec, p=p, seed=RNG.data_ptr(), stream=3, rng_layout=0)
    assert not torch.equal(dq_bad, dqkv)


# ---------------------------------------------------------------------------------------------------------
def test_embeddings_text_and_sources():
    n, S, H, V = 3, 20, 768, 1000
    g = torch.Generator(device=DEV).manual_seed(7)
    word = (0.05 * torch.randn(V, H, device=DEV, generator=g)).requires_grad_()
    pos = (0.05 * torch.randn(64, H, device=DEV, generator=g)).requires_grad_()
    typ = (0.05 * torch.randn(2, H, device=DEV, generator=g)).requires_grad_()
    gamma = (1 + 0.1 * torch.randn(H, device=DEV, generator=g)).requires_grad_()
    beta = (0.1 * torch.randn(H, device=DEV, generator=g)).requires_grad_()
    ids = torch.randint(0, V, (n, S), device=DEV)
    ids[0, :5] = 7  # repeated ids exercise the scatter-add
    tids = torch.randint(0, 2, (n, S), device=DEV)

    class Holder(torch.nn.Module):
        pass
    holder = Holder()
    with rt.use_model(holder, torch.device("cuda", torch.cuda.current_device())):
        y = ops.EmbedTextFn.apply(ids, tids, word, pos, typ, gamma, beta, 0.0, True)
        dy = _bf(torch.randn(n * S, H, device=DEV, generator=g))
        y.backward(dy)
    got = {k: t.grad.clone() for k, t in dict(word=word, pos=pos, typ=typ, gamma=gamma, beta=beta).items()}
    for t in (word, pos, typ, gamma, beta):
        t.grad = None
    ref = _ln_ref(word[ids] + pos[torch.arange(S, device=DEV)].unsqueeze(0) + typ[tids], gamma, beta).view(n * S, H)
    assert (y.float() - ref).abs().max() <= 2e-2
    ref.backward(dy.float())
    for k, t in dict(word=word, pos=pos, typ=typ, gamma=gamma, beta=beta).items():
        assert (got[k] - t.grad).abs().max() <= 2e-2 * max(1.0, float(t.grad.abs().max())), k

    # sources, all-pairs: y[(i,j)] = LN(concat(a_i, b_j) + pos + type)
    Na, Nb, W, F = 2, 3, 6, 5
    a = _bf(torch.randn(Na * W, H, device=DEV, generator=g)).requires_grad_()
    b = _bf(torch.randn(Nb * F, H, device=DEV, generator=g)).requires_grad_()
    for t in (pos, typ, gamma, beta):
        t.grad = None
    with rt.use_model(holder, torch.device("cuda", torch.cuda.current_device())):
        y = ops.EmbedSrcFn.apply(a, b, Na, W, Nb, F, True, pos, typ, gamma, beta, 0.0, True)
        dy = _bf(torch.randn(Na * Nb * (W + F), H, device=DEV, generator=g))
        y.backward(dy)
    got = dict(a=a.grad.float(), b=b.grad.float(), pos=pos.grad.clone(), typ=typ.grad.clone(), gamma=gamma.grad.clone())
    for t in (pos, typ, gamma, beta):
        t.grad = None
    af = a.detach().float().view(Na, W, H).requires_grad_()
    bfl = b.detach().float().view(Nb, F, H).requires_grad_()
    cat = torch.cat([af.unsqueeze(1).expand(Na, Nb, W, H), bfl.unsqueeze(0).expand(Na, Nb, F, H)], 2)
    types = torch.cat([torch.zeros(W, dtype=torch.long), torch.ones(F, dtype=torch.long)]).to(DEV)
    ref = _ln_ref(cat + pos[:W + F] + typ[types], gamma, beta).reshape(-1, H)
    assert (y.float() - ref).abs().max() <= 2e-2
    ref.backward(dy.float())
    assert (got["a"] - af.grad.view(-1, H)).abs().max() <= 3e-2 * max(1.0, float(af.grad.abs().max()))
    assert (got["b"] - bfl.grad.view(-1, H)).abs().max() <= 3e-2 * max(1.0, float(bfl.grad.abs().max()))
    assert (got["pos"] - pos.grad).abs().max() <= 3e-2 * max(1.0, float(pos.grad.abs().max()))
    assert (got["typ"] - typ.grad).abs().max() <= 3e-2 * max(1.0, float(typ.grad.abs().max()))
    assert (got["gamma"] - gamma.grad).abs().max() <= 3e-2 * max(1.0, float(gamma.grad.abs().max()))


# ---------------------------------------------------------------------------------------------------------
def test_similarity_losses_match_oracle():
    import argparse
    from oracle import univl_oracle as O
    g = torch.Generator().manual_seed(8)
    for B, P in ((6, 1), (8, 2), (9, 3)):
        sim = torch.randn(B, B, generator=g)
        cfg = argparse.Namespace(margin=0.1, batch_size=B // P, n_gpu=1, n_pair=P, negative_weighting=1,
                                 hard_negative_rate=0.5)
        from univl_b200.modules.until_module import CrossEn, MaxMarginRankingLoss, MILNCELoss
        cases = [(MaxMarginRankingLoss(margin=0.1, negative_weighting=1, batch_size=B // P, n_pair=P,
                                       hard_negative_rate=0.5), lambda s: O.max_margin_loss(s, cfg)),
                 (CrossEn(), O.cross_en_loss),
                 (MILNCELoss(batch_size=B // P, n_pair=P), lambda s: O.mil_nce_loss(s, cfg))]
        for mod, ref_fn in cases:
            s_ref = sim.clone().requires_grad_()
            ref = ref_fn(s_ref)
            ref.backward()
            s = sim.clone().to(DEV).requires_grad_()
            got = mod(s)
            (got * 0.5).backward()
            assert abs(float(got) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref))), type(mod).__name__
            torch.testing.assert_close(s.grad.cpu() * 2, s_ref.grad, rtol=1e-4, atol=1e-6)


def test_meanpool_edge_cases():
    N, S, H = 4, 12, 768
    g = torch.Generator(device=DEV).manual_seed(9)
    x = _bf(torch.randn(N * S, H, device=DEV, generator=g))
    mask = torch.ones(N, S, dtype=torch.long, device=DEV)
    mask[1, 5:] = 0
    mask[2, :] = 0            # fully padded video: guarded denominator -> zeros (modeling.py:335-336)
    mask[3, 2:] = 0           # text with only [CLS][SEP]: position 0 excluded -> denominator 1
    out_v = ops.MeanPoolFn.apply(x, mask, N, S, False, True, False)
    xf = x.float().view(N, S, H)
    m = mask.float().unsqueeze(-1)
    den = m.sum(1)
    den[den == 0] = 1
    torch.testing.assert_close(out_v, (xf * m).sum(1) / den, rtol=1e-4, atol=1e-4)
    assert float(out_v[2].abs().max()) == 0.0
    out_t = ops.MeanPoolFn.apply(x, mask[[0, 1, 3]].contiguous(), 3, S, True, False, True)
    mt = mask[[0, 1, 3]].float().unsqueeze(-1).clone()
    mt[:, 0] = 0
    want = torch.nn.functional.normalize((xf[[0, 1, 3]] * mt).sum(1) / mt.sum(1), dim=-1)
    # rows of x are consecutive per sequence, so sequences 0,1,3 of the masked call read x rows of 0,1,2:
    want = torch.nn.functional.normalize((xf[:3] * mt).sum(1) / mt.sum(1), dim=-1)
    torch.testing.assert_close(out_t, want, rtol=1e-4, atol=1e-4)


def test_bert_adam_matches_reference_formula():
    from univl_b200.optim import FusedBertAdam
    torch.manual_seed(0)
    shapes = [(768, 768), (3072,), (5, 7)]
    params = [torch.nn.Parameter(torch.randn(s, device=DEV) * 0.1) for s in shapes]
    ref_p = [p.detach().clone() for p in params]
    opt = FusedBertAdam([{"params": params[:2], "weight_decay": 0.01, "lr": 1e-3},
                         {"params": params[2:], "weight_decay": 0.0, "lr": 3e-3}], lr=1e-3, warmup=0.1, t_total=100,
                        max_grad_norm=1.0, global_clip_norm=1.0)
    m = [torch.zeros_like(p) for p in ref_p]
    v = [torch.zeros_like(p) for p in ref_p]
    for step in range(3):
        grads = [torch.randn_like(p) * (0.5 if step else 5.0) for p in ref_p]
        for p, gr in zip(params, grads):
            p.grad = gr.clone()
        opt.step()
        # reference: driver clip over all params, then per-tensor clip, Adam without bias correction, decoupled wd
        total = torch.sqrt(sum((gr ** 2).sum() for gr in grads))
        cg = min(1.0, 1.0 / (float(total) + 1e-6))
        x = step / 100.0
        sched = x / 0.1 if x < 0.1 else max((x - 1.0) / (0.1 - 1.0), 0.0)
        for i, (p, gr) in enumerate(zip(ref_p, grads)):
            gr = gr * cg
            ct = min(1.0, 1.0 / (float(gr.norm()) + 1e-6))
            gr = gr * ct
            m[i] = 0.9 * m[i] + 0.1 * gr
            v[i] = 0.999 * v[i] + 0.001 * gr * gr
            wd, lr = (0.01, 1e-3) if i < 2 else (0.0, 3e-3)
            p -= lr * sched * (m[i] / (v[i].sqrt() + 1e-6) + wd * p)
        for p, q in zip(params, ref_p):
            torch.testing.assert_close(p.detach(), q, rtol=1e-4, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------
# ordered reductions: fp64 references at production and edge shapes, and bit-for-bit repeatability.  Every cross-block
# sum of these kernels goes through per-block partial rows added in block order (csrc/api.cu partials_reduce) or per-key
# row-ordered sums (csrc/embed.cu keyed_rows_sum_kernel), so the same launch gives the same bits, with or without SMs
# reserved for a concurrent collective.
# ---------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24


def _same_bits(run, launches=3):
    """run() -> list of tensors: identical bits over `launches` launches and with 40 SMs reserved"""
    base = [t.clone() for t in run()]
    torch.cuda.synchronize()
    for i in range(launches - 1):
        for a, b in zip(base, run()):
            assert torch.equal(a, b), "launch %d differs" % (i + 1)
    rt.reserve_sms(40)
    try:
        for a, b in zip(base, run()):
            assert torch.equal(a, b), "differs with 40 SMs reserved"
    finally:
        rt.reserve_sms(0)
    return base


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = tuple(int(v) for v in (~ok).nonzero()[0])
        raise AssertionError("%s: %d elements outside the bound; first %s: got %r ref %r bound %r"
                             % (what, int((~ok).sum()), i, float(got[i]), float(ref[i]), float(bound[i])))


@pytest.mark.parametrize("rows,cols", [(1536, 768), (98304, 3072), (1, 768), (1000, 771)])
def test_colsum_fp64_and_repeatable(rows, cols):
    """bias column sums (b1 of every FFN, the vocab bias): odd cols take the scalar loads"""
    g = torch.Generator(device=DEV).manual_seed(rows + cols)
    x = _bf(torch.randn(rows, cols, device=DEV, generator=g))

    def run():
        out = torch.ones(cols, device=DEV)          # accumulated into
        ops.colsum(x, out)
        return [out]
    got = _same_bits(run)[0]
    xd = x.double()
    _within(got - 1.0, xd.sum(0), colsum_bound(x, torch.ones(cols, device=DEV)), "colsum")


@pytest.mark.parametrize("rows,cols,p", [(1, 768, 0.0), (37, 1024, 0.0), (1536, 768, 0.1), (98304, 768, 0.1)])
def test_layernorm_bwd_param_grads_fp64_and_repeatable(rows, cols, p):
    """dgamma / dbeta / dbias (the column sums of the residual LayerNorm backward, dropout mode 1 as every block runs
    it); 98304 rows is the all-pairs cross encoder, where each CTA walks many rows into its partial"""
    g = torch.Generator(device=DEV).manual_seed(rows + cols)
    x = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    res = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    gamma = 1 + 0.1 * torch.randn(cols, device=DEV, generator=g)
    beta = 0.1 * torch.randn(cols, device=DEV, generator=g)
    dy = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    dy2 = _bf(torch.randn(rows, cols, device=DEV, generator=g))
    _, mean, rstd = ops.layernorm_fwd(x, res, gamma, beta, p=p, mode=1, seed=RNG.data_ptr(), stream=5)

    def run():
        dx, dxd, dgamma, dbeta, dbias = ops.layernorm_bwd(dy, dy2, x, res, gamma, mean, rstd, p=p, mode=1,
                                                          seed=RNG.data_ptr(), stream=5)
        return [dx, dxd, dgamma, dbeta, dbias]
    dx, dxd, dgamma, dbeta, dbias = _same_bits(run)
    scale = float(torch.tensor(1.0 / (1.0 - p), dtype=torch.float32)) if p > 0 else 1.0
    keep = (dxd != 0).double() if p > 0 else torch.ones(rows, cols, dtype=torch.float64, device=DEV)
    if p > 0:
        assert abs(float(keep.mean()) - (1 - p)) < 0.02
    z = x.double() * keep * scale + res.double()
    d = dy.double() + dy2.double()
    xhat, dz, e_xhat, e_dz = _ln_bwd64(z, d, gamma)
    n = rows + 2
    _within(dbeta, d.sum(0), n * U32 * d.abs().sum(0) + 1e-30, "dbeta")
    _within(dgamma, (d * xhat).sum(0), n * U32 * (d * xhat).abs().sum(0) + (d.abs() * e_xhat).sum(0), "dgamma")
    kd = keep * scale
    _within(dbias, (dz * kd).sum(0), n * U32 * (dz * kd).abs().sum(0) + (e_dz * kd).sum(0), "dbias")
    _within(dx, dz, e_dz + 2.0 ** -8 * dz.abs(), "dx")


def _embed_holder():
    class Holder(torch.nn.Module):
        pass
    return Holder()


def test_embed_text_table_grads_fp64_and_repeatable():
    """the text embedding backward of the FT-Align step: 32 x 48 rows, most of them [PAD] (id 0, hundreds of rows of
    one key spread over many CTAs), every sequence starting with [CLS], every position 32 times.  Word / position /
    type tables and gamma / beta against fp64 index_add_; with dropout, the same bits on every launch."""
    n, S, H, V = 32, 48, 768, 30522
    g = torch.Generator(device=DEV).manual_seed(17)
    word = 0.05 * torch.randn(V, H, device=DEV, generator=g)
    pos = 0.05 * torch.randn(512, H, device=DEV, generator=g)
    typ = 0.05 * torch.randn(2, H, device=DEV, generator=g)
    gamma = 1 + 0.1 * torch.randn(H, device=DEV, generator=g)
    beta = 0.1 * torch.randn(H, device=DEV, generator=g)
    lens = torch.randint(4, 40, (n,), generator=torch.Generator().manual_seed(3))
    ids = torch.zeros(n, S, dtype=torch.long)
    for i, L in enumerate(lens.tolist()):
        ids[i, 0] = 101                                                     # [CLS]
        ids[i, 1:L - 1] = torch.randint(1000, 3000, (L - 2,), generator=torch.Generator().manual_seed(i))
        ids[i, L - 1] = 102                                                 # [SEP]
    ids = ids.to(DEV)
    tids = torch.zeros(n, S, dtype=torch.long, device=DEV)
    tids[:, S // 2:] = 1
    dy = _bf(torch.randn(n * S, H, device=DEV, generator=g))
    holder = _embed_holder()
    dev = torch.device("cuda", torch.cuda.current_device())

    def run(p):
        ws = [t.clone().requires_grad_() for t in (word, pos, typ, gamma, beta)]
        with rt.use_model(holder, dev) as arena:
            arena.stream_counter = 0
            arena.rng_state[1] = 3                                          # same dropout epoch every launch
            y = ops.EmbedTextFn.apply(ids, tids, *ws, p, True)
            y.backward(dy)
        return [t.grad for t in ws]
    dword, dpos, dtyp, dgamma, dbeta = _same_bits(lambda: run(0.0))
    _same_bits(lambda: run(0.1), launches=2)
    # fp64 reference
    flat_ids, s_idx, t_idx = ids.reshape(-1), torch.arange(S, device=DEV).repeat(n), tids.reshape(-1)
    z = word.double()[flat_ids] + pos.double()[s_idx] + typ.double()[t_idx]
    d = dy.double()
    xhat, dz, e_xhat, e_dz = _ln_bwd64(z, d, gamma)
    for got, idx, rows_of, name in ((dword, flat_ids, V, "word"), (dpos, s_idx, 512, "position"),
                                    (dtyp, t_idx, 2, "type")):
        ref = torch.zeros(rows_of, H, dtype=torch.float64, device=DEV).index_add_(0, idx, dz)
        cnt = torch.zeros(rows_of, dtype=torch.float64, device=DEV).index_add_(0, idx, torch.ones_like(idx, dtype=torch.float64))
        mag = torch.zeros_like(ref).index_add_(0, idx, dz.abs())
        err = torch.zeros_like(ref).index_add_(0, idx, e_dz)
        _within(got, ref, (cnt.unsqueeze(1) + 2) * U32 * mag + err + 1e-30, name)
    assert int((flat_ids == 0).sum()) > 500                              # [PAD] rows span many CTAs
    nrow = n * S + 2
    _within(dbeta, d.sum(0), nrow * U32 * d.abs().sum(0), "beta")
    _within(dgamma, (d * xhat).sum(0), nrow * U32 * (d * xhat).abs().sum(0) + (d.abs() * e_xhat).sum(0), "gamma")


def test_embed_src_all_pairs_grads_fp64_and_repeatable():
    """the cross embedding of the all-pairs FT-Align step: Na = Nb = 32, W = F = 48 (98304 rows).  Position, type,
    gamma, beta and the source gradients da / db (each summed over its 32-way fan-out) against fp64."""
    Na, Nb, W, F, H = 32, 32, 48, 48, 768
    S = W + F
    g = torch.Generator(device=DEV).manual_seed(23)
    a = _bf(torch.randn(Na * W, H, device=DEV, generator=g))
    b = _bf(torch.randn(Nb * F, H, device=DEV, generator=g))
    pos = 0.05 * torch.randn(512, H, device=DEV, generator=g)
    typ = 0.05 * torch.randn(2, H, device=DEV, generator=g)
    gamma = 1 + 0.1 * torch.randn(H, device=DEV, generator=g)
    beta = 0.1 * torch.randn(H, device=DEV, generator=g)
    dy = _bf(torch.randn(Na * Nb * S, H, device=DEV, generator=g))
    holder = _embed_holder()
    dev = torch.device("cuda", torch.cuda.current_device())

    def run():
        av, bv = a.clone().requires_grad_(), b.clone().requires_grad_()
        ws = [t.clone().requires_grad_() for t in (pos, typ, gamma, beta)]
        with rt.use_model(holder, dev):
            y = ops.EmbedSrcFn.apply(av, bv, Na, W, Nb, F, True, *ws, 0.0, True)
            y.backward(dy)
        return [av.grad, bv.grad] + [t.grad for t in ws]
    da, db, dpos, dtyp, dgamma, dbeta = _same_bits(run)
    cat = torch.cat([a.double().view(Na, 1, W, H).expand(Na, Nb, W, H), b.double().view(1, Nb, F, H).expand(Na, Nb, F, H)],
                    2)
    types = torch.cat([torch.zeros(W, dtype=torch.long), torch.ones(F, dtype=torch.long)]).to(DEV)
    z = (cat + pos.double()[:S] + typ.double()[types]).reshape(-1, H)
    del cat
    d = dy.double()
    xhat, dz, e_xhat, e_dz = _ln_bwd64(z, d, gamma)
    dz4, e4, m4 = dz.view(Na, Nb, S, H), e_dz.view(Na, Nb, S, H), dz.abs().view(Na, Nb, S, H)
    R = Na * Nb + 2
    _within(dpos[:S], dz4.sum((0, 1)), R * U32 * m4.sum((0, 1)) + e4.sum((0, 1)), "position")
    assert bool((dpos[S:] == 0).all())
    for t, sl in ((0, slice(0, W)), (1, slice(W, S))):
        _within(dtyp[t], dz4[:, :, sl].sum((0, 1, 2)), (R * S) * U32 * m4[:, :, sl].sum((0, 1, 2))
                + e4[:, :, sl].sum((0, 1, 2)), "type %d" % t)
    ref_a = dz4[:, :, :W].sum(1).reshape(-1, H)
    _within(da, ref_a, (Nb + 2) * U32 * m4[:, :, :W].sum(1).reshape(-1, H) + e4[:, :, :W].sum(1).reshape(-1, H)
            + 2.0 ** -8 * ref_a.abs(), "da")
    ref_b = dz4[:, :, W:].sum(0).reshape(-1, H)
    _within(db, ref_b, (Na + 2) * U32 * m4[:, :, W:].sum(0).reshape(-1, H) + e4[:, :, W:].sum(0).reshape(-1, H)
            + 2.0 ** -8 * ref_b.abs(), "db")
    nrow = z.shape[0] + 2
    _within(dbeta, d.sum(0), nrow * U32 * d.abs().sum(0), "beta")
    _within(dgamma, (d * xhat).sum(0), nrow * U32 * (d * xhat).abs().sum(0) + (d.abs() * e_xhat).sum(0), "gamma")


@pytest.mark.parametrize("N", [1024, 37])
def test_pooler_sim_bwd_param_grads_fp64_and_repeatable(N):
    """similarity head dw / db over the N = 32 x 32 pooled pairs, and N not a multiple of the 16 rows per CTA"""
    H = 768
    g = torch.Generator(device=DEV).manual_seed(N)
    u = _bf(torch.randn(N, H, device=DEV, generator=g))
    w = 0.05 * torch.randn(H, device=DEV, generator=g)
    dout = torch.randn(N, device=DEV, generator=g)
    from univl_b200.runtime import call

    def run():
        du = torch.empty(N, H, device=DEV, dtype=torch.bfloat16)
        dw, db = torch.ones(H, device=DEV), torch.ones(1, device=DEV)        # accumulated into
        call("univl_pooler_sim_bwd", u.data_ptr(), w.data_ptr(), dout.data_ptr(), du.data_ptr(), dw.data_ptr(),
             db.data_ptr(), N, H)
        return [du, dw, db]
    du, dw, db = _same_bits(run)
    th = torch.tanh(u.double())
    d = dout.double()
    # tanhf compiles to MUFU.TANH under --use_fast_math: relative error below 2^-10.9
    th_err = 2.0 ** -10 * th.abs() + 2.0 ** -20
    terms = (d.unsqueeze(1) * th).abs().sum(0)
    _within(dw - 1.0, (d.unsqueeze(1) * th).sum(0), (N + 2) * U32 * terms + (d.abs().unsqueeze(1) * th_err).sum(0), "dw")
    _within(db - 1.0, d.sum().view(1), (N + 2) * U32 * d.abs().sum().view(1), "db")
    dw_ = (d.unsqueeze(1) * w.double()).abs()
    ref_du = d.unsqueeze(1) * w.double() * (1 - th * th)
    _within(du, ref_du, 2.0 ** -8 * ref_du.abs() + dw_ * (2 * th.abs() * th_err + 4 * U32), "du")
