"""GPU: each C-ABI kernel against a plain PyTorch fp32 statement of the same op on the same (bf16-rounded) inputs,
plus the reference's semantic edge cases (SURVEY.md §4): -10000 additive mask on fully masked rows, causal mask
applied once, zero frames, guarded denominators, eps inside the sqrt, ragged / non-multiple-of-tile shapes."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402

DEV = "cuda"
# device-resident dropout RNG state {seed, epoch} (the kernels' `rng_state` argument)
RNG = torch.tensor([123, 0], dtype=torch.int64, device=DEV) if torch.cuda.is_available() else None


def _bf(t):
    return t.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("shape", [(128, 64, 64), (300, 200, 136), (1536, 768, 768), (520, 30522, 768)])
def test_gemm_all_operand_majors(a_mn, b_mn, shape):
    M, N, K = shape
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major storage needs the MN extent to be a multiple of 8")
    g = torch.Generator(device=DEV).manual_seed(1)
    A = _bf(torch.randn(M, K, device=DEV, generator=g) * 0.5)
    B = _bf(torch.randn(N, K, device=DEV, generator=g) * 0.5)
    bias = torch.randn(N, device=DEV, generator=g)
    ref = A.float() @ B.float().t() + bias
    Am = A.t().contiguous() if a_mn else A
    Bm = B.t().contiguous() if b_mn else B
    out = torch.empty(M, N, device=DEV, dtype=torch.float32)
    ops.gemm(Am, Bm, M, N, K, out, epi=ops.EPI_F32, bias=bias, a_mn=a_mn, b_mn=b_mn)
    assert (out - ref).abs().max() <= 2e-3 * ref.abs().max()
    acc = torch.ones(M, N, device=DEV)
    ops.gemm(Am, Bm, M, N, K, acc, epi=ops.EPI_ATOMIC, a_mn=a_mn, b_mn=b_mn)  # split-K + accumulate
    assert (acc - (ref - bias + 1.0)).abs().max() <= 2e-3 * ref.abs().max()


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
    M, N, K = 384, 3072, 768
    g = torch.Generator(device=DEV).manual_seed(2)
    A = _bf(torch.randn(M, K, device=DEV, generator=g) * 0.3)
    B = _bf(torch.randn(N, K, device=DEV, generator=g) * 0.05)
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    pre_ref = A.float() @ B.float().t() + bias
    pre = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    h = torch.empty_like(pre)
    ops.gemm(A, B, M, N, K, h, epi=ops.EPI_GELU, bias=bias, aux_out=pre)
    gelu_ref = pre_ref * 0.5 * (1 + torch.erf(pre_ref / math.sqrt(2)))
    assert (pre.float() - pre_ref).abs().max() <= 2e-2
    assert (h.float() - gelu_ref).abs().max() <= 2e-2
    # gelu backward epilogue: out = acc * gelu'(aux)
    dy = _bf(torch.randn(M, K, device=DEV, generator=g) * 0.3)
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(dy, B, M, N, K, out, epi=ops.EPI_GELU_BWD, aux_in=pre)
    x = pre.float()
    gp = 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    ref = (dy.float() @ B.float().t()) * gp
    assert (out.float() - ref).abs().max() <= 3e-2 * max(1.0, float(ref.abs().max()))


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
def _attn_ref(q, k, v, add_mask):
    s = torch.matmul(q, k.transpose(-1, -2)) / 8.0 + add_mask
    return torch.matmul(torch.softmax(s, -1), v)


@pytest.mark.parametrize("n_seq,Sq,Sk,causal", [(3, 48, 48, False), (2, 96, 96, False), (2, 20, 52, False),
                                                 (2, 128, 128, True), (1, 224, 224, False), (2, 33, 33, True),
                                                 (3, 1, 96, False)])  # Sq = 1: first-token-only last cross layer
def test_attention_fwd_bwd(n_seq, Sq, Sk, causal):
    H, h = 768, 12
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

    def heads(t, S):
        return t.float().view(n_seq, S, h, 64).permute(0, 2, 1, 3)
    qf, kf, vf = heads(q, Sq).requires_grad_(), heads(k, Sk).requires_grad_(), heads(v, Sk).requires_grad_()
    add = (1.0 - mask.float()).view(n_seq, 1, 1, Sk) * -10000.0
    if causal:
        fut = torch.triu(torch.ones(Sq, Sk, device=DEV), diagonal=1).view(1, 1, Sq, Sk)
        add = ((1.0 - mask.float()).view(n_seq, 1, 1, Sk) + fut).gt(0).float() * -10000.0
    ref = _attn_ref(qf, kf, vf, add)
    ref2d = ref.permute(0, 2, 1, 3).reshape(n_seq * Sq, H)
    assert torch.isfinite(o.float()).all()
    assert (o.float() - ref2d).abs().max() <= 3e-2
    d_o = _bf(torch.randn(n_seq * Sq, H, device=DEV, generator=g))
    ref2d.backward(d_o.float())
    dq = torch.empty_like(q)
    dkv = torch.empty_like(kv)
    dbias = torch.ones(3, H, device=DEV)  # accumulated into: starts at 1
    ops.attention_bwd(q, k, v, o, lse, d_o, dq, dkv[:, :H], dkv[:, H:], n_seq, Sq, Sk, spec,
                      dbias=(dbias[0], dbias[1], dbias[2]))

    def unheads(t, S):
        return t.permute(0, 2, 1, 3).reshape(n_seq * S, H)
    for n, (got, want, S) in enumerate(((dq, qf.grad, Sq), (dkv[:, :H], kf.grad, Sk), (dkv[:, H:], vf.grad, Sk))):
        want = unheads(want, S)
        assert (got.float() - want).abs().max() <= 4e-2 * max(1.0, float(want.abs().max()))
        # fused projection-bias gradient = column sums of the same gradient (fp32 accumulators, before the bf16
        # rounding of the stored tile): equal to the column sums of what was stored up to that rounding, 2^-9 per
        # element.  (The sums themselves may cancel to ~0 — dK columns do, exactly, in exact arithmetic — so the bound
        # is relative to the summed magnitudes, not to the sum.)
        tol = got.float().abs().sum(0) * 2.0 ** -8 + 1e-3
        assert bool(((dbias[n] - 1.0 - got.float().sum(0)).abs() <= tol).all())
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
    """ONE wgmma kernel (projection + softmax(QK^T)V) against (a) fp32 PyTorch on the same bf16 inputs and (b) the
    QKV-GEMM + attention-core pair; packed sequences (S = 16 ... 64), partial last row block, several items per CTA."""
    H, h = 768, 12
    assert ops.fused_attention_supported(n_seq, S, H)
    x, w, b, mask = _fused_inputs(n_seq, S, S + n_seq)
    spec = ops.MaskSpec(mask, causal=causal)
    o, lse, qkv = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec)
    torch.cuda.synchronize()
    assert torch.isfinite(o.float()).all() and torch.isfinite(lse).all()
    qkv_ref = _bf(x.float() @ w.float().t() + b)                      # the kernel rounds q/k/v to bf16 operand tiles
    assert (qkv.float() - qkv_ref.float()).abs().max() <= 2.0 ** -7 * max(1.0, float(qkv_ref.float().abs().max()))

    def heads(t):
        return t.float().view(n_seq, S, h, 64).permute(0, 2, 1, 3)
    qf, kf, vf = heads(qkv_ref[:, :H]), heads(qkv_ref[:, H:2 * H]), heads(qkv_ref[:, 2 * H:])
    add = (1.0 - mask.float()).view(n_seq, 1, 1, S) * -10000.0
    if causal:
        fut = torch.triu(torch.ones(S, S, device=DEV), diagonal=1).view(1, 1, S, S)
        add = ((1.0 - mask.float()).view(n_seq, 1, 1, S) + fut).gt(0).float() * -10000.0
    sc = torch.matmul(qf, kf.transpose(-1, -2)) / 8.0 + add
    ref = torch.matmul(torch.softmax(sc, -1), vf).permute(0, 2, 1, 3).reshape(n_seq * S, H)
    assert (o.float() - ref).abs().max() <= 3e-2
    lse_ref = torch.logsumexp(sc, -1).reshape(-1)
    assert (lse - lse_ref).abs().max() <= 2e-2 + 2e-3 * float(lse_ref.abs().max())
    # the unfused pair on the kernel's own q/k/v
    o2, lse2 = ops.attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], n_seq, S, S, spec)
    assert (o.float() - o2.float()).abs().max() <= 2e-2
    assert (lse - lse2).abs().max() <= 2e-3 * max(1.0, float(lse2.abs().max()))
    # no q/k/v copy requested: same context
    o3, _, none = ops.fused_qkv_attention_fwd(x, w, b, n_seq, S, spec, save_qkv=False)
    assert none is None and torch.equal(o3, o)


@pytest.mark.parametrize("n_seq,S,causal,p", [(3, 48, False, 0.0), (2, 96, False, 0.0), (2, 128, True, 0.0),
                                              (5, 32, False, 0.0), (9, 16, True, 0.0), (1, 112, False, 0.0),
                                              (40, 96, False, 0.0), (3, 48, False, 0.25), (2, 128, False, 0.25),
                                              (301, 48, False, 0.1)])
def test_fused_attention_bwd_matches_fp32_and_unfused_backward(n_seq, S, causal, p):
    """wgmma attention backward: (p = 0) against fp32 autograd of the same op, and (any p) against the mma.sync
    backward kernel regenerating the same row-major dropout mask; bias-gradient column sums included."""
    H, h = 768, 12
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
    scale = max(1.0, float(dq2.float().abs().max()))
    assert (dqkv.float() - dq2.float()).abs().max() <= 3e-2 * scale
    rel = float((dqkv.float() - dq2.float()).norm() / dq2.float().norm())
    assert rel <= 1e-2, rel
    tol = dqkv.float().abs().sum(0) * 2.0 ** -7 + 2e-3
    assert bool(((dbias - 1.0 - dqkv.float().sum(0)).abs() <= tol).all())
    if p == 0.0:
        # (b) fp32 autograd
        def heads(t):
            return t.float().view(n_seq, S, h, 64).permute(0, 2, 1, 3)
        qf = heads(qkv[:, :H]).requires_grad_()
        kf = heads(qkv[:, H:2 * H]).requires_grad_()
        vf = heads(qkv[:, 2 * H:]).requires_grad_()
        add = (1.0 - mask.float()).view(n_seq, 1, 1, S) * -10000.0
        if causal:
            fut = torch.triu(torch.ones(S, S, device=DEV), diagonal=1).view(1, 1, S, S)
            add = ((1.0 - mask.float()).view(n_seq, 1, 1, S) + fut).gt(0).float() * -10000.0
        ref = _attn_ref(qf, kf, vf, add).permute(0, 2, 1, 3).reshape(n_seq * S, H)
        ref.backward(d_o.float())
        for n, gr in enumerate((qf.grad, kf.grad, vf.grad)):
            want = gr.permute(0, 2, 1, 3).reshape(n_seq * S, H)
            got = dqkv[:, n * H:(n + 1) * H].float()
            assert (got - want).abs().max() <= 4e-2 * max(1.0, float(want.abs().max())), n


def test_fused_qkv_attention_all_pairs_masks():
    Na, Nb, W, F, H = 3, 4, 16, 32, 768
    S = W + F
    x, w, b, _ = _fused_inputs(Na * Nb, S, 11)
    ma = (torch.arange(W, device=DEV).unsqueeze(0) < torch.tensor([5, 16, 1], device=DEV).unsqueeze(1)).long()
    mb = (torch.arange(F, device=DEV).unsqueeze(0) < torch.tensor([3, 32, 9, 20], device=DEV).unsqueeze(1)).long()
    o, _, _ = ops.fused_qkv_attention_fwd(x, w, b, Na * Nb, S, ops.MaskSpec(ma, mb, all_pairs=True))
    full = torch.cat([ma.unsqueeze(1).expand(Na, Nb, W), mb.unsqueeze(0).expand(Na, Nb, F)], -1).reshape(Na * Nb, S)
    o2, _, _ = ops.fused_qkv_attention_fwd(x, w, b, Na * Nb, S, ops.MaskSpec(full))
    assert torch.equal(o, o2)


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
