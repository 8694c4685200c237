"""GPU: the persistent wgmma GEMM (csrc/gemm_wgmma.cu) against an fp64 statement of the same product
(tests/gemm_check.py: per-element bounds).

Every template instance (block_n in {64, 128, 256} x the four operand-major combinations) on tail and many-tile
shapes with MN-major operands stored in padded leading dimensions (the vocab layout), the scalar epilogue path, forced
split-K plans, the production GEMMs of one FT-Align and one caption step, and the argument checks.  The automatic-plan
and per-epilogue tests (test_gemm_all_operand_majors, test_gemm_fused_epilogues) are in test_gpu_kernels.py and use the
same checker."""
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.gemm_check import (BF16, BF16_ROUND, C_ACC, DEV, EPI_ROUND, GELU_ABS, GELU_LIP, OUT_F32, U,  # noqa: E402
                              bf_randn, elem_bound, gelu64, gelu_grad64, mm64, run_epi, store, within)
from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402


# ---------------------------------------------------------------------------------------------------------
# the checker itself
# ---------------------------------------------------------------------------------------------------------
def test_checker_rejects_a_dropped_k_slice_and_a_missing_tail_bias():
    """the per-element bound is tight enough to see one 16-wide k slice missing from the reference, or the bias of a
    single tail row missing, on a kernel output that passes against the correct reference"""
    g = torch.Generator(device=DEV).manual_seed(11)
    M, N, K = 300, 200, 200
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.5, g)
    bias = torch.randn(N, device=DEV, generator=g)
    out = torch.empty(M, N, device=DEV, dtype=torch.float32)
    ops.gemm(A, B, M, N, K, out, epi=ops.EPI_F32, bias=bias)
    acc, mag = mm64(A, B)
    b64 = bias.double()
    bound = elem_bound(mag, K, b64.abs())
    within(out, acc + b64, bound, "checker: correct reference")
    keep = torch.ones(K, dtype=torch.float64, device=DEV)
    keep[K - 24:K - 8] = 0.0                      # one 16-wide k slice inside the last k-block
    short = (A.double() * keep) @ B.double().t() + b64
    with pytest.raises(AssertionError):
        within(out, short, bound, "checker: k slice dropped")
    no_bias = (acc + b64).clone()
    no_bias[M - 1] -= b64                           # the last (tail) row without its bias
    with pytest.raises(AssertionError):
        within(out, no_bias, bound, "checker: tail row bias missing")


# ---------------------------------------------------------------------------------------------------------
# every template instance
# ---------------------------------------------------------------------------------------------------------
INSTANCES = [(bn, a_mn, b_mn) for bn in (64, 128, 256) for a_mn in (0, 1) for b_mn in (0, 1)]


@pytest.mark.parametrize("block_n,a_mn,b_mn", INSTANCES)
def test_gemm_instance_tail_and_many_tile_shapes(block_n, a_mn, b_mn):
    """tail: M % 128 not in {0, 64}, N % block_n != 0, K % 64 in {8, 56} (one K < 64), M / N not multiples of 8 stored
    MN-major in buffers padded to 8 or 64.  many-tile: > 132 work items, more k-blocks than pipeline stages, so every
    CTA walks several tiles and the mbarrier ring wraps across tiles."""
    g = torch.Generator(device=DEV).manual_seed(100 + block_n + 2 * a_mn + b_mn)
    tails = [(301, 2 * block_n + 37, 200, 8), (173, block_n + 5, 120, 64), (45, block_n - 3, 56, 8)]
    for M, N, K, pad in tails:
        A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.5, g)
        run_epi(ops.EPI_F32, A, B, store(A, a_mn, pad), store(B, b_mn, pad), a_mn, b_mn, block_n=block_n, g=g,
                 ldo=N + 3, what="tail %s bn%d a_mn%d b_mn%d" % ((M, N, K), block_n, a_mn, b_mn))
    M, N, K = 1200, 3400, 696                      # work items: 140 / 270 / 540; 11 k-blocks > 4 / 6 / 8 stages
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.5, g)
    run_epi(ops.EPI_F32, A, B, store(A, a_mn, 8), store(B, b_mn, 8), a_mn, b_mn, block_n=block_n, g=g,
             what="many-tile bn%d a_mn%d b_mn%d" % (block_n, a_mn, b_mn))


# ---------------------------------------------------------------------------------------------------------
# the scalar epilogue path
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi", [ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_ADD, ops.EPI_F32, ops.EPI_ATOMIC])
@pytest.mark.parametrize("layout", ["odd_n", "odd_ld", "offset"])
def test_gemm_scalar_epilogue_path(epi, layout):
    """outputs that cannot take 2-element vector stores (odd N with an unpadded output, odd ldo, a base one element
    off alignment) run the scalar epilogue: fp64-exact within the bound, and bit-identical to the vector path on the
    same accumulators"""
    g = torch.Generator(device=DEV).manual_seed(40 + epi)
    M, N, K = 200, (201 if layout == "odd_n" else 200), 136
    A, B = bf_randn((M, K), 0.3, g), bf_randn((N, K), 0.1, g)
    f32 = epi in OUT_F32
    dt = torch.float32 if f32 else BF16
    bias = torch.randn(N, device=DEV, generator=g) if epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_F32) else None
    aux_in = bf_randn((M, N + N % 2), 1.0, g)[:, :N] if epi == ops.EPI_ADD else None   # even ld: vector-capable
    init = torch.randn(M, N, device=DEV, generator=g).to(dt)

    def run(out, aux_out=None):
        out.copy_(init)
        ops.gemm(A, B, M, N, K, out, epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, split_k=1)
        return out

    # vector path: aligned, even leading dimension
    vbuf = torch.empty(M, N + 1 if N % 2 else N + 2, dtype=dt, device=DEV)
    vaux = torch.empty(M, vbuf.shape[1], dtype=BF16, device=DEV)[:, :N] if epi == ops.EPI_GELU else None
    vec = run(vbuf[:, :N], vaux)
    if layout == "odd_n":
        sbuf = torch.empty(M, N, dtype=dt, device=DEV)
        sout = sbuf
    elif layout == "odd_ld":
        sbuf = torch.empty(M, N + 1, dtype=dt, device=DEV)
        sout = sbuf[:, :N]
    else:
        flat = torch.empty(M * (N + 2) + 1, dtype=dt, device=DEV)
        sout = flat[1:].view(M, N + 2)[:, :N]
    saux = torch.empty(M, N + 1, dtype=BF16, device=DEV)[:, :N] if epi == ops.EPI_GELU else None
    sc = run(sout, saux)
    torch.cuda.synchronize()
    assert torch.equal(sc, vec), layout
    if saux is not None:
        assert torch.equal(saux, vaux), layout
    acc, mag = mm64(A, B)
    b64 = bias.double() if bias is not None else 0.0
    what = "scalar %s epi%d" % (layout, epi)
    if epi == ops.EPI_GELU:
        pre = acc + b64
        bpre = elem_bound(mag, K, b64.abs())
        within(saux, pre, bpre + BF16_ROUND * pre.abs(), what + " aux_out")
        ref = gelu64(pre)
        within(sc, ref, GELU_LIP * bpre + GELU_ABS * pre.abs() + BF16_ROUND * ref.abs(), what)
    elif epi == ops.EPI_ADD:
        ref = acc + aux_in.double()
        within(sc, ref, elem_bound(mag, K, aux_in.double().abs(), ref), what)
    elif epi == ops.EPI_ATOMIC:
        ref = acc + init.double()
        within(sc, ref, elem_bound(mag, K, init.double().abs()), what)
    else:
        ref = acc + b64
        within(sc, ref, elem_bound(mag, K, b64.abs(), None if f32 else ref), what)


# ---------------------------------------------------------------------------------------------------------
# split-K
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,split_k", [(448, 1), (448, 2), (448, 3), (448, 7), (448, 9), (200, 7)])
def test_gemm_split_k_exact_and_bitwise_repeatable(K, split_k):
    """forced splits (448 = 7 k-blocks: 2 -> 4 + 3 and 3 -> 3 + 3 + 1 leave an uneven last split; 9 > 7 and 7 > 4
    k-blocks are clamped) added into a non-zero strided output: within the fp64 bound, and the same bits on a second
    launch and with 16 or 40 SMs reserved — the plan is a function of the problem, not of the free SMs"""
    g = torch.Generator(device=DEV).manual_seed(50 + K + split_k)
    M, N = 300, 200
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.5, g)
    for a_mn, b_mn, bn in ((1, 1, 128), (0, 0, 64)):
        As, Bs = store(A, a_mn, 8), store(B, b_mn, 8)
        alpha = 0.5 if bn == 64 else 1.0
        run_epi(ops.EPI_ATOMIC, A, B, As, Bs, a_mn, b_mn, alpha=alpha, ldo=N + 16, block_n=bn,
                         split_k=split_k, g=g, what="split_k %d K %d a_mn%d b_mn%d" % (split_k, K, a_mn, b_mn))
        init = torch.randn(M, N, device=DEV, generator=g)

        def run():
            out = torch.empty(M, N + 16, device=DEV)[:, :N]
            out.copy_(init)
            ops.gemm(As, Bs, M, N, K, out, epi=ops.EPI_ATOMIC, a_mn=a_mn, b_mn=b_mn, alpha=alpha, block_n=bn,
                     split_k=split_k)
            torch.cuda.synchronize()
            return out
        base = run()
        assert torch.equal(run(), base)
        try:
            for n in (16, 40):
                rt.reserve_sms(n)
                assert torch.equal(run(), base), n
        finally:
            rt.reserve_sms(0)


# ---------------------------------------------------------------------------------------------------------
# the GEMMs of one FT-Align step (batch 32, 48 words, 48 frames: 1536-row text / visual stacks, 32 x 32 all-pairs
# cross encoder = 98304 rows) and one caption step (vocab 30522, logits padded to 30528)
# ---------------------------------------------------------------------------------------------------------
H, I, V, LDV = 768, 3072, 30522, 30528
PROD = {
    # name: (T, kind, N, K, epilogue)   kind: fwd X W^T | dgrad dY W | wgrad dY^T X
    "text_qkv_fwd": (1536, "fwd", 3 * H, H, ops.EPI_BIAS),
    "text_ffn1_fwd": (1536, "fwd", I, H, ops.EPI_GELU),
    "text_ffn2_fwd": (1536, "fwd", H, I, ops.EPI_BIAS),
    "text_attn_dgrad_add": (1536, "dgrad", H, 3 * H, ops.EPI_ADD),
    "text_qkv_wgrad": (1536, "wgrad", 3 * H, H, ops.EPI_ATOMIC),
    "visual_in_fwd": (1536, "fwd", H, 1024, ops.EPI_BIAS),
    "visual_in_wgrad": (1536, "wgrad", H, 1024, ops.EPI_ATOMIC),
    "cross_ffn1_fwd": (98304, "fwd", I, H, ops.EPI_GELU),
    "cross_ffn2_fwd": (98304, "fwd", H, I, ops.EPI_BIAS),
    "cross_ffn2_dgrad_gelu": (98304, "dgrad", I, H, ops.EPI_GELU_BWD),
    "cross_ffn1_dgrad": (98304, "dgrad", H, I, ops.EPI_BIAS),
    "cross_ffn1_wgrad": (98304, "wgrad", I, H, ops.EPI_ATOMIC),
    "cross_attn_dgrad_add": (98304, "dgrad", H, 3 * H, ops.EPI_ADD),
    "vocab_fwd": (1536, "fwd", V, H, ops.EPI_F32),
    "vocab_dgrad": (1536, "dgrad", H, V, ops.EPI_BIAS),
    "vocab_wgrad": (1536, "wgrad", V, H, ops.EPI_ATOMIC),
}


@pytest.mark.parametrize("name", list(PROD))
def test_gemm_production_shapes(name):
    """each GEMM as ops.py issues it (operand majors, padded vocab leading dimensions, automatic plan) once against
    fp64; the 98304-row outputs are checked on a row sample (every 61st row and the last 40)"""
    T, kind, N_, K_, epi = PROD[name]
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()))
    vocab = N_ == V or K_ == V
    if kind == "fwd":            # Y[T, N] = X[T, K] W[N, K]^T
        X, W = bf_randn((T, K_), 0.5, g), bf_randn((N_, K_), 0.05, g)
        A, B, As, Bs, a_mn, b_mn, M, N, K = X, W, X, W, 0, 0, T, N_, K_
    elif kind == "dgrad":        # dX[T, N] = dY[T, K] W[K, N]: W MN-major; dY of the vocab padded to 30528 columns
        dY, W = bf_randn((T, K_), 0.5, g), bf_randn((K_, N_), 0.05, g)
        As = store(dY, 0, 64) if vocab else dY
        A, B, Bs, a_mn, b_mn, M, N, K = dY, W.t(), W, 0, 1, T, N_, K_
    else:                        # dW[N, K] = dY[T, N]^T X[T, K]: both MN-major, contraction over the T rows
        dY, X = bf_randn((T, N_), 0.5, g), bf_randn((T, K_), 0.5, g)
        As = store(dY.t(), 1, 64) if vocab else dY
        A, B, Bs, a_mn, b_mn, M, N, K = dY.t(), X.t(), X, 1, 1, N_, K_, T
    sample = None
    if M > 4096:
        sample = torch.cat([torch.arange(0, M - 40, 61, device=DEV), torch.arange(M - 40, M, device=DEV)])
    f32 = epi in OUT_F32
    ldo = LDV if N == V else N
    out_full = torch.zeros(M, ldo, device=DEV, dtype=torch.float32 if f32 else BF16)
    out = out_full[:, :N]
    bias = torch.randn(N, device=DEV, generator=g) * 0.1 if epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_F32) else None
    aux_in = bf_randn((M, N), 1.0, g) if epi in (ops.EPI_ADD, ops.EPI_GELU_BWD) else None
    aux_out = torch.empty(M, N, device=DEV, dtype=BF16) if epi == ops.EPI_GELU else None
    if epi == ops.EPI_ATOMIC:
        out.normal_(generator=g)
    out0 = out.clone() if epi == ops.EPI_ATOMIC else None
    ops.gemm(As, Bs, M, N, K, out, epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, a_mn=a_mn, b_mn=b_mn)
    torch.cuda.synchronize()
    if sample is not None:
        A = A[sample]
        out = out[sample]
        aux_in = aux_in[sample] if aux_in is not None else None
        aux_out = aux_out[sample] if aux_out is not None else None
        out0 = out0[sample] if out0 is not None else None
    acc, mag = mm64(A, B)
    b64 = bias.double() if bias is not None else 0.0
    if epi in (ops.EPI_BIAS, ops.EPI_F32):
        ref = acc + b64
        within(out, ref, elem_bound(mag, K, b64.abs(), None if f32 else ref), name)
    elif epi == ops.EPI_GELU:
        pre = acc + b64
        bpre = elem_bound(mag, K, b64.abs())
        within(aux_out, pre, bpre + BF16_ROUND * pre.abs(), name + " aux_out")
        ref = gelu64(pre)
        within(out, ref, GELU_LIP * bpre + GELU_ABS * pre.abs() + BF16_ROUND * ref.abs(), name)
    elif epi == ops.EPI_GELU_BWD:
        gd = gelu_grad64(aux_in.double())
        ref = acc * gd
        within(out, ref, (C_ACC * K * U + EPI_ROUND) * mag * gd.abs() + GELU_ABS * mag + BF16_ROUND * ref.abs(), name)
    elif epi == ops.EPI_ADD:
        ref = acc + aux_in.double()
        within(out, ref, elem_bound(mag, K, aux_in.double().abs(), ref), name)
    else:
        ref = out0.double() + acc
        within(out, ref, elem_bound(mag, K, out0.double().abs()), name)
    if ldo > N:
        assert bool((out_full[:, N:] == 0).all()), name + ": padding columns written"


# ---------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------
def test_gemm_argument_errors_raise():
    g = torch.Generator(device=DEV).manual_seed(9)
    M, N, K = 128, 128, 128
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.5, g)
    out = torch.empty(M, N, device=DEV, dtype=BF16)
    f32 = torch.zeros(M, N, device=DEV)
    aux = torch.empty(M, N, device=DEV, dtype=BF16)
    bad = [
        lambda: ops.gemm(A, B, M, N, K, out, block_n=96),                          # not a tile width
        lambda: ops.gemm(A, B, M, N, K, out, block_n=32),
        lambda: ops.gemm(A, B, M, N, K, out, epi=ops.EPI_BIAS, split_k=2),           # split-K needs the atomic epilogue
        lambda: ops.gemm(A, B, M, N, K, f32, epi=ops.EPI_F32, split_k=3),
        lambda: ops.gemm(torch.empty(M, 100, device=DEV, dtype=BF16), B, M, N, 100, out),   # lda % 8 != 0
        lambda: ops.gemm(torch.empty(M * K + 1, device=DEV, dtype=BF16)[1:].view(M, K), B, M, N, K, out),  # misaligned
        lambda: ops.gemm(A, B, M, N, K, out, epi=ops.EPI_ADD),                       # missing aux_in
        lambda: ops.gemm(A, B, M, N, K, out, epi=ops.EPI_GELU_BWD),
        lambda: ops.gemm(A, B, M, N, K, out, epi=ops.EPI_GELU),                      # missing aux_out
        lambda: ops.gemm(A, B, M, N, K, f32, epi=ops.EPI_ATOMIC, split_k=-1),
        lambda: ops.gemm(A, B, M, N, K, out, epi=6),
    ]
    for fn in bad:
        with pytest.raises(RuntimeError):
            fn()
    ops.gemm(A, B, M, N, K, out, aux_out=aux)          # the checks leave the library usable
    torch.cuda.synchronize()
