"""GPU: the ping-pong schedule of the wgmma GEMM (csrc/gemm_wgmma.cu, tile widths 64 and 128: each consumer warpgroup
owns whole tiles and the two alternate) against the cooperative schedule of the 256-wide tile, bit for bit, and against
fp64 (tests/gemm_check.py) where a CTA walks many tiles.

Both schedules give every output element the same chain of k16 wgmmas in the same k order and the same epilogue, so
any difference in the bits is a schedule bug: a tile taken by both warpgroups or by neither, a ring slot read before
its load landed or after it was refilled, an accumulator half paired with the wrong rows.  The 16-byte stores of the
bf16 outputs are held to the bits of the 4-byte stores in the same way."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.gemm_check import BF16, DEV, bf_randn, run_epi, store  # noqa: E402
from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402

EPIS = [ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_GELU_BWD, ops.EPI_ADD, ops.EPI_F32, ops.EPI_ATOMIC]
MAJORS = [(a_mn, b_mn) for a_mn in (0, 1) for b_mn in (0, 1)]


def _inputs(M, N, K, epi, g):
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.1, g)
    bias = torch.randn(N, device=DEV, generator=g) if epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_F32) else None
    aux_in = bf_randn((M, N), 1.0, g) if epi in (ops.EPI_GELU_BWD, ops.EPI_ADD) else None
    init = torch.randn(M, N, device=DEV, generator=g) if epi == ops.EPI_ATOMIC else None
    return A, B, bias, aux_in, init


def _run(As, Bs, M, N, K, epi, a_mn, b_mn, block_n, bias=None, aux_in=None, init=None, alpha=1.0, split_k=0):
    """the outputs of one launch (out, and aux_out for the GELU forward), synchronised"""
    f32 = epi in (ops.EPI_F32, ops.EPI_ATOMIC)
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.float32 if f32 else BF16)
    if init is not None:
        out.copy_(init)
    aux_out = torch.full((M, N), float("nan"), device=DEV, dtype=BF16) if epi == ops.EPI_GELU else None
    ops.gemm(As, Bs, M, N, K, out, epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, a_mn=a_mn, b_mn=b_mn,
             alpha=alpha, block_n=block_n, split_k=split_k)
    torch.cuda.synchronize()
    return [out] if aux_out is None else [out, aux_out]


def _same(got, ref, what):
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), "%s (output %d): %d elements differ" % (what, i, int((a != b).sum()))


# (M, N, K): 8192 rows, and 33 x 1472 tiles, where on 132 SMs a CTA walks 3 items of 128 columns (the last column tile
# an edge tile) or 5 / 6 of 64 — an odd count leaves one warpgroup with one item more than the other
SHAPES = [(8192, 768, 768), (4224, 1472, 768)]


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("epi", EPIS)
def test_pingpong_matches_cooperative_bitwise(epi, a_mn, b_mn):
    """block_n 128 and 64 (ping-pong) give the bits of block_n 256 (cooperative) for every epilogue, with and without
    bias and at alpha 1 and 0.75, in all four operand majors; and the same bits with 40 SMs reserved (fewer CTAs, more
    items each).  The fp32 accumulation runs at split_k 1 and at split_k 3 over 19 k-blocks (7 + 7 + 5: an uneven last
    split, so the items a warpgroup skips have different k-block counts)."""
    g = torch.Generator(device=DEV).manual_seed(300 + 4 * epi + 2 * a_mn + b_mn)
    for M, N, K in SHAPES:
        splits = [0]
        if epi == ops.EPI_ATOMIC:
            K, splits = 1216, [1, 3]
        A, B, bias, aux_in, init = _inputs(M, N, K, epi, g)
        As, Bs = store(A, a_mn, 8), store(B, b_mn, 8)
        for split_k in splits:
            for with_bias in ((True, False) if bias is not None else (False,)):
                for alpha in (1.0, 0.75):
                    args = dict(bias=bias if with_bias else None, aux_in=aux_in, init=init, alpha=alpha,
                                split_k=split_k)
                    what = "M %d N %d K %d epi %d a_mn %d b_mn %d split_k %d bias %d alpha %g" % (
                        M, N, K, epi, a_mn, b_mn, split_k, with_bias, alpha)
                    ref = _run(As, Bs, M, N, K, epi, a_mn, b_mn, 256, **args)
                    for bn in (128, 64):
                        _same(_run(As, Bs, M, N, K, epi, a_mn, b_mn, bn, **args), ref, what + " bn %d" % bn)
                    try:
                        rt.reserve_sms(40)
                        _same(_run(As, Bs, M, N, K, epi, a_mn, b_mn, 128, **args), ref, what + " bn 128, 40 SMs "
                              "reserved")
                    finally:
                        rt.reserve_sms(0)


@pytest.mark.parametrize("epi", [ops.EPI_GELU, ops.EPI_ATOMIC])
def test_pingpong_fewer_items_than_sms(epi):
    """a launch with fewer work items than SMs: every CTA has one item and its second warpgroup never runs an MMA —
    within the fp64 bound and the cooperative bits (the fp32 accumulation split 2 ways: 8 items of 128 columns)"""
    g = torch.Generator(device=DEV).manual_seed(400 + epi)
    M, N, K = 256, 256, 776
    A, B, bias, aux_in, init = _inputs(M, N, K, epi, g)
    split_k = 2 if epi == ops.EPI_ATOMIC else 0
    for bn in (128, 64):
        run_epi(epi, A, B, A, B, 0, 0, block_n=bn, split_k=split_k, g=g, what="one item per CTA bn %d" % bn)
        args = dict(bias=bias, aux_in=aux_in, init=init, split_k=split_k)
        _same(_run(A, B, M, N, K, epi, 0, 0, bn, **args), _run(A, B, M, N, K, epi, 0, 0, 256, **args),
              "one item per CTA bn %d" % bn)


@pytest.mark.parametrize("block_n", [128, 64])
@pytest.mark.parametrize("epi", [ops.EPI_GELU, ops.EPI_ADD, ops.EPI_F32])
def test_pingpong_many_items_per_cta(epi, block_n):
    """8269 x 3072 x 776: 65 x 24 (bn 128) or 65 x 48 (bn 64) items, about 12 or 24 per CTA, 13 k-blocks each, so each
    warpgroup's ring position wraps the 6- or 8-stage ring many times over the other's k-blocks; the last row tile is
    partial (77 rows) and K ends in an 8-wide tail.  Checked against fp64 per element."""
    g = torch.Generator(device=DEV).manual_seed(500 + 2 * epi + block_n)
    M, N, K = 8269, 3072, 776
    A, B = bf_randn((M, K), 0.5, g), bf_randn((N, K), 0.1, g)
    run_epi(epi, A, B, A, B, 0, 0, block_n=block_n, g=g, what="many items epi %d bn %d" % (epi, block_n))


def test_pingpong_repeatable_and_graph_replay():
    """one ping-pong instance (bn 128, bias + GELU, the FFN up-projection's epilogue) gives the same bits on a second
    launch and when replayed from a captured CUDA graph"""
    g = torch.Generator(device=DEV).manual_seed(600)
    M, N, K = 8192, 3072, 768
    A, B, bias, _, _ = _inputs(M, N, K, ops.EPI_GELU, g)
    first = _run(A, B, M, N, K, ops.EPI_GELU, 0, 0, 128, bias=bias)
    _same(_run(A, B, M, N, K, ops.EPI_GELU, 0, 0, 128, bias=bias), first, "second launch")
    out, aux_out = torch.empty_like(first[0]), torch.empty_like(first[1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm up on a side stream before capture
        ops.gemm(A, B, M, N, K, out, epi=ops.EPI_GELU, bias=bias, aux_out=aux_out, block_n=128)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm(A, B, M, N, K, out, epi=ops.EPI_GELU, bias=bias, aux_out=aux_out, block_n=128)
    for _ in range(2):
        out.fill_(float("nan"))
        aux_out.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _same([out, aux_out], first, "graph replay")


@pytest.mark.parametrize("block_n", [256, 128])
@pytest.mark.parametrize("epi", [ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_GELU_BWD, ops.EPI_ADD])
def test_wide_stores_match_four_byte_stores(epi, block_n):
    """bf16 outputs with a 16-byte aligned base and a leading dimension that is a multiple of 8 take the 16-byte
    stores of whole 8-column groups (a quad transpose); an output whose leading dimension is 2 mod 8 takes the 4-byte
    stores.  Both give the same bits, and neither writes outside the output."""
    g = torch.Generator(device=DEV).manual_seed(700 + epi + block_n)
    M, N, K = 1024, 768, 776
    A, B, bias, aux_in, _ = _inputs(M, N, K, epi, g)
    outs = []
    for ld in (N, N + 2):
        buf = torch.full((M, ld), -77.0, device=DEV, dtype=BF16)
        abuf = torch.full((M, ld), -77.0, device=DEV, dtype=BF16)
        aux_out = abuf[:, :N] if epi == ops.EPI_GELU else None
        ops.gemm(A, B, M, N, K, buf[:, :N], epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, block_n=block_n)
        torch.cuda.synchronize()
        assert bool((buf[:, N:] == -77.0).all()) and bool((abuf[:, N:] == -77.0).all()), ld
        outs.append([buf[:, :N]] + ([aux_out] if aux_out is not None else []))
    _same(outs[0], outs[1], "16-byte vs 4-byte stores epi %d bn %d" % (epi, block_n))
