"""GPU: the two epilogue paths of the wgmma GEMM (csrc/gemm_wgmma.cu).

Tiles that lie wholly inside the output, with 2-element vector access, run the unchecked chunked epilogue (epi_tile);
edge tiles and outputs without vector access run the checked per-pair epilogue (epi_pair).  Both must compute the
same bits.  The other epilogues' scalar-path tests are in test_gpu_gemm.py; the GELU backward's is here."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.gemm_check import (BF16, BF16_ROUND, C_ACC, DEV, EPI_ROUND, GELU_ABS, OUT_F32, U,  # noqa: E402
                              bf_randn, gelu_grad64, mm64, within)
from univl_b200 import ops  # noqa: E402


@pytest.mark.parametrize("layout", ["odd_n", "odd_ld", "offset"])
def test_gemm_gelu_bwd_scalar_epilogue_path(layout):
    """the GELU backward epilogue (out = acc * gelu'(aux_in)) on outputs that cannot take 2-element vector stores (odd
    N with an unpadded output, odd ldo, a base one element off alignment) runs the scalar epilogue: fp64-exact within
    the bound, and bit-identical to the vector path on the same accumulators and the same aux_in"""
    g = torch.Generator(device=DEV).manual_seed(40 + ops.EPI_GELU_BWD)
    M, N, K = 200, (201 if layout == "odd_n" else 200), 136
    A, B = bf_randn((M, K), 0.3, g), bf_randn((N, K), 0.1, g)
    aux_in = bf_randn((M, N + N % 2), 1.0, g)[:, :N]       # even leading dimension: vector-capable

    def run(out):
        ops.gemm(A, B, M, N, K, out, epi=ops.EPI_GELU_BWD, aux_in=aux_in, split_k=1)
        return out

    vec = run(torch.empty(M, N + 1 if N % 2 else N + 2, dtype=BF16, device=DEV)[:, :N])
    if layout == "odd_n":
        sout = torch.empty(M, N, dtype=BF16, device=DEV)
    elif layout == "odd_ld":
        sout = torch.empty(M, N + 1, dtype=BF16, device=DEV)[:, :N]
    else:
        sout = torch.empty(M * (N + 2) + 1, dtype=BF16, device=DEV)[1:].view(M, N + 2)[:, :N]
    sc = run(sout)
    torch.cuda.synchronize()
    assert torch.equal(sc, vec), layout
    acc, mag = mm64(A, B)
    gd = gelu_grad64(aux_in.double())
    ref = acc * gd
    within(sc, ref, (C_ACC * K * U + EPI_ROUND) * mag * gd.abs() + GELU_ABS * mag + BF16_ROUND * ref.abs(),
           "scalar %s gelu_bwd" % layout)


UNCHECKED = [  # (epilogue, bias, split_k)
    (ops.EPI_BIAS, True, 1), (ops.EPI_BIAS, False, 1), (ops.EPI_GELU, True, 1), (ops.EPI_GELU, False, 1),
    (ops.EPI_GELU_BWD, False, 1), (ops.EPI_ADD, False, 1), (ops.EPI_F32, True, 1), (ops.EPI_F32, False, 1),
    (ops.EPI_ATOMIC, False, 1), (ops.EPI_ATOMIC, False, 0),   # 0: the automatic plan, 2 splits into partial sums
]


@pytest.mark.parametrize("block_n", [64, 128, 256])
@pytest.mark.parametrize("epi,with_bias,split_k", UNCHECKED)
def test_gemm_unchecked_epilogue_matches_checked(epi, with_bias, split_k, block_n):
    """with M = 384 every tile is interior and runs the unchecked epilogue; with M = 383 the last m-tile is an edge
    tile and runs the checked one.  Rows [0, 383) — the accumulators are the same — must be bit-identical, aux_out
    included, with alpha 1 and 0.75"""
    g = torch.Generator(device=DEV).manual_seed(60 + 7 * epi + block_n + split_k + int(with_bias))
    M, N, K = 384, 2 * block_n, 200
    A, B = bf_randn((M, K), 0.3, g), bf_randn((N, K), 0.1, g)
    dt = torch.float32 if epi in OUT_F32 else BF16
    bias = torch.randn(N, device=DEV, generator=g) if with_bias else None
    aux_in = bf_randn((M, N), 1.0, g) if epi in (ops.EPI_ADD, ops.EPI_GELU_BWD) else None
    init = torch.randn(M, N, device=DEV, generator=g).to(dt)
    for alpha in (1.0, 0.75):
        res = []
        for m in (M, M - 1):
            out = init[:m].clone()
            aux_out = torch.empty(m, N, dtype=BF16, device=DEV) if epi == ops.EPI_GELU else None
            ops.gemm(A[:m], B, m, N, K, out, epi=epi, bias=bias, aux_in=aux_in[:m] if aux_in is not None else None,
                     aux_out=aux_out, alpha=alpha, block_n=block_n, split_k=split_k)
            res.append((out, aux_out))
        torch.cuda.synchronize()
        (full, full_aux), (edge, edge_aux) = res
        assert torch.equal(full[:M - 1], edge), alpha
        if epi == ops.EPI_GELU:
            assert torch.equal(full_aux[:M - 1], edge_aux), alpha
