"""GPU: the ordered reduction behind every deterministic cross-block sum (univl_partials_reduce, csrc/api.cu).

Each element's partial rows are added in row order (t = 0; t += row k), then t is added into dst.  The result is
checked bit for bit against that sum written in fp32 PyTorch, and within its fp64 bound, at the shapes of the
FT-Align step and at edge shapes; and for the same bits on repeated launches, with SMs reserved and under CUDA-graph
replay."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from univl_b200 import runtime as rt  # noqa: E402

DEV = "cuda"
U32 = 2.0 ** -24


def _reduce(part, dst):
    """dst[r, :cols] += row-order sum over k of part[k, r, :] (part [nparts, rows, cols], dst [rows, ld])"""
    nparts, rows, cols = part.shape
    rt.call("univl_partials_reduce", part.data_ptr(), nparts, rows, cols, dst.data_ptr(), dst.stride(0))
    return dst


def _row_order_fp32(part):
    """t = 0; t += part[k] for k ascending, in fp32: [nparts, n] -> [n]"""
    t = torch.zeros(part.shape[1], device=part.device, dtype=torch.float32)
    for k in range(part.shape[0]):
        t = t + part[k]
    return t


def _same_bits(run, launches=3):
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


# (nparts, rows, cols, ld): the step's reductions (fused attention bias rows of the all-pairs cross layer, LayerNorm
# parameter rows over 98304 tokens, FFN bias column sums), then edge shapes: one part, nparts not a multiple of the
# 256-row stage (and of the 8 loading warps), exactly one stage, cols not a multiple of 32, rows > 1 with ld != cols
SHAPES = [(8192, 1, 2304, 2304), (660, 1, 768, 768), (192, 1, 768, 768), (44, 1, 3072, 3072),
          (1, 1, 768, 768), (33, 1, 771, 771), (256, 1, 300, 300), (1057, 1, 300, 300), (70, 3, 130, 136),
          (5, 4, 7, 9)]


@pytest.mark.parametrize("nparts,rows,cols,ld", SHAPES)
def test_partials_reduce_row_order_bits_and_fp64(nparts, rows, cols, ld):
    g = torch.Generator(device=DEV).manual_seed(nparts * 7 + cols)
    part = torch.randn(nparts, rows, cols, device=DEV, generator=g)
    dst0 = torch.randn(rows, ld, device=DEV, generator=g)
    keep = part.clone()
    got = _reduce(part, dst0.clone())
    torch.cuda.synchronize()
    assert torch.equal(part, keep), "the caller's partial rows were modified"
    # bit for bit: the row-order sum in fp32, then one add into dst
    want = dst0.clone()
    want[:, :cols] = dst0[:, :cols] + _row_order_fp32(part.reshape(nparts, rows * cols)).view(rows, cols)
    assert torch.equal(got, want)
    assert torch.equal(got[:, cols:], dst0[:, cols:]), "columns past cols were written"
    # within the fp64 bound of nparts + 1 ordered fp32 additions
    pd = part.double()
    ref = dst0.double()[:, :cols] + pd.sum(0)
    bound = (nparts + 1) * U32 * (pd.abs().sum(0) + dst0.double()[:, :cols].abs())
    assert bool(((got.double()[:, :cols] - ref).abs() <= bound).all())


@pytest.mark.parametrize("nparts,cols", [(8192, 2304), (660, 768), (33, 771)])
def test_partials_reduce_repeatable_reserved_sms_and_graph(nparts, cols):
    g = torch.Generator(device=DEV).manual_seed(nparts)
    part = torch.randn(nparts, 1, cols, device=DEV, generator=g)
    dst0 = torch.randn(1, cols, device=DEV, generator=g)

    def run():
        return [_reduce(part, dst0.clone())]
    base = _same_bits(run)[0]
    out = dst0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        _reduce(part, out)
    for _ in range(2):
        out.copy_(dst0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, base), "graph replay differs from the eager launch"


def test_partials_reduce_rejects_bad_arguments():
    part = torch.zeros(2, 1, 8, device=DEV)
    dst = torch.zeros(1, 8, device=DEV)
    with pytest.raises(RuntimeError, match="partials_reduce"):
        rt.call("univl_partials_reduce", part.data_ptr(), 2, 1, 8, dst.data_ptr(), 4)
    with pytest.raises(RuntimeError, match="partials_reduce"):
        rt.call("univl_partials_reduce", part.data_ptr(), -1, 1, 8, dst.data_ptr(), 8)
