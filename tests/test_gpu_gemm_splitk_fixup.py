"""GPU: the in-kernel split-K fix-up of the fp32 weight-gradient GEMM (csrc/gemm_wgmma.cu, EPI_ATOMIC_F32 with more
than one split).

Every work item stores its split's partial tile, and the tile's last arriver adds all of them in split order and then
into the output.  So the result is fixed by the plan alone: it must equal, bit for bit, one split_k = 1 GEMM per K
slice into zeroed fp32 outputs, summed in split order by torch and added to the output.  Below K = 4096 the automatic
plan runs unsplit and sums the same k-segments in registers, which must give the same bits.  The small-K weight
gradients of the text and visual layers (1536 rows) and of the first-token cross layer (1024 rows) are checked under
their automatic plan against their split plan's bits and fp64, and for the same bits across launches, reserved SMs,
CUDA-graph replay and a second weight gradient running concurrently on another stream."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.gemm_check import DEV, bf_randn, elem_bound, mm64, within  # noqa: E402
from univl_b200 import ops  # noqa: E402
from univl_b200 import runtime as rt  # noqa: E402

BK = 64  # k-block width of the GEMM


def _k_slices(K, split_k):
    """the K ranges of the plan's splits: ceil(k-blocks / split_k) k-blocks each, the last one shorter"""
    kb = -(-K // BK)
    per = -(-kb // min(split_k, kb))
    return [(k0 * BK, min(K, (k0 + per) * BK)) for k0 in range(0, kb, per)]


def _wgrad(dY, X, out, **kw):
    """out[M, N] += alpha dY[K, M]^T X[K, N] as linear_wgrad issues it (both operands MN-major)"""
    K, M = dY.shape
    ops.gemm(dY, X, M, X.shape[1], K, out, epi=ops.EPI_ATOMIC, a_mn=1, b_mn=1, **kw)
    return out


@pytest.mark.parametrize("M,N,K,block_n", [(296, 200, 1416, 64), (296, 200, 1416, 256), (768, 768, 1416, 0)])
@pytest.mark.parametrize("split_k", [2, 3, 5, 12])
def test_forced_splits_match_split_order_reconstruction(M, N, K, block_n, split_k):
    """K = 1416 is 23 k-blocks, the last 8 wide: 2 -> 12 + 11, 3 -> 8 + 8 + 7, 5 -> 5 + 5 + 5 + 5 + 3, 12 -> 11 x 2
    + 1 (an uneven last split every time), added at alpha 0.5 into a non-zero output with a padded leading
    dimension"""
    g = torch.Generator(device=DEV).manual_seed(7000 + M + block_n + split_k)
    dY, X = bf_randn((K, M), 0.5, g), bf_randn((K, N), 0.5, g)
    out0 = torch.randn(M, N, device=DEV, generator=g)
    buf = torch.empty(M, N + 12, device=DEV)
    out = buf[:, :N]
    out.copy_(out0)
    _wgrad(dY, X, out, alpha=0.5, block_n=block_n, split_k=split_k)
    t = torch.zeros(M, N, device=DEV)
    for k0, k1 in _k_slices(K, split_k):
        part = _wgrad(dY[k0:k1], X[k0:k1], torch.zeros(M, N, device=DEV), alpha=0.5, block_n=block_n, split_k=1)
        t = t + part
    torch.cuda.synchronize()
    assert torch.equal(out, out0 + t)


@pytest.mark.parametrize("M,N", [(296, 200), (768, 768)])
def test_in_register_segments_match_split_order_reconstruction(M, N):
    """the automatic plan below K = 4096 sums its split plan's k-segments in registers: at K = 1416 that plan has 11
    splits of 3 k-blocks, hence 8 segments (7 x 3 + 2), added at alpha 0.5 into a non-zero strided output, with edge
    tiles in the 296 x 200 case"""
    g = torch.Generator(device=DEV).manual_seed(7200 + M)
    K = 1416
    dY, X = bf_randn((K, M), 0.5, g), bf_randn((K, N), 0.5, g)
    out0 = torch.randn(M, N, device=DEV, generator=g)
    out = torch.empty(M, N + 12, device=DEV)[:, :N]
    out.copy_(out0)
    _wgrad(dY, X, out, alpha=0.5)
    splits = _split_plan(M, N, K)
    t = torch.zeros(M, N, device=DEV)
    for k0, k1 in _k_slices(K, splits):
        t = t + _wgrad(dY[k0:k1], X[k0:k1], torch.zeros(M, N, device=DEV), alpha=0.5, split_k=1)
    torch.cuda.synchronize()
    assert len(_k_slices(K, splits)) > 1
    assert torch.equal(out, out0 + t)


def test_cross_shape_matches_split_order_reconstruction():
    """a 98304-row cross-encoder weight gradient (attention output, 768 x 768) split 5 ways: 308 x 4 + 304 k-blocks"""
    g = torch.Generator(device=DEV).manual_seed(7100)
    M, N, K = 768, 768, 98304
    dY, X = bf_randn((K, M), 0.5, g), bf_randn((K, N), 0.5, g)
    out0 = torch.randn(M, N, device=DEV, generator=g)
    out = _wgrad(dY, X, out0.clone(), split_k=5)
    t = torch.zeros(M, N, device=DEV)
    for k0, k1 in _k_slices(K, 5):
        t = t + _wgrad(dY[k0:k1], X[k0:k1], torch.zeros(M, N, device=DEV), split_k=1)
    torch.cuda.synchronize()
    assert torch.equal(out, out0 + t)


H, I = 768, 3072
# name: (M, N, K) of dW[M, N] += dY[K, M]^T X[K, N]: the text / visual layers run 1536 rows, the first-token cross
# layer (one query row per pair, 32 x 32 pairs) 1024
SMALL_K = {
    "text_qkv_wgrad": (3 * H, H, 1536),
    "text_attn_out_wgrad": (H, H, 1536),
    "text_ffn1_wgrad": (I, H, 1536),
    "text_ffn2_wgrad": (H, I, 1536),
    "visual_in_wgrad": (H, 1024, 1536),
    "first_token_q_wgrad": (H, H, 1024),
    "first_token_ffn1_wgrad": (I, H, 1024),
    "first_token_ffn2_wgrad": (H, I, 1024),
}


def _problem(name):
    M, N, K = SMALL_K[name]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    dY, X = bf_randn((K, M), 0.5, g), bf_randn((K, N), 0.5, g)
    return dY, X, torch.randn(M, N, device=DEV, generator=g)


def _split_plan(M, N, K):
    """the split count of the automatic fp32 split-K plan: 2 x 132 work items of the 256-wide tile (narrower for
    N <= 128), at least 2 k-blocks per split"""
    bn = 64 if N <= 64 else 128 if N <= 128 else 256
    tiles = -(-M // 128) * -(-N // bn)
    kb = -(-K // BK)
    return max(1, min(-(-264 // tiles), kb // 2))


@pytest.mark.parametrize("name", list(SMALL_K))
def test_small_k_plans_exact_and_repeatable(name):
    """the automatic plan (unsplit, 64 wide, its split plan's k-segments summed in registers): the bits of that split
    plan forced through the split-K fix-up, within the fp64 bound, and the same bits on a second launch and with 40
    SMs reserved"""
    dY, X, out0 = _problem(name)
    K, M = dY.shape

    def run(**kw):
        out = _wgrad(dY, X, out0.clone(), **kw)
        torch.cuda.synchronize()
        return out
    base = run()
    splits = _split_plan(M, X.shape[1], K)
    assert splits > 1, name
    assert torch.equal(run(split_k=splits), base), "split_k %d" % splits
    acc, mag = mm64(dY.t(), X.t())
    within(base, out0.double() + acc, elem_bound(mag, K, out0.double().abs()), name)
    assert torch.equal(run(), base)
    try:
        rt.reserve_sms(40)
        assert torch.equal(run(), base), "40 SMs reserved"
    finally:
        rt.reserve_sms(0)


@pytest.mark.parametrize("name", ["text_attn_out_wgrad", "text_ffn2_wgrad", "first_token_q_wgrad"])
def test_small_k_plans_graph_replay(name):
    """captured once, replayed twice: the same bits as an eager launch each time"""
    dY, X, out0 = _problem(name)
    base = _wgrad(dY, X, out0.clone())
    out = out0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm up on a side stream before capture
        _wgrad(dY, X, out)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _wgrad(dY, X, out)
    for i in range(2):
        out.copy_(out0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, base), "replay %d" % i


def test_small_k_plans_concurrent_streams():
    """two different weight gradients launched together on two streams, several times over, give their own bits"""
    names = ["text_qkv_wgrad", "text_attn_out_wgrad"]
    probs = [_problem(n) for n in names]
    bases = [_wgrad(dY, X, out0.clone()) for dY, X, out0 in probs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rep in range(3):
        outs = [out0.clone() for _, _, out0 in probs]
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
        for s, (dY, X, _), out in zip(streams, probs, outs):
            with torch.cuda.stream(s):
                _wgrad(dY, X, out)
        for s in streams:
            torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for n, out, base in zip(names, outs, bases):
            assert torch.equal(out, base), "%s, repetition %d" % (n, rep)
