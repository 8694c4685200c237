"""GPU: the beam top-k over the vocabulary without logits (univl_vocab_beam_topk, csrc/gemm_wgmma.cu).

Exact checks: the logits of `cls.logits` (ops.gemm, EPI_F32 with the bias), the kernel's own lse, and in torch fp32
key = (logit - lse) + score, sorted by key descending then flat index k V + c ascending (a stable sort of the flat
row-major keys).  The kernel's (key, index) lists must equal that bit for bit; every selected key having the bits of
that fp32 formula also pins the kernel's recomputed logits to the GEMM's bits.

fp64 bounds (U = 2^-24; C_ACC, EPI_ROUND, MUFU and the lse bound B_lse as tests/test_gpu_vocab_xent.py writes them):
  logit  eL = C_ACC K U |x||W|^T + EPI_ROUND (|x||W|^T + |bias|)
  key    eL[c] + B_lse + U |logit - lse| + U |key|: the logit and lse errors, then the subtraction's and the addition's
         roundings.
The selected set must equal the fp64 top n_beam of every instance whose fp64 gap between its n_beam-th and next key
exceeds twice the largest key bound (elsewhere a rounding may legitimately swap the boundary candidates)."""
import pytest
import torch

from tests.gemm_check import C_ACC, EPI_ROUND, U, within
from tests.test_cpu_vocab_xent_args import vx_chunks
from tests.test_gpu_vocab_xent import MUFU
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
K = 768


def _inputs(n_inst, n_beam, V, seed, live=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = n_inst * n_beam
    x = torch.randn(R, K, device=DEV, generator=g).to(BF16)
    w16 = (0.05 * torch.randn(V, K, device=DEV, generator=g)).to(BF16)
    bias = torch.randn(V, device=DEV, generator=g)
    score = -3.0 * torch.rand(R, device=DEV, generator=g)
    if live is None:
        live = torch.randint(1, n_beam + 1, (n_inst,), device=DEV, generator=g)
    live = torch.as_tensor(live, device=DEV).to(torch.int32).expand(n_inst).contiguous()
    return x, w16, bias, score, live


def _logits(x, w16, bias):
    """what cls.logits computes: the fp32 GEMM with the bias in its epilogue"""
    R, V = x.shape[0], w16.shape[0]
    out = torch.empty((R, ops._ld_pad(V)), dtype=torch.float32, device=DEV)[:, :V]
    return ops.gemm(x, w16, R, V, K, out, epi=ops.EPI_F32, bias=bias)


def _reference(logits, lse, score, live, n_beam):
    """(key, index) [n_inst, n_beam] by key descending, then flat index ascending"""
    R, V = logits.shape
    n_inst = R // n_beam
    keys = (logits - lse[:, None]) + score[:, None]
    keys = keys.view(n_inst, n_beam * V)
    rows = torch.arange(n_beam * V, device=DEV) // V
    keys = torch.where(rows[None] < live[:, None].long(), keys, torch.full_like(keys, -float("inf")))
    k, i = torch.sort(keys, dim=1, descending=True, stable=True)
    return k[:, :n_beam], i[:, :n_beam].to(torch.int32)


def _check_exact(n_inst, n_beam, V, seed, live=None):
    x, w16, bias, score, live = _inputs(n_inst, n_beam, V, seed, live)
    lse, key, index = ops.vocab_beam_topk(x, w16, bias, score, live, n_beam)
    want_k, want_i = _reference(_logits(x, w16, bias), lse, score, live, n_beam)
    assert torch.equal(index, want_i), (index, want_i)
    assert torch.equal(key.view(torch.int32), want_k.view(torch.int32))
    return x, w16, bias, score, live, lse, key, index


@pytest.mark.parametrize("n_beam", range(1, 9))
def test_exact_every_beam_width(n_beam):
    _check_exact(13, n_beam, 30522, seed=n_beam)


@pytest.mark.parametrize("n_inst,n_beam,V", [(64, 5, 30522), (21, 6, 1000), (3, 8, 30522), (50, 3, 257)])
def test_exact_shapes(n_inst, n_beam, V):
    # R = 320 (the MSRVTT batch of 64 x 5), R not a multiple of 128, V not a multiple of 128
    _check_exact(n_inst, n_beam, V, seed=n_inst + V)


@pytest.mark.parametrize("n_beam", [1, 5, 8])
def test_first_step_reads_row_zero_only(n_beam):
    """one live hypothesis per instance (the first step): every pick is a word of row 0, flat index < V"""
    V = 30522
    *_, index = _check_exact(9, n_beam, V, seed=40 + n_beam, live=1)
    assert bool((index < V).all())


def test_ties_take_the_lower_flat_index():
    n_inst, n_beam, V = 4, 5, 1000
    x, w16, bias, score, live = _inputs(n_inst, n_beam, V, seed=77, live=n_beam)
    # word ties inside a row: columns 2c + 1 copy column 2c (weights and bias) for the first 200 columns
    w16[1:400:2] = w16[0:400:2]
    bias[1:400:2] = bias[0:400:2]
    # beam ties: every row of an instance holds the same x and score
    x = x.view(n_inst, n_beam, K)[:, :1].expand(n_inst, n_beam, K).reshape(-1, K).contiguous()
    score = score.view(n_inst, n_beam)[:, :1].expand(n_inst, n_beam).reshape(-1).contiguous()
    # push the tied columns to the top
    bias[:400] += 20.0
    lse, key, index = ops.vocab_beam_topk(x, w16, bias, score, live, n_beam)
    want_k, want_i = _reference(_logits(x, w16, bias), lse, score, live, n_beam)
    assert torch.equal(index, want_i) and torch.equal(key, want_k)
    # every row of an instance ties with row 0, so the picks come from row 0 first; equal keys in ascending index
    for i in range(n_inst):
        ks, ix = key[i].tolist(), index[i].tolist()
        assert ix[0] < V
        for a in range(n_beam - 1):
            assert ks[a] > ks[a + 1] or (ks[a] == ks[a + 1] and ix[a] < ix[a + 1]), (ks, ix)
        assert any(ks[a] == ks[a + 1] for a in range(n_beam - 1)), "the case must contain a tie"


@pytest.mark.parametrize("n_inst,n_beam,V", [(64, 5, 30522), (7, 8, 1000)])
def test_against_fp64(n_inst, n_beam, V):
    x, w16, bias, score, live = _inputs(n_inst, n_beam, V, seed=5 + V, live=n_beam)
    lse, key, index = ops.vocab_beam_topk(x, w16, bias, score, live, n_beam)
    R = n_inst * n_beam
    x64, w64, b64 = x.double(), w16.double(), bias.double()
    l = x64 @ w64.t() + b64
    mag = x64.abs() @ w64.abs().t()
    eL = C_ACC * K * U * mag + EPI_ROUND * (mag + b64.abs())
    del mag
    lse64 = torch.logsumexp(l, 1)
    chunks, ct = vx_chunks(R, V)
    rng = l.max(1).values - l.min(1).values
    b_lse = eL.max(1).values + (33 * ct + 3 * chunks + 8) * U + 2 * MUFU + 2 * U * rng + 2 * U * lse64.abs()
    within(lse, lse64, b_lse, "beam lse R=%d V=%d" % (R, V))
    key64 = (l - lse64[:, None]) + score.double()[:, None]
    b_key = eL + b_lse[:, None] + U * (l - lse64[:, None]).abs() + U * key64.abs()
    flat64, flatb = key64.view(n_inst, n_beam * V), b_key.view(n_inst, n_beam * V)
    picked = index.long()
    within(key, flat64.gather(1, picked), flatb.gather(1, picked), "beam keys R=%d V=%d" % (R, V))
    top = torch.topk(flat64, n_beam + 1, dim=1)
    gap = top.values[:, n_beam - 1] - top.values[:, n_beam]
    clear = gap > 2 * flatb.max(1).values
    assert int(clear.sum()) >= n_inst // 2, "too few instances with a clear boundary to check the set"
    for i in torch.nonzero(clear).flatten().tolist():
        assert sorted(picked[i].tolist()) == sorted(top.indices[i, :n_beam].tolist()), i


def test_deterministic_repeat_reserved_streams_and_graph():
    n_inst, n_beam, V = 64, 5, 30522
    x, w16, bias, score, live = _inputs(n_inst, n_beam, V, seed=11)
    base = ops.vocab_beam_topk(x, w16, bias, score, live, n_beam)
    torch.cuda.synchronize()

    def same(out, what):
        for a, b in zip(base, out):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what

    same(ops.vocab_beam_topk(x, w16, bias, score, live, n_beam), "second launch")
    rt.reserve_sms(40)
    try:
        same(ops.vocab_beam_topk(x, w16, bias, score, live, n_beam), "40 SMs reserved")
    finally:
        rt.reserve_sms(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        other = ops.vocab_beam_topk(x, w16, bias, score, live, n_beam)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    same(other, "second stream")
    ws = ops.vocab_beam_topk_workspace(n_inst, n_beam, V, x)
    out = tuple(torch.empty_like(t) for t in base)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.vocab_beam_topk(x, w16, bias, score, live, n_beam, ws, out=out)
    for t in out:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    same(out, "graph replay")


def test_advance_bookkeeping():
    """univl_beam_advance against its statement on random picks: live and done instances, tables, tokens, ancestors"""
    n_inst, n_beam, V, max_words, t, eos = 5, 4, 1000, 6, 2, 102
    R = n_inst * n_beam
    g = torch.Generator(device=DEV).manual_seed(3)
    key = torch.randn(n_inst, n_beam, device=DEV, generator=g)
    index = torch.randint(0, n_beam * V, (n_inst, n_beam), device=DEV, generator=g).to(torch.int32)
    index[1, 0] = 2 * V + eos                         # instance 1 finishes now
    done = torch.tensor([0, 0, 1, 0, 0], dtype=torch.int32, device=DEV)    # instance 2 finished before
    score = torch.randn(R, device=DEV, generator=g)
    tables = torch.randint(0, 9, (2, max_words, n_inst, n_beam), device=DEV, generator=g).to(torch.int32)
    tokens = torch.randint(0, V, (R,), device=DEV, generator=g)
    anc_in = torch.randint(0, 1000, (R, max_words), device=DEV, generator=g).to(torch.int32)
    anc_out = torch.full((R, max_words), -5, dtype=torch.int32, device=DEV)
    before = [t_.clone() for t_ in (score, done, tables, tokens)]
    ops.beam_advance(key, index, V, t, eos, score, done, tables[0], tables[1], tokens, anc_in, anc_out)
    torch.cuda.synchronize()
    want_score, want_done, want_tables, want_tokens = [t_.clone() for t_ in before]
    want_anc = torch.full_like(anc_out, -5)
    for i in range(n_inst):
        frozen = bool(before[1][i])
        for j in range(n_beam):
            r = i * n_beam + j
            k = j
            if not frozen:
                flat = int(index[i, j])
                k, c = flat // V, flat % V
                want_score[r] = key[i, j]
                want_tables[0, t, i, j], want_tables[1, t, i, j] = k, c
                want_tokens[r] = c
            want_anc[r, :t + 1] = anc_in[i * n_beam + k, :t + 1]
            want_anc[r, t + 1] = (t + 1) * R + r
        if not frozen and int(index[i, 0]) % V == eos:
            want_done[i] = 1
    assert torch.equal(score, want_score)
    assert torch.equal(done, want_done) and done.tolist() == [0, 1, 1, 0, 0]
    assert torch.equal(tables, want_tables)
    assert torch.equal(tokens, want_tokens)
    assert torch.equal(anc_out, want_anc)
