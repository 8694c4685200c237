"""CPU: the packing and chunk planning of the gallery encoders (retrieval.RowPacking) against a Python loop, and the
argument checks of retrieval.embed_texts / embed_videos / topk."""
import types

import numpy as np
import pytest
import torch

from univl_b200 import lib
from univl_b200 import retrieval


def test_the_new_entries_are_declared():
    decl = lib.parse_header()
    for name in ("univl_embed_text_packed_fwd", "univl_embed_src_packed_fwd", "univl_layernorm_f32_rows_fwd",
                 "univl_meanpool_packed_fwd"):
        assert name in decl


def _mask(N, S, seed):
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand((N, S), generator=g) < 0.6).long()
    if N > 2:
        m[1] = 0  # an empty row
        m[2] = 1  # a full row
    return m


@pytest.mark.parametrize("budget", [1, 5, 7, 12, 1 << 20])
@pytest.mark.parametrize("N,S", [(9, 7), (1, 1), (0, 4), (6, 1)])
def test_chunks_and_packing_match_a_python_loop(budget, N, S):
    m = _mask(N, S, seed=N + S)
    rp = retrieval.RowPacking(m, budget)
    counts = [int(m[i].ne(0).sum()) for i in range(N)]
    assert rp.counts.tolist() == counts and rp.max_len == max(counts, default=0)
    # consecutive ranges covering every row once, in order, each within both bounds unless it is a single row
    cap = max(1, retrieval.RowPacking.ROW_SPAN * budget // S)
    flat = [i for a, b in rp.chunks for i in range(a, b)]
    assert flat == list(range(N))
    for a, b in rp.chunks:
        assert b > a and (b - a == 1 or (sum(counts[a:b]) <= budget and b - a <= cap))
    # greedy: no chunk could have taken the next row
    for (a, b), (c, _) in zip(rp.chunks, rp.chunks[1:]):
        assert (sum(counts[a:b + 1]) > budget or b + 1 - a > cap) and c == b
    for a, b in rp.chunks:
        idx, cu, seqs = rp.chunk(a, b)
        ref = [(i - a) * S + s for i in range(a, b) for s in range(S) if m[i, s] != 0]
        assert idx.dtype == cu.dtype == torch.int32 and idx.tolist() == ref
        assert cu.tolist() == list(np.concatenate([[0], np.cumsum(counts[a:b])]))
        assert seqs.total == len(ref) and seqs.max_sk == rp.max_len and seqs.n_seq == b - a
        assert seqs.idx_a is None  # packed addressing


@pytest.mark.parametrize("budget", [1, 16, 1000])
def test_runs_of_empty_rows_do_not_grow_a_chunk(budget):
    """rows without a valid token cost no budget; the padded-token bound still caps a chunk's rows, and with them the
    index arrays chunk() builds"""
    N, S = 5000, 48
    m = torch.zeros((N, S), dtype=torch.long)
    m[::997, 0] = 1  # one valid frame every 997 rows
    rp = retrieval.RowPacking(m, budget)
    bound = retrieval.RowPacking.ROW_SPAN * budget
    assert [i for a, b in rp.chunks for i in range(a, b)] == list(range(N))
    for a, b in rp.chunks:
        assert b - a == 1 or (b - a) * S <= bound
        idx, cu, seqs = rp.chunk(a, b)
        assert idx.numel() == int(m[a:b].sum()) <= max(budget, 1) and cu.numel() == b - a + 1


def test_any_mask_dtype_selects_the_nonzero_entries():
    m = _mask(5, 6, seed=1)
    ref = retrieval.RowPacking(m, 8)
    for other in (m.bool(), m.int(), m.float() * 3):
        got = retrieval.RowPacking(other, 8)
        assert got.chunks == ref.chunks
        for a, b in got.chunks:
            assert torch.equal(got.chunk(a, b)[0], ref.chunk(a, b)[0])


def _stub(training=False, W=512, F=512, video_dim=1024):
    emb = lambda n: types.SimpleNamespace(position_embeddings=types.SimpleNamespace(weight=torch.empty(n, 1)))
    return types.SimpleNamespace(training=training, task_config=types.SimpleNamespace(video_dim=video_dim, use_mil=False),
                                 bert=types.SimpleNamespace(embeddings=emb(W)),
                                 visual=types.SimpleNamespace(embeddings=emb(F)))


def test_embed_texts_checks():
    ids, am = torch.zeros(3, 8, dtype=torch.long), torch.ones(3, 8, dtype=torch.long)
    with torch.no_grad():
        with pytest.raises(ValueError):
            retrieval.embed_texts(_stub(), ids, am[:, :7])
        with pytest.raises(ValueError):
            retrieval.embed_texts(_stub(), ids, am, torch.zeros(3, 7, dtype=torch.long))
        with pytest.raises(ValueError):
            retrieval.embed_texts(_stub(W=7), ids, am)
        with pytest.raises(RuntimeError):  # CPU tensors: no CPU path
            retrieval.embed_texts(_stub(), ids, am)
        with pytest.raises(RuntimeError):
            retrieval.embed_texts(_stub(training=True), ids, am)
    with pytest.raises(RuntimeError):
        retrieval.embed_texts(_stub(), ids, am)  # gradients enabled


def test_embed_videos_checks():
    video, vm = torch.zeros(3, 5, 1024), torch.ones(3, 5, dtype=torch.long)
    with torch.no_grad():
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(), video.half(), vm)
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(), video, vm[:, :4])
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(), video, vm[:2])
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(video_dim=512), video, vm)
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(F=4), video, vm)
        with pytest.raises(ValueError):
            retrieval.embed_videos(_stub(), video[0, 0], vm)
        with pytest.raises(RuntimeError):
            retrieval.embed_videos(_stub(), video.double(), vm)
        with pytest.raises(RuntimeError):
            retrieval.embed_videos(_stub(training=True), video, vm)


@pytest.mark.parametrize("q,g,k", [((4, 8), (5, 8), 0), ((4, 8), (5, 8), 6), ((4, 8), (300, 8), 257),
                                   ((4, 8), (5, 12), 1), ((4, 6), (5, 6), 1), ((4,), (5, 4), 1)])
def test_topk_checks(q, g, k):
    with pytest.raises(ValueError):
        retrieval.topk(torch.zeros(q), torch.zeros(g), k)


def test_topk_checks_dtype_and_device():
    with pytest.raises(ValueError):
        retrieval.topk(torch.zeros(4, 8, dtype=torch.float64), torch.zeros(5, 8), 1)
    with pytest.raises(ValueError):
        retrieval.topk(torch.zeros(4, 8), torch.zeros(5, 8), True)
    with pytest.raises(ValueError):  # one device for both
        retrieval.topk(torch.zeros(4, 8), torch.zeros(5, 8, device="meta"), 2)
    with pytest.raises(RuntimeError):
        retrieval.topk(torch.zeros(4, 8), torch.zeros(5, 8), 2)
