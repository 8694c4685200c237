"""CPU: the list metadata of retrieval.score_pairs (ops.PairPacking.pairs, ops.padded_pair_seqs) against the grid's
own tile() and a Python loop, the list tiling, and the argument checks of the retrieval entry points."""
import numpy as np
import pytest
import torch

from tests.test_cpu_packed_eval import _masks
from univl_b200 import lib
from univl_b200 import ops
from univl_b200 import retrieval


def test_the_new_entries_are_declared():
    decl = lib.parse_header()
    for name in ("univl_sim_topk", "univl_attention_pair_list_fwd"):
        assert name in decl


@pytest.mark.parametrize("kind", ["prefix", "scattered", "zero_video"])
def test_pairs_over_the_grid_list_equal_tile(kind):
    Nt, W, Nv, F = 5, 9, 4, 7
    tm, vm = _masks(kind, Nt, W, Nv, F, seed=3)
    pk = ops.PairPacking(tm, vm)
    for t0, t1, v0, v1 in [(0, Nt, 0, Nv), (1, 4, 2, 4), (4, 5, 0, 1)]:
        ti = torch.arange(t0, t1).repeat_interleave(v1 - v0)
        vi = torch.arange(v0, v1).repeat(t1 - t0)
        got, ref = pk.pairs(ti.int(), vi), pk.tile(t0, t1, v0, v1)
        assert got.total == ref.total and got.max_sk == ref.max_sk == pk.max_sk and got.n_seq == ref.n_seq
        for name in ("cu", "start_a", "start_b", "len_a"):
            a, b = getattr(got, name), getattr(ref, name)
            assert a.dtype == torch.int32 and torch.equal(a, b), name
        assert got.idx_a is pk.idx_t and got.idx_b is pk.idx_v


def _loop_rows(tm, vm, ti, vi, padded):
    W, F = tm.shape[1], vm.shape[1]
    out = []
    for i, j in zip(ti, vi):
        rows = [("t", i * W + s) for s in range(W) if padded or tm[i, s] != 0]
        rows += [("v", j * F + s) for s in range(F) if padded or vm[j, s] != 0]
        out.append(rows)
    return out


def _rows_of(seqs, p):
    la, n = int(seqs.len_a[p]), int(seqs.cu[p + 1] - seqs.cu[p])
    got = [("t", int(seqs.idx_a[int(seqs.start_a[p]) + r])) for r in range(la)]
    return got + [("v", int(seqs.idx_b[int(seqs.start_b[p]) + r])) for r in range(n - la)]


@pytest.mark.parametrize("kind", ["prefix", "scattered", "zero_video"])
def test_arbitrary_lists_match_a_python_loop(kind):
    Nt, W, Nv, F = 6, 9, 5, 7
    tm, vm = _masks(kind, Nt, W, Nv, F, seed=4)
    g = torch.Generator().manual_seed(1)
    ti = torch.randint(0, Nt, (23,), generator=g)
    vi = torch.randint(0, Nv, (23,), generator=g)
    ti[5], vi[5] = ti[2], vi[2]  # a repeated pair
    pk = ops.PairPacking(tm, vm)
    for padded in (False, True):
        seqs = ops.padded_pair_seqs(ti.int(), vi.int(), Nt, W, Nv, F) if padded else pk.pairs(ti, vi.int())
        ref = _loop_rows(tm, vm, ti.tolist(), vi.tolist(), padded)
        assert seqs.n_seq == len(ref) and seqs.total == int(seqs.cu[-1]) == sum(len(r) for r in ref)
        assert seqs.max_sk == (W + F if padded else pk.max_sk)
        for p, rows in enumerate(ref):
            assert _rows_of(seqs, p) == rows, (padded, p)
    empty = pk.pairs(torch.zeros(0, dtype=torch.int32), torch.zeros(0, dtype=torch.int32))
    assert empty.n_seq == 0 and empty.total == 0


@pytest.mark.parametrize("budget", [1, 50, 1000])
def test_list_chunks_cover_the_list_in_order_within_the_budget(budget):
    cost = np.random.default_rng(budget).integers(1, 97, 400)
    chunks = retrieval._pair_chunks(cost, budget)
    assert chunks[0][0] == 0 and chunks[-1][1] == cost.size
    for (a, b), (c, _) in zip(chunks, chunks[1:] + [(cost.size, None)]):
        assert b == c and a < b
        assert cost[a:b].sum() <= budget or b - a == 1
    assert retrieval._pair_chunks(cost[:0], budget) == []


def test_host_index_checks():
    assert retrieval._host_index(torch.tensor([0, 3], dtype=torch.int32), 4, "x").tolist() == [0, 3]
    assert retrieval._host_index([1, 2], 4, "x").dtype == np.int64
    assert retrieval._host_index([], 4, "x").size == 0
    for bad in (torch.tensor([0, 4]), torch.tensor([-1]), [5], np.array([0.0, 1.0]), torch.tensor([0.0]),
                torch.tensor([[0, 1]]), torch.tensor([True])):
        with pytest.raises(ValueError):
            retrieval._host_index(bad, 4, "x")


class _Model:
    """the attributes score_pairs reads before any device work"""
    training = False
    cross = object()
    _stage_two = False
    train_sim_after_cross = True

    def _device(self):
        return torch.device("cpu")


def test_score_pairs_rules_and_list_checks():
    seq, vis = torch.zeros(3, 4, 8), torch.zeros(2, 5, 8)
    am, vm = torch.ones(3, 4, dtype=torch.long), torch.ones(2, 5, dtype=torch.long)
    m = _Model()
    with torch.no_grad():
        for ti, vi in (([0, 3], [0, 1]), ([0, 1], [0, 2]), ([0, 1], [0]), (torch.tensor([0.5]), [0])):
            with pytest.raises(ValueError):
                retrieval.score_pairs(m, seq, vis, am, vm, ti, vi)
        m.cross = None
        with pytest.raises(ValueError, match="cross-encoder"):
            retrieval.score_pairs(m, seq, vis, am, vm, [0], [0])
    m = _Model()
    with torch.enable_grad(), pytest.raises(RuntimeError, match="no_grad"):
        retrieval.score_pairs(m, seq, vis, am, vm, [0], [0])
    m.training = True
    with torch.no_grad(), pytest.raises(RuntimeError, match="eval"):
        retrieval.score_pairs(m, seq, vis, am, vm, [0], [0])
    for k, ks in ((0, 5), (6, 5), (-1, 5)):
        with pytest.raises(ValueError):
            retrieval.search(m, m, seq, vis, am, vm, ks, k)


@pytest.mark.parametrize("k,Nv", [(0, 10), (-3, 10), (257, 300), (11, 10)])
def test_sim_topk_rejects_k_outside_1_to_min_256_nv(k, Nv):
    """the kernel entry checks its arguments before touching the device"""
    fake = 1 << 20  # non-null, 16-byte aligned: never dereferenced, the check fails first
    with pytest.raises(RuntimeError, match="k="):
        lib.call("univl_sim_topk", fake, fake, fake, fake, 4, Nv, 768, k, None)


def test_sim_topk_rejects_bad_shapes():
    fake = 1 << 20
    for Nt, Nv, H in ((4, 0, 768), (4, 10, 6), (-1, 10, 768)):
        with pytest.raises(RuntimeError, match="sim_topk"):
            lib.call("univl_sim_topk", fake, fake, fake, fake, Nt, Nv, H, 1, None)
