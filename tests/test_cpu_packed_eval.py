"""CPU: the packed evaluation layout's switch (UNIVL_EVAL_LAYOUT), its attention_mask[:, 0] fallback rule, the packing
metadata (ops.PairPacking) against a plain Python loop, and the tile choice's packed-token budget."""
import pytest
import torch

from univl_b200 import lib
from univl_b200 import ops
from univl_b200.modules import modeling


def test_switch_default_packed_and_bad_values(monkeypatch):
    monkeypatch.delenv("UNIVL_EVAL_LAYOUT", raising=False)
    assert modeling.eval_layout() == "padded"
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", "packed")
    assert modeling.eval_layout() == "packed"
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", "padded")
    assert modeling.eval_layout() == "padded"
    for bad in ("", "PACKED", "varlen", "packed "):
        monkeypatch.setenv("UNIVL_EVAL_LAYOUT", bad)
        with pytest.raises(ValueError):
            modeling.eval_layout()


def test_fallback_rule_reads_token_0_of_every_text_row():
    m = torch.tensor([[1, 1, 0], [1, 0, 1]])
    v = torch.tensor([[0, 1], [0, 0]])
    assert ops.PairPacking(m, v).token0_valid
    m2 = m.clone()
    m2[1, 0] = 0
    assert not ops.PairPacking(m2, v).token0_valid


@pytest.mark.parametrize("p", [0.0, 0.3, 1.0])
def test_valid_rows_without_a_sync_equal_nonzero(p):
    g = torch.Generator().manual_seed(int(p * 10))
    m = torch.rand(37, 11, generator=g) < p
    n = int(m.sum())
    got = ops._valid_rows(m, n)
    assert got.dtype == torch.int32 and got.tolist() == m.reshape(-1).nonzero().view(-1).tolist()


def test_the_new_entries_are_declared():
    decl = lib.parse_header()
    for name in ("univl_attention_varlen_fwd", "univl_gather_rows_varlen"):
        assert name in decl


def _masks(kind, Nt, W, Nv, F, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "prefix":
        lt = torch.randint(1, W + 1, (Nt,), generator=g)
        lv = torch.randint(1, F + 1, (Nv,), generator=g)
        return ((torch.arange(W)[None] < lt[:, None]).long(), (torch.arange(F)[None] < lv[:, None]).long())
    tm = (torch.rand(Nt, W, generator=g) < 0.6).long()
    vm = (torch.rand(Nv, F, generator=g) < 0.5).long()
    tm[:, 0] = 1
    if kind == "zero_video":
        vm[::2] = 0
    elif kind == "token0_padded":
        tm[1, 0] = 0
    return tm, vm


def _loop_reference(tm, vm, t0, t1, v0, v1):
    """per pair p = (i - t0) * nv + (j - v0): its packed rows as ("t", source row) / ("v", source row), by loops"""
    Nt, W = tm.shape
    Nv, F = vm.shape
    seqs = []
    for i in range(t0, t1):
        for j in range(v0, v1):
            rows = [("t", i * W + s) for s in range(W) if tm[i, s] != 0]
            rows += [("v", j * F + s) for s in range(F) if vm[j, s] != 0]
            seqs.append(rows)
    return seqs


@pytest.mark.parametrize("kind", ["prefix", "scattered", "zero_video", "token0_padded"])
def test_packing_metadata_matches_a_python_loop(kind):
    Nt, W, Nv, F = 5, 9, 4, 7
    tm, vm = _masks(kind, Nt, W, Nv, F, seed=3)
    pk = ops.PairPacking(tm, vm)
    assert pk.len_t == [int(r.sum()) for r in tm] and pk.len_v == [int(r.sum()) for r in vm]
    assert pk.max_sk == max(pk.len_t) + max(pk.len_v)
    for t0, t1, v0, v1 in [(0, Nt, 0, Nv), (1, 4, 2, 4), (4, 5, 0, 1)]:
        seqs = pk.tile(t0, t1, v0, v1)
        ref = _loop_reference(tm, vm, t0, t1, v0, v1)
        assert seqs.n_seq == len(ref)
        cu = seqs.cu.tolist()
        assert cu[0] == 0 and seqs.total == cu[-1] == sum(len(r) for r in ref) == pk.tokens(t0, t1, v0, v1)
        assert seqs.max_sk == pk.max_sk >= max(len(r) for r in ref)
        for p, rows in enumerate(ref):
            assert cu[p + 1] - cu[p] == len(rows)
            la = int(seqs.len_a[p])
            got = [("t", int(seqs.idx_a[int(seqs.start_a[p]) + r])) for r in range(la)]
            got += [("v", int(seqs.idx_b[int(seqs.start_b[p]) + r])) for r in range(len(rows) - la)]
            assert got == rows, (kind, p)
        for t in (seqs.cu, seqs.idx_a, seqs.idx_b, seqs.start_a, seqs.start_b, seqs.len_a):
            assert t.dtype == torch.int32
        packed = seqs.packed()
        assert packed.idx_a is None and packed.cu is seqs.cu and packed.total == seqs.total


@pytest.mark.parametrize("budget", [1, 40, 300, 1000, 1 << 18])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_tiles_cover_every_pair_once_within_the_packed_token_budget(budget, seed):
    g = torch.Generator().manual_seed(seed)
    Nt, Nv = int(torch.randint(1, 40, (1,), generator=g)), int(torch.randint(1, 40, (1,), generator=g))
    len_t = torch.randint(1, 49, (Nt,), generator=g).tolist()
    len_v = torch.randint(0, 49, (Nv,), generator=g).tolist()
    tiles = modeling._packed_eval_tiles(len_t, len_v, budget)
    seen = torch.zeros(Nt, Nv, dtype=torch.int64)
    for t0, t1, v0, v1 in tiles:
        assert 0 <= t0 < t1 <= Nt and 0 <= v0 < v1 <= Nv
        seen[t0:t1, v0:v1] += 1
        tokens = (v1 - v0) * sum(len_t[t0:t1]) + (t1 - t0) * sum(len_v[v0:v1])
        # within the budget, unless the tile is a single pair that alone exceeds it
        assert tokens <= budget or (t1 - t0, v1 - v0) == (1, 1), (t0, t1, v0, v1, tokens)
    assert bool((seen == 1).all())
    if budget >= 1 << 18:
        assert len(tiles) == 1


def test_tiles_use_the_budget_on_short_sequences():
    """at W = F = 48 with lengths 8..20 / 12..30 the tiles are sized by packed tokens, not by W + F"""
    g = torch.Generator().manual_seed(5)
    len_t = torch.randint(8, 21, (3500,), generator=g).tolist()
    len_v = torch.randint(12, 31, (3500,), generator=g).tolist()
    budget = 1 << 18
    tiles = modeling._packed_eval_tiles(len_t, len_v, budget)
    padded_tiles = -(-3500 // modeling._eval_tile(3500, 3500, 96, budget)[0]) * \
        -(-3500 // modeling._eval_tile(3500, 3500, 96, budget)[1])
    assert len(tiles) < padded_tiles
    full = [(v1 - v0) * sum(len_t[t0:t1]) + (t1 - t0) * sum(len_v[v0:v1]) for t0, t1, v0, v1 in tiles]
    assert max(full) <= budget
    assert sorted(full)[len(full) // 2] >= budget * 0.9  # most tiles are nearly full
