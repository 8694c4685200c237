"""CPU: ground-truth ranks of retrieval (retrieval.ranks / ranks_from_scores / rank_metrics).  The argument checks, the
positive ranges, rank_metrics against numpy, and the rank rule (host_ranks, the reference the GPU tests also use)
against np.lexsort and the reference's compute_metrics formula."""
import numpy as np
import pytest
import torch

from univl_b200 import lib
from univl_b200 import retrieval


def host_ranks(scores, query_labels=None, gallery_labels=None):
    """The rank rule on the host: per query, the best positive by (score desc, index asc), then the count of gallery
    rows ranked above it.  scores: a 2-D array; labels default to arange."""
    s = np.asarray(scores)
    Nq, Ng = s.shape
    ql = np.arange(Nq) if query_labels is None else np.asarray(query_labels)
    gl = np.arange(Ng) if gallery_labels is None else np.asarray(gallery_labels)
    out = np.empty(Nq, dtype=np.int64)
    for i in range(Nq):
        pos = np.flatnonzero(gl == ql[i])
        b = pos[np.argmax(s[i, pos])]  # argmax: the first (lowest index) of equal best scores
        out[i] = np.sum((s[i] > s[i, b]) | ((s[i] == s[i, b]) & (np.arange(Ng) < b)))
    return out


def reference_ind(x):
    """the `ind` of the reference's metrics.compute_metrics (the diagonal's rank), as it computes it"""
    sx = np.sort(-x, axis=1)
    d = np.diag(-x)[:, np.newaxis]
    return np.where(sx - d == 0)[1]


def _tied(Nq, Ng, seed):
    """scores on a coarse grid: every row full of exact ties"""
    return np.random.default_rng(seed).integers(-3, 4, (Nq, Ng)).astype(np.float32)


def test_the_new_entries_are_declared():
    decl = lib.parse_header()
    for name in ("univl_sim_best_positive", "univl_sim_rank"):
        assert name in decl


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_rule_against_lexsort_on_tied_matrices(seed):
    rng = np.random.default_rng(seed)
    Nq, Ng = 40, 57
    s = _tied(Nq, Ng, seed)
    s[:, 10] = s[:, 3]  # a duplicated gallery column
    s[7] = s[2]  # a duplicated query row
    for ql, gl in ((None, None), (rng.integers(0, 6, Nq), rng.integers(0, 6, Ng))):
        if gl is not None:
            gl[:6] = np.arange(6)  # every label has a row
        r = host_ranks(s, ql, gl)
        qlab = np.arange(Nq) if ql is None else ql
        glab = np.arange(Ng) if gl is None else gl
        for i in range(Nq):
            order = np.lexsort((np.arange(Ng), -s[i]))  # score descending, then index ascending
            first = int(np.flatnonzero(glab[order] == qlab[i])[0])
            assert r[i] == first, (i, r[i], first)
            assert not np.any(glab[order[:first]] == qlab[i])  # every row ranked above is a negative


def test_host_rule_is_compute_metrics_without_ties_and_counts_once_with_them():
    x = np.random.default_rng(3).standard_normal((50, 50)).astype(np.float32)
    assert np.array_equal(host_ranks(x), reference_ind(x))
    ref = reference_ind(x)
    for k in (1, 5, 10):
        assert retrieval.rank_metrics(host_ranks(x))["R%d" % k] == float(np.sum(ref < k)) / len(ref)
    assert retrieval.rank_metrics(host_ranks(x))["MR"] == np.median(ref) + 1
    # with ties the reference lists one entry per tied value, so its `ind` outgrows N; the rule gives one rank per query
    t = _tied(50, 50, 4)
    assert len(reference_ind(t)) > 50 and host_ranks(t).shape == (50,)


@pytest.mark.parametrize("r", [[0], [3, 0], [0, 1, 2, 9, 4, 30], [5, 5, 5, 5], [7] * 9,
                               list(np.random.default_rng(5).integers(0, 40, 101))])
def test_rank_metrics_against_numpy(r):
    a = np.array(r, dtype=np.int64)
    n = a.size
    s = np.sort(a)
    median = s[n // 2] if n % 2 else (s[n // 2 - 1] + s[n // 2]) / 2
    want = {"R1": sum(x < 1 for x in r) / n, "R5": sum(x < 5 for x in r) / n, "R10": sum(x < 10 for x in r) / n,
            "MR": median + 1.0, "MeanR": sum(r) / n + 1.0}
    for arg in (a, torch.tensor(a), list(r)):
        got = retrieval.rank_metrics(arg)
        assert set(got) == set(want)
        for key in want:
            assert got[key] == pytest.approx(want[key], rel=1e-12, abs=0), key
            assert isinstance(got[key], float)
    with pytest.raises(ValueError):
        retrieval.rank_metrics(np.zeros((0,), dtype=np.int64))
    with pytest.raises(ValueError):
        retrieval.rank_metrics(np.zeros((2, 2), dtype=np.int64))


def test_positive_ranges_on_the_host():
    gl = torch.tensor([3, 1, 3, 0, 1, 3, 7])
    ql = torch.tensor([3, 0, 7, 1, 3])
    perm, lo, hi = retrieval._positive_ranges("ranks", ql, gl)
    for i in range(ql.numel()):
        assert perm[lo[i]:hi[i]].tolist() == [j for j in range(gl.numel()) if gl[j] == ql[i]]
    with pytest.raises(ValueError, match="2 queries have no positive"):
        retrieval._positive_ranges("ranks", torch.tensor([3, 2, 5]), gl)


def _meta(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def test_ranks_argument_checks():
    q, g = _meta(4, 8), _meta(6, 8)
    lab = dict(dtype=torch.int64, device="meta")
    bad = [
        ((_meta(4, 8, dtype=torch.float16), g), {}, "float32"),
        ((_meta(4, 8, 1), g), {}, "float32"),
        ((q, _meta(6, 12)), {}, "width"),
        ((_meta(4, 6), _meta(6, 6)), {}, "width"),
        ((_meta(7, 8), g), {}, "Nq <= Ng"),
        ((q, g), {"query_labels": torch.empty(5, **lab)}, "query_labels holds 5"),
        ((q, g), {"gallery_labels": torch.empty(4, **lab)}, "gallery_labels holds 4"),
        ((q, g), {"query_labels": torch.empty(4, 1, **lab)}, "1-D"),
        ((q, g), {"query_labels": torch.empty(4, dtype=torch.float32, device="meta")}, "int32 or int64"),
        ((q, g), {"gallery_labels": [0, 1, 2, 3, 4, 5]}, "int32 or int64"),
        ((q, g), {"query_labels": torch.zeros(4, dtype=torch.int32)}, "is on cpu"),
        ((q, torch.zeros(6, 8)), {}, "one device"),
    ]
    for args, kw, match in bad:
        with pytest.raises(ValueError, match=match):
            retrieval.ranks(*args, **kw)
    # Nq > Ng is fine when labels say where the positives are
    with pytest.raises(RuntimeError, match="CUDA"):
        retrieval.ranks(torch.zeros(7, 8), torch.zeros(6, 8), query_labels=torch.zeros(7, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        retrieval.ranks(torch.zeros(4, 8), torch.zeros(6, 8))


def test_ranks_from_scores_argument_checks():
    lab = dict(dtype=torch.int64, device="meta")
    for args, kw, match in (((_meta(4, 6, dtype=torch.float64),), {}, "float32"), ((_meta(4),), {}, "2-D"),
                            ((_meta(7, 6),), {}, "Nq <= Ng"),
                            ((_meta(4, 6),), {"gallery_labels": torch.empty(5, **lab)}, "holds 5"),
                            ((_meta(4, 6),), {"query_labels": torch.zeros(4, dtype=torch.int64)}, "is on cpu")):
        with pytest.raises(ValueError, match=match):
            retrieval.ranks_from_scores(*args, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        retrieval.ranks_from_scores(torch.zeros(4, 6))


def test_kernel_entries_check_their_arguments():
    fake = 1 << 20  # non-null, 16-byte aligned: never dereferenced, the check fails first
    for Nt, Nv, H in ((4, 0, 768), (4, 10, 6), (-1, 10, 768)):
        with pytest.raises(RuntimeError, match="sim_rank"):
            lib.call("univl_sim_rank", fake, fake, fake, fake, fake, Nt, Nv, H, None)
    with pytest.raises(RuntimeError, match="aligned"):
        lib.call("univl_sim_rank", fake + 4, fake, fake, fake, fake, 4, 10, 768, None)
    with pytest.raises(RuntimeError, match="null"):
        lib.call("univl_sim_rank", fake, None, fake, fake, fake, 4, 10, 768, None)
    for Nt, Nv, H in ((4, 0, 768), (-1, 10, 768), (4, 10, 0)):
        with pytest.raises(RuntimeError, match="sim_best_positive"):
            lib.call("univl_sim_best_positive", fake, fake, fake, fake, fake, fake, fake, Nt, Nv, H, None)
    with pytest.raises(RuntimeError, match="null"):
        lib.call("univl_sim_best_positive", fake, fake, None, fake, fake, fake, fake, 4, 10, 768, None)
