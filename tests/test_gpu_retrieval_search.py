"""GPU: retrieval over large galleries (univl_b200.retrieval).  The exact streaming top-k (topk_similarity) against the
full mean-pooled similarity matrix and a strict host ranking, ties, gallery sizes and splits, repeat launches;
score_pairs against the dense evaluation's own logits bit for bit under both layouts and precisions; search against
the brute-force composition; and the memory both keep."""
import numpy as np
import pytest
import torch

from oracle import synth
from tests.model_util import build_model
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200 import runtime as rt
from univl_b200.modules import modeling

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _model(mode, cross_layers=2, use_mil=False, W=12, F=10, seed=0):
    cfg = synth.task_config(mode=mode, batch_size=2, text_layers=1, visual_layers=1, cross_layers=cross_layers,
                            max_words=W, max_frames=F, use_mil=use_mil)
    return build_model(cfg, sd=synth.make_state_dict(cfg, seed=seed)).eval()


def _outputs(Nt, W, Nv, F, seed):
    """bf16 encoder outputs and ragged int64 masks (prefixes and scattered rows, tokens 0 and 1 of every text row
    valid)"""
    g = _g(seed)
    seq = torch.randn((Nt, W, H), generator=g).to(torch.bfloat16).to(DEV)
    vis = torch.randn((Nv, F, H), generator=g).to(torch.bfloat16).to(DEV)
    tm = (torch.arange(W)[None] < torch.randint(1, W + 1, (Nt,), generator=g)[:, None]).long()
    tm[1::2] = (torch.rand(tm[1::2].shape, generator=g) < 0.5).long()
    tm[:, :2] = 1  # token 0 and one more: the text mean pool skips token 0 and would divide by zero without another
    vm = (torch.arange(F)[None] < torch.randint(1, F + 1, (Nv,), generator=g)[:, None]).long()
    vm[1::3] = (torch.rand(vm[1::3].shape, generator=g) < 0.5).long()
    return seq, vis, tm.to(DEV), vm.to(DEV)


def _mean_pool_matrix(model, seq, vis, am, vm):
    with torch.no_grad(), rt.use_model(model, model._device()):
        return model._mean_pool_similarity(seq.reshape(-1, H).contiguous(), vis.reshape(-1, H).contiguous(), am, vm)


def _strict_topk(sim, k):
    """per row: indices of the k largest by (score desc, index asc), on the host"""
    s = sim.cpu().numpy()
    cols = np.arange(s.shape[1])
    return np.stack([np.lexsort((cols, -row))[:k] for row in s])


def _check_topk(sim, scores, index, k):
    assert scores.shape == index.shape == (sim.shape[0], k) and index.dtype == torch.int64
    assert torch.equal(scores, sim.gather(1, index))  # the matrix's own bits
    assert np.array_equal(index.cpu().numpy(), _strict_topk(sim, k))


@pytest.mark.parametrize("use_mil", [False, True])
def test_topk_values_and_order_equal_the_full_matrix(use_mil):
    model = _model("ft_joint", use_mil=use_mil)
    seq, vis, am, vm = _outputs(37, 12, 1000, 10, seed=1)
    sim = _mean_pool_matrix(model, seq, vis, am, vm)
    with torch.no_grad():  # FT-Joint: get_similarity_logits is the mean-pooled similarity
        assert torch.equal(model.get_similarity_logits(seq, vis, am, vm), sim)
    for k in (1, 50, 256):
        _check_topk(sim, *retrieval.topk_similarity(model, seq, vis, am, vm, k), k)


def test_exact_ties_put_the_lower_index_first():
    model = _model("ft_joint")
    seq, vis, am, vm = _outputs(9, 12, 300, 10, seed=2)
    vis, vm = vis.clone(), vm.clone()
    for src, dups in ((4, (70, 150, 299)), (10, (11, 12, 200))):
        for d in dups:
            vis[d], vm[d] = vis[src], vm[src]
    sim = _mean_pool_matrix(model, seq, vis, am, vm)
    assert bool((sim[:, 4] == sim[:, 299]).all())
    for k in (3, 40, 256):
        _check_topk(sim, *retrieval.topk_similarity(model, seq, vis, am, vm, k), k)
    # k cutting through a run of equal scores keeps the lower indices
    t = torch.randn(3, H, generator=_g(3)).to(DEV)
    v = torch.randn(1, H, generator=_g(4)).to(DEV).repeat(100, 1)
    s, i = ops.sim_topk(t, v, 7)
    assert i.tolist() == [list(range(7))] * 3 and bool((s == s[:, :1]).all())


@pytest.mark.parametrize("Nt", [3, 300])
def test_gallery_sizes_splits_and_repeats_give_the_same_result(Nt):
    g = _g(5 + Nt)
    t = torch.nn.functional.normalize(torch.randn(Nt, H, generator=g), dim=1).to(DEV)
    v = torch.nn.functional.normalize(torch.randn(5000, H, generator=g), dim=1).to(DEV)
    k = 64
    for Nv in (64, 95, 96, 257, 4096, 5000):
        sim = ops.SimMatmulFn.apply(t, v[:Nv], 1)
        s, i = ops.sim_topk(t, v[:Nv], k)
        _check_topk(sim, s, i.long(), k)
        s2, i2 = ops.sim_topk(t, v[:Nv], k)  # a second launch: the same bytes
        assert torch.equal(s, s2) and torch.equal(i, i2)
    # the caller splits the gallery into chunks and merges the chunk lists by the same order
    sim = ops.SimMatmulFn.apply(t, v, 1)
    parts = [(0, 1700), (1700, 1800), (1800, 5000)]
    cs = torch.cat([ops.sim_topk(t, v[a:b], k)[0] for a, b in parts], 1)
    ci = torch.cat([ops.sim_topk(t, v[a:b], k)[1].long() + a for a, b in parts], 1)
    order = [np.lexsort((ci_r, -cs_r))[:k] for cs_r, ci_r in zip(cs.cpu().numpy(), ci.cpu().numpy())]
    merged = np.take_along_axis(ci.cpu().numpy(), np.stack(order), 1)
    assert np.array_equal(merged, _strict_topk(sim, k))
    rt.reserve_sms(40)  # fewer usable SMs change the split, not the result
    try:
        s3, i3 = ops.sim_topk(t, v, k)
    finally:
        rt.reserve_sms(0)
    assert torch.equal(s3, ops.sim_topk(t, v, k)[0]) and torch.equal(i3, ops.sim_topk(t, v, k)[1])


def _grid(model, args, layout, precision, monkeypatch):
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", layout)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", precision)
    with torch.no_grad():
        return model.get_similarity_logits(*args)


@pytest.mark.parametrize("W,F,cross_layers", [(12, 10, 1), (12, 10, 2), (128, 160, 2)])
@pytest.mark.parametrize("layout", ["padded", "packed"])
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_score_pairs_equal_the_grid_bit_for_bit(W, F, cross_layers, layout, precision, monkeypatch):
    model = _model("ft_align", cross_layers=cross_layers, W=W, F=F, seed=cross_layers)
    Nt, Nv = 7, 6
    seq, vis, am, vm = _outputs(Nt, W, Nv, F, seed=6)
    am, vm = am.clone(), vm.clone()
    am[0], vm[0] = 1, 1  # the longest pair has every token: (128, 160) runs the key-tiled kernel
    args = (seq, vis, am, vm)
    grid = _grid(model, args, layout, precision, monkeypatch).cpu()
    g = _g(7)
    ti = torch.randint(0, Nt, (40,), generator=g)
    vi = torch.randint(0, Nv, (40,), generator=g)
    ti[7], vi[7] = ti[3], vi[3]  # unsorted, with a repeat
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 6 * (W + F))  # several list tiles, the last partial
    with torch.no_grad():
        got = retrieval.score_pairs(model, seq, vis, am, vm, ti.to(DEV), vi.int())
        assert torch.equal(got.cpu(), grid[ti, vi])
        empty = retrieval.score_pairs(model, seq, vis, am, vm, [], [])
        assert empty.shape == (0,) and empty.dtype == torch.float32
        # one list tile holding everything gives the same bits
        monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 1 << 30)
        assert torch.equal(retrieval.score_pairs(model, seq, vis, am, vm, ti, vi).cpu(), got.cpu())


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_a_text_row_without_token_0_scores_like_the_grid(precision, monkeypatch):
    model = _model("ft_align", cross_layers=2, seed=3)
    seq, vis, am, vm = _outputs(5, 12, 4, 10, seed=8)
    am = am.clone()
    am[2, 0] = 0
    args = (seq, vis, am, vm)
    padded = _grid(model, args, "padded", precision, monkeypatch).cpu()
    grid = _grid(model, args, "packed", precision, monkeypatch).cpu()
    assert torch.equal(grid, padded)  # the grid fell back to the padded layout
    ti = torch.tensor([2, 0, 4, 2, 1])
    vi = torch.tensor([3, 1, 0, 3, 2])
    with torch.no_grad():
        assert torch.equal(retrieval.score_pairs(model, seq, vis, am, vm, ti, vi).cpu(), grid[ti, vi])


def test_score_pairs_refuses_training_mode_and_gradients():
    model = _model("ft_align", cross_layers=1)
    seq, vis, am, vm = _outputs(3, 12, 3, 10, seed=9)
    with pytest.raises(RuntimeError):
        retrieval.score_pairs(model, seq, vis, am, vm, [0], [0])
    model.train()
    with torch.no_grad(), pytest.raises(RuntimeError):
        retrieval.score_pairs(model, seq, vis, am, vm, [0], [0])
    with torch.no_grad(), pytest.raises(ValueError):
        retrieval.score_pairs(_model("ft_joint").eval(), seq, vis, am, vm, [0], [0])


def _brute_search(sim1, sim2, ks, k):
    short = _strict_topk(sim1, ks)
    s2 = np.take_along_axis(sim2.cpu().numpy(), short, 1)
    order = np.stack([np.lexsort((np.arange(ks), -row))[:k] for row in s2])  # rerank desc, then shortlist rank
    return np.take_along_axis(s2, order, 1), np.take_along_axis(short, order, 1)


@pytest.mark.parametrize("layout", ["padded", "packed"])
def test_search_equals_the_brute_force_composition(layout, monkeypatch):
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", layout)
    align = _model("ft_align", cross_layers=2, seed=4)
    joint = _model("ft_joint", seed=5)
    Nt, Nv, ks, k = 11, 90, 20, 5
    seq, vis, am, vm = _outputs(Nt, 12, Nv, 10, seed=10)
    seq2, vis2, _, _ = _outputs(Nt, 12, Nv, 10, seed=11)  # the re-ranking model's own encoder outputs
    with torch.no_grad():
        # one model for both stages
        sim1 = _mean_pool_matrix(align, seq, vis, am, vm)
        sim2 = align.get_similarity_logits(seq, vis, am, vm)
        s, i = retrieval.search(align, align, seq, vis, am, vm, ks, k)
        rs, ri = _brute_search(sim1, sim2, ks, k)
        assert np.array_equal(i.cpu().numpy(), ri) and np.array_equal(s.cpu().numpy(), rs)
        # FT-Joint shortlist, FT-Align re-rank on its own outputs
        sim1 = joint.get_similarity_logits(seq, vis, am, vm)
        sim2 = align.get_similarity_logits(seq2, vis2, am, vm)
        s, i = retrieval.search(joint, align, seq, vis, am, vm, ks, k, seq2, vis2)
        rs, ri = _brute_search(sim1, sim2, ks, k)
        assert np.array_equal(i.cpu().numpy(), ri) and np.array_equal(s.cpu().numpy(), rs)
        assert i.dtype == torch.int64 and s.dtype == torch.float32


def test_topk_over_a_gallery_past_8_gib_of_similarity_stays_bounded():
    """4096 x 530,000 fp32 similarities would take 8.1 GiB; the shortlist holds the pooled rows, its [Nt, k] outputs and
    at most 128 MiB more above its inputs"""
    model = _model("ft_joint", F=2)
    Nt, Nv, k = 4096, 530_000, 100
    g = torch.Generator(device=DEV).manual_seed(12)
    seq = torch.randn((Nt, 12, H), generator=g, device=DEV).to(torch.bfloat16)
    vis = torch.randn((Nv, 2, H), generator=g, device=DEV).to(torch.bfloat16)
    am = torch.ones((Nt, 12), dtype=torch.long, device=DEV)
    vm = torch.ones((Nv, 2), dtype=torch.long, device=DEV)
    assert Nt * Nv * 4 > 8 * 2 ** 30
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    s, i = retrieval.topk_similarity(model, seq, vis, am, vm, k)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = (Nt + Nv) * H * 4 + Nt * k * 16 + 128 * 2 ** 20
    print("topk over %d x %d: peak %.2f GiB above the inputs (bound %.2f GiB)" % (Nt, Nv, peak / 2 ** 30,
                                                                                 bound / 2 ** 30))
    assert peak <= bound
    assert bool((s[:, :-1] >= s[:, 1:]).all()) and int(i.min()) >= 0 and int(i.max()) < Nv


def test_one_million_listed_pairs_stay_within_the_grid_tile_peak(monkeypatch):
    """1024 x 1024 random listed pairs against the 1024 x 1024 grid at W = F = 48: the same tiles' peak"""
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", "padded")
    model = _model("ft_align", cross_layers=2, W=48, F=48, seed=6)
    Nt = Nv = 1024
    seq, vis, am, vm = _outputs(Nt, 48, Nv, 48, seed=13)
    peaks = {}
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        grid = model.get_similarity_logits(seq, vis, am, vm)
    torch.cuda.synchronize()
    peaks["grid"] = torch.cuda.max_memory_allocated() - base
    g = _g(14)
    ti = torch.randint(0, Nt, (Nt * Nv,), generator=g)
    vi = torch.randint(0, Nv, (Nt * Nv,), generator=g)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        got = retrieval.score_pairs(model, seq, vis, am, vm, ti, vi)
    torch.cuda.synchronize()
    peaks["list"] = torch.cuda.max_memory_allocated() - base
    print("1M pairs, W = F = 48: peak grid %.2f GiB, list %.2f GiB" % (peaks["grid"] / 2 ** 30,
                                                                       peaks["list"] / 2 ** 30))
    # the list path keeps the per-source embedding rows for its tiles' residuals (as the packed layout does) and the
    # device copies of the two int32 lists; its tiles are the grid's size
    extra = (Nt * 48 + Nv * 48) * H * 2 + ti.numel() * 8
    assert peaks["list"] <= peaks["grid"] + extra
    assert torch.equal(got, grid[ti.to(DEV), vi.to(DEV)])
