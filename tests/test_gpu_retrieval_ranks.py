"""GPU: ground-truth ranks of retrieval (retrieval.ranks / ranks_from_scores).  The streaming ranks against the dense
SimMatmulFn matrix exactly, on both sides of the gallery split, with many positives per query and with ties; their
agreement with topk; repeat, side-stream, reserved-SM and graph-replayed launches; a cross encoder's logits; and an
FT-Joint model end to end."""
import numpy as np
import pytest
import torch

from oracle import synth
from tests.model_util import build_model
from tests.test_cpu_retrieval_ranks import host_ranks, reference_ind
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture
def pairs():
    """(queries, gallery, query_labels, gallery_labels) for a labelling kind: gallery rows are noisy copies of their
    query's vector, so ranks spread from 0 to far down the list"""
    def make(Nq, Ng, H, kind, seed):
        noise = 0.3 * H ** 0.5  # a positive's margin is ~H, a negative's spread ~noise sqrt(H): ranks spread
        g = torch.Generator(device="cpu").manual_seed(seed)
        if kind == "one_to_one":
            ql, gl = None, None
            owner = torch.arange(Ng) % Nq
        elif kind == "many_gallery":  # several gallery rows per query (video-to-text with many captions)
            ql, gl = torch.arange(Nq), torch.arange(Ng) % Nq
            owner = gl
        else:  # "many_queries": several queries per gallery row (text-to-video with many captions)
            ql, gl = torch.arange(Nq) % Ng, None
            owner = torch.arange(Ng)
        q = torch.randn((Nq, H), generator=g)
        base = q[owner] if kind != "many_queries" else torch.randn((Ng, H), generator=g)
        if kind == "many_queries":
            q = base[ql] + noise * torch.randn((Nq, H), generator=g)
        gal = base + noise * torch.randn((Ng, H), generator=g)
        dev = lambda x: None if x is None else x.to(DEV)
        return q.to(DEV), gal.to(DEV), dev(ql), dev(gl)
    return make


def _dense(q, g):
    return ops.SimMatmulFn.apply(q, g, 1)


@pytest.mark.parametrize("Nq,Ng,H", [(37, 5000, 768), (3001, 517, 768), (5, 70, 4), (203, 1201, 132),
                                     (16, 2048, 768)])
@pytest.mark.parametrize("kind", ["one_to_one", "many_gallery", "many_queries"])
def test_ranks_equal_the_dense_matrix_exactly(pairs, Nq, Ng, H, kind):
    if kind != "many_queries" and Nq > Ng:  # every query needs a positive
        Nq, Ng = Ng, Nq
    q, g, ql, gl = pairs(Nq, Ng, H, kind, seed=Nq + Ng + H)
    with torch.no_grad():
        r = retrieval.ranks(q, g, ql, gl)
        ref = retrieval.ranks_from_scores(_dense(q, g), ql, gl)
        assert r.dtype == torch.int64 and r.shape == (Nq,)
        assert torch.equal(r, ref)
        assert np.array_equal(r.cpu().numpy(), host_ranks(_dense(q, g).cpu().numpy(),
                                                          None if ql is None else ql.cpu().numpy(),
                                                          None if gl is None else gl.cpu().numpy()))
        # the other direction: the gallery's rows as queries, scored by the transposed matrix's bits
        if kind == "one_to_one":
            r2 = retrieval.ranks(g[:Nq], q)
            assert torch.equal(r2, retrieval.ranks_from_scores(_dense(q, g[:Nq]).t().contiguous()))
        else:  # the gallery rows that some query shares a label with
            gl_ = torch.arange(Ng, device=DEV) if gl is None else gl
            ql_ = torch.arange(Nq, device=DEV) if ql is None else ql
            keep = torch.isin(gl_, ql_)
            r2 = retrieval.ranks(g[keep], q, gl_[keep], ql_)
            assert torch.equal(r2, retrieval.ranks_from_scores(_dense(q, g).t()[keep].contiguous(), gl_[keep], ql_))
    print("Nq=%d Ng=%d H=%d %s: median rank %d, max %d" % (Nq, Ng, H, kind, int(r.median()), int(r.max())))


def _tied_vectors(Nq, Ng, H, seed):
    """entries in {-1, 0, 1} / 4: every dot product is exact, and rows are full of equal scores; duplicated gallery
    rows and queries on top"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randint(-1, 2, (Nq, H), generator=g).float() / 4
    v = torch.randint(-1, 2, (Ng, H), generator=g).float() / 4
    v[100:140] = v[100].clone()
    v[[5, 77, 299]] = v[2].clone()
    q[[3, 9]] = q[1].clone()
    return q.to(DEV), v.to(DEV)


def test_ties_follow_the_index_and_agree_with_topk():
    Nq, Ng, H = 48, 600, 16
    q, v = _tied_vectors(Nq, Ng, H, seed=3)
    ql = (torch.arange(Nq) * 7 % 30).to(DEV)
    gl = (torch.arange(Ng) % 30).to(DEV)
    gl[[2, 5, 77, 299]] = torch.tensor([0, 1, 2, 3], device=DEV)  # equal rows, different labels
    for labels in ((None, None), (ql, gl)):
        with torch.no_grad():
            r = retrieval.ranks(q, v, *labels)
            dense = _dense(q, v)
        assert torch.equal(r, retrieval.ranks_from_scores(dense, *labels))
        lab = [None if x is None else x.cpu().numpy() for x in labels]
        assert np.array_equal(r.cpu().numpy(), host_ranks(dense.cpu().numpy(), *lab))
        qlab = np.arange(Nq) if lab[0] is None else lab[0]
        glab = np.arange(Ng) if lab[1] is None else lab[1]
        for k in (1, 10, 256):
            _, idx = retrieval.topk(q, v, k)
            hit = glab[idx.cpu().numpy()] == qlab[:, None]
            for i in range(Nq):
                first = np.flatnonzero(hit[i])
                if r[i] < k:
                    assert first.size and first[0] == r[i], (k, i)
                else:
                    assert first.size == 0, (k, i)
    assert int((dense[:, 100:140] == dense[:, 100:101]).all()) == 1  # the ties are there


def test_repeats_streams_reserved_sms_and_graph_replay(pairs):
    q, g, ql, gl = pairs(24, 40000, 768, "many_gallery", seed=11)
    with torch.no_grad():
        ref = retrieval.ranks(q, g, ql, gl)
        assert torch.equal(retrieval.ranks(q, g, ql, gl), ref)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            got = retrieval.ranks(q, g, ql, gl)
        torch.cuda.current_stream().wait_stream(side)
        assert torch.equal(got, ref)
        rt.reserve_sms(100)  # fewer SMs: another gallery split
        try:
            assert torch.equal(retrieval.ranks(q, g, ql, gl), ref)
        finally:
            rt.reserve_sms(0)
        # the two kernels on ranges built in advance, captured once and replayed
        perm, lo, hi = (x.to(ops.I32) for x in retrieval._positive_ranges("ranks", ql, gl))
        out = torch.empty_like(ref)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):  # warm-up outside the capture
            ops.sim_rank(q, g, *ops.sim_best_positive(q, g, perm, lo, hi))
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out.copy_(ops.sim_rank(q, g, *ops.sim_best_positive(q, g, perm, lo, hi)))
        for _ in range(2):
            out.zero_()
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref)


def test_ranks_from_scores_on_cross_encoder_logits():
    W, F = 12, 10
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=2,
                            max_words=W, max_frames=F)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=5)).eval()
    N = 24
    batch = synth.make_batch(cfg, seed=6, b=N)
    ids, types, am = (batch[k].to(DEV) for k in ("input_ids", "token_type_ids", "attention_mask"))
    video, vm = batch["video"].to(DEV), batch["video_mask"].to(DEV)
    with torch.no_grad():
        seq, vis = model.get_sequence_visual_output(ids, types, am, video, vm)
        logits = model.get_similarity_logits(seq, vis, am, vm).float().contiguous()
    assert logits.shape == (N, N)
    host = logits.cpu().numpy()
    assert np.array_equal(retrieval.ranks_from_scores(logits).cpu().numpy(), host_ranks(host))
    gl = (torch.arange(N) // 3).to(DEV)  # three texts per video: video-to-text with three positives
    got = retrieval.ranks_from_scores(logits.t().contiguous()[::3].contiguous(), torch.arange(N // 3, device=DEV), gl)
    assert np.array_equal(got.cpu().numpy(), host_ranks(host.T[::3], np.arange(N // 3), gl.cpu().numpy()))


def test_ft_joint_end_to_end():
    W, F, N = 16, 12, 96
    cfg = synth.task_config(mode="ft_joint", batch_size=2, text_layers=2, visual_layers=1, cross_layers=1,
                            max_words=W, max_frames=F)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=7)).eval()
    batch = synth.make_batch(cfg, seed=8, b=N)
    ids, types, am = (batch[k].to(DEV) for k in ("input_ids", "token_type_ids", "attention_mask"))
    video, vm = batch["video"].to(DEV), batch["video_mask"].to(DEV)
    with torch.no_grad():
        t = retrieval.embed_texts(model, ids, am, types)
        v = retrieval.embed_videos(model, video, vm)
        t2v, v2t = retrieval.ranks(t, v), retrieval.ranks(v, t)
        dense = _dense(t, v)
    assert torch.equal(t2v, retrieval.ranks_from_scores(dense))
    assert torch.equal(v2t, retrieval.ranks_from_scores(dense.t().contiguous()))
    for r, x in ((t2v, dense), (v2t, dense.t())):
        x = x.cpu().numpy()
        ind = reference_ind(x)
        assert len(ind) == N  # tie-free
        m = retrieval.rank_metrics(r)
        for k in (1, 5, 10):
            assert m["R%d" % k] == float(np.sum(ind < k)) / len(ind)
        assert m["MR"] == np.median(ind) + 1 and np.array_equal(r.cpu().numpy(), ind)


def test_a_dense_matrix_of_more_than_2_27_entries():
    """SimMatmulFn launches a warp per entry: past 2^27 entries the thread index needs 64 bits"""
    g = torch.Generator(device="cuda").manual_seed(12)
    q = torch.randn((1200, 128), device=DEV, generator=g)
    v = torch.randn((120000, 128), device=DEV, generator=g)
    with torch.no_grad():
        dense = _dense(q, v)
        assert torch.equal(retrieval.ranks(q, v), retrieval.ranks_from_scores(dense))
        s, i = retrieval.topk(q, v, 5)
        assert torch.equal(s, dense.gather(1, i))
        assert torch.equal(dense[-1, -3:], _dense(q[-1:], v[-3:])[0])


def test_errors_on_the_device():
    q = torch.randn(4, 8, device=DEV)
    with pytest.raises(ValueError, match="1 queries have no positive"):
        retrieval.ranks(q, q, torch.tensor([0, 1, 2, 9], device=DEV), torch.arange(4, device=DEV))
    with pytest.raises(ValueError, match="no positive"):
        retrieval.ranks_from_scores(_dense(q, q), torch.tensor([0, 1, 2, 9], device=DEV), torch.arange(4, device=DEV))
    assert retrieval.ranks(q[:0], q).shape == (0,)
