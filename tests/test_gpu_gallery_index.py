"""GPU: gallery indexing on valid tokens (retrieval.embed_texts / embed_videos / topk).  Each packed stage against the
padded kernels bit for bit, the pooled vectors against pooling get_sequence_visual_output and the fp32 CPU oracle, the
search against topk_similarity and the similarity matrix, and the independence of the chunking."""
import pytest
import torch
import torch.nn.functional as Fn

from oracle import synth
from oracle import univl_oracle as O
from tests.model_util import build_model
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200 import runtime as rt
from univl_b200.modules import modeling

pytestmark = pytest.mark.gpu

DEV = "cuda"
# Packed vs padded encoders: the same GEMM, LayerNorm and FFN kernels run on every valid row, and a padded key adds
# exactly 0 to a row's softmax sums, so the two differ only in the order of the fp32 sums inside attention (a context
# element may round to a neighbouring bf16 value).  The pooled vectors are L2-normalised, entries ~ 768^-0.5.
PACKED_VS_PADDED = 1e-2
# Against the fp32 oracle the packed error may exceed the padded path's by the noise of that reordering
ORACLE_SLACK = 1.25


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _model(W, F, use_mil=False, seed=0):
    cfg = synth.task_config(mode="ft_joint", batch_size=2, text_layers=2, visual_layers=1, cross_layers=1,
                            max_words=W, max_frames=F, use_mil=use_mil)
    sd = synth.make_state_dict(cfg, seed=seed)
    return cfg, sd, build_model(cfg, sd=sd).eval()


def _inputs(sd, Nt, W, Nv, F, seed, video_dtype=torch.float32):
    """ragged masks of every kind: prefixes, scattered (token 0 sometimes off), [CLS][SEP]-only texts, a text with
    token 0 alone (no pooled token), all-padded clips; row 0 of each is full"""
    g = _g(seed)
    vocab = sd["bert.embeddings.word_embeddings.weight"].shape[0]
    ids = torch.randint(0, vocab, (Nt, W), generator=g)
    types = torch.randint(0, 2, (Nt, W), generator=g)
    lt = torch.randint(1, W + 1, (Nt,), generator=g)
    am = (torch.arange(W)[None] < lt[:, None]).long()
    am[1::3] = (torch.rand(am[1::3].shape, generator=g) < 0.5).long()
    am[0] = 1
    if Nt > 3 and W > 1:
        am[2] = 0
        am[2, :2] = 1  # [CLS] [SEP]
    if Nt > 5:
        am[5] = 0
        am[5, 0] = 1  # nothing to pool: 0 / 0, as the padded pooling
    lv = torch.randint(1, F + 1, (Nv,), generator=g)
    vm = (torch.arange(F)[None] < lv[:, None]).long()
    vm[1::3] = (torch.rand(vm[1::3].shape, generator=g) < 0.5).long()
    vm[0] = 1
    if Nv > 2:
        vm[-1] = 0
    video = torch.randn((Nv, F, synth.VIDEO_DIM), generator=g, dtype=torch.float64).to(video_dtype)
    return [t.to(DEV) for t in (ids, types, am, video, vm)]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _padded_vectors(model, ids, types, am, video, vm):
    """get_sequence_visual_output, then MeanPoolFn: the vectors _mean_pool_similarity multiplies"""
    l2 = model.task_config.use_mil is False
    with torch.no_grad():
        seq, vis = model.get_sequence_visual_output(ids, types, am, video, vm)
    Nt, W = am.shape
    Nv, F = vm.shape
    seq2d, vis2d = seq.reshape(-1, seq.shape[-1]), vis.reshape(-1, vis.shape[-1])
    with rt.use_model(model, model._device()), torch.no_grad():
        t = ops.MeanPoolFn.apply(seq2d, am, Nt, W, True, False, l2)
        v = ops.MeanPoolFn.apply(vis2d, vm, Nv, F, False, True, l2)
    return t, v, seq, vis


def _oracle_vectors(sd, cfg, ids, types, am, video, vm, l2):
    seq = O.text_encoder(ids.cpu(), types.cpu(), am.cpu(), sd, cfg.text_num_hidden_layers)
    vis = O.visual_encoder(O.normalize_video(video.cpu(), sd), vm.cpu(), sd, cfg.visual_num_hidden_layers)
    t, v = O.mean_pool(seq, vis, am.cpu(), vm.cpu())
    if l2:
        t, v = Fn.normalize(t, dim=-1), Fn.normalize(v, dim=-1)
    return t, v


@pytest.mark.parametrize("W,F", [(16, 12), (48, 48), (300, 280)])
def test_packed_stages_equal_the_padded_kernels(W, F):
    cfg, sd, model = _model(W, F)
    ids, types, am, video, vm = _inputs(sd, 7, W, 5, F, seed=1)
    bert, visual = model.bert.embeddings, model.visual.embeddings
    norm = model.normalize_video.visual_norm2d
    with rt.use_model(model, model._device()), torch.no_grad():
        # text embedding rows
        tp = retrieval.RowPacking(am, 1 << 30)
        idx, cu, _ = tp.chunk(0, am.shape[0])
        pad = ops.EmbedTextFn.apply(ids, types, bert.word_embeddings.weight, bert.position_embeddings.weight,
                                    bert.token_type_embeddings.weight, bert.LayerNorm.weight, bert.LayerNorm.bias,
                                    0.1, False)
        got = ops.embed_text_packed(ids, types, idx, W, bert.word_embeddings.weight, bert.position_embeddings.weight,
                                    bert.token_type_embeddings.weight, bert.LayerNorm.weight, bert.LayerNorm.bias)
        assert _same_bits(got, pad[idx.long()])
        # NormalizeVideo, projection, position + LayerNorm
        vp = retrieval.RowPacking(vm, 1 << 30)
        vidx, vcu, _ = vp.chunk(0, vm.shape[0])
        v2d = video.reshape(-1, video.shape[-1])
        norm_pad = ops.VideoNormFn.apply(video, norm.weight, norm.bias).reshape(-1, video.shape[-1])
        norm_got = ops.video_norm_rows(v2d, vidx, norm.weight, norm.bias)
        assert _same_bits(norm_got, norm_pad[vidx.long()])
        w16 = rt.current().bf16(visual.word_embeddings.weight)
        # forward GEMMs (epilogue 0) never split K, so a row's projection does not depend on M: compared exactly
        proj_pad = ops.LinearFn.apply(norm_pad, visual.word_embeddings.weight, visual.word_embeddings.bias, False,
                                      False)
        proj_got = ops.linear_fwd(norm_got, w16, visual.word_embeddings.bias)
        assert _same_bits(proj_got, proj_pad[vidx.long()])
        src_pad = ops.EmbedSrcFn.apply(proj_pad, None, vm.shape[0], F, 0, 0, False, visual.position_embeddings.weight,
                                       None, visual.LayerNorm.weight, visual.LayerNorm.bias, 0.1, False)
        src_got = ops.embed_src_packed(proj_got, vidx, F, visual.position_embeddings.weight, visual.LayerNorm.weight,
                                       visual.LayerNorm.bias)
        assert _same_bits(src_got, src_pad[vidx.long()])
        # mean pool of the padded encoders' valid rows, with and without L2 normalisation
        seq = model.bert.encode(ids, types, am)
        vis = model.visual.encode(ops.VideoNormFn.apply(video, norm.weight, norm.bias), vm)
        Nt, Nv = am.shape[0], vm.shape[0]
        for l2 in (True, False):
            t_pad = ops.MeanPoolFn.apply(seq, am, Nt, W, True, False, l2)
            v_pad = ops.MeanPoolFn.apply(vis, vm, Nv, F, False, True, l2)
            assert _same_bits(ops.meanpool_packed(seq[idx.long()], cu, idx, W, True, False, l2), t_pad)
            assert _same_bits(ops.meanpool_packed(vis[vidx.long()], vcu, vidx, F, False, True, l2), v_pad)
            assert bool(torch.isnan(t_pad[5]).all()) and bool((v_pad[-1] == 0).all())


@pytest.mark.parametrize("W,F,video_dtype", [(16, 1, torch.float32), (48, 48, torch.float64),
                                             (300, 280, torch.float32)])
@pytest.mark.parametrize("use_mil", [False, True])
def test_embeddings_against_pooled_encoder_outputs_and_the_oracle(W, F, video_dtype, use_mil):
    cfg, sd, model = _model(W, F, use_mil=use_mil, seed=2)
    ids, types, am, video, vm = _inputs(sd, 7, W, 5, F, seed=3, video_dtype=video_dtype)
    with torch.no_grad():
        t = retrieval.embed_texts(model, ids, am, types)
        v = retrieval.embed_videos(model, video, vm)
    t_pad, v_pad, _, _ = _padded_vectors(model, ids, types, am, video, vm)
    t_ref, v_ref = _oracle_vectors(sd, cfg, ids, types, am, video, vm, not use_mil)
    assert t.dtype == v.dtype == torch.float32 and t.shape == (7, 768) and v.shape == (5, 768)
    # the row without a pooled text token is 0 / 0 in all three; an all-padded clip is exactly zero
    assert bool(torch.isnan(t[5]).all()) and bool(torch.isnan(t_pad[5]).all())
    assert bool((v[-1] == 0).all()) and bool((v_pad[-1] == 0).all())
    keep = torch.arange(7) != 5
    margins = {}
    for name, got, pad, ref in (("text", t[keep], t_pad[keep], t_ref[keep]), ("video", v, v_pad, v_ref)):
        assert bool(torch.isfinite(got).all())
        d = float((got - pad).abs().max())
        e_packed = float((got.cpu().double() - ref.double()).abs().max())
        e_padded = float((pad.cpu().double() - ref.double()).abs().max())
        margins[name] = (d, e_packed, e_padded)
        assert d <= PACKED_VS_PADDED, (name, d)
        assert e_packed <= ORACLE_SLACK * e_padded + 1e-6, (name, e_packed, e_padded)
    print("W=%d F=%d mil=%s: text |packed-padded| %.3g, |packed-oracle| %.3g, |padded-oracle| %.3g; video %.3g, "
          "%.3g, %.3g" % ((W, F, use_mil) + margins["text"] + margins["video"]))


def test_topk_equals_topk_similarity_and_the_similarity_matrix():
    W, F = 24, 20
    cfg, sd, model = _model(W, F, seed=4)
    ids, types, am, video, vm = _inputs(sd, 40, W, 60, F, seed=5)
    am[5, 1] = 1  # every text row pools at least one token: the search takes finite vectors
    t_pad, v_pad, seq, vis = _padded_vectors(model, ids, types, am, video, vm)
    k = 17
    with torch.no_grad():
        ref_s, ref_i = retrieval.topk_similarity(model, seq, vis, am, vm, k)
    s, i = retrieval.topk(t_pad, v_pad, k)
    assert i.dtype == torch.int64 and _same_bits(s, ref_s) and torch.equal(i, ref_i)
    # video-to-text: the transposed entries of _mean_pool_similarity, bit for bit
    with rt.use_model(model, model._device()), torch.no_grad():
        sim = model._mean_pool_similarity(seq.reshape(-1, 768), vis.reshape(-1, 768), am, vm)
    s2, i2 = retrieval.topk(v_pad, t_pad, k)
    assert _same_bits(s2, sim.t().gather(1, i2))
    order = torch.sort(sim.t(), dim=1, descending=True, stable=True)
    assert torch.equal(i2, order.indices[:, :k]) and _same_bits(s2, order.values[:, :k].contiguous())
    s3, i3 = retrieval.topk(v_pad, t_pad, k)
    assert _same_bits(s3, s2) and torch.equal(i3, i2)
    # the same on the stored embeddings of embed_*: scores are the dot products of those vectors
    with torch.no_grad():
        t = retrieval.embed_texts(model, ids, am, types)
        v = retrieval.embed_videos(model, video, vm)
        s4, i4 = retrieval.topk(t, v, k)
        full = ops.SimMatmulFn.apply(t, v, 1)
    assert _same_bits(s4, full.gather(1, i4))


@pytest.mark.parametrize("W,F", [(20, 16), (300, 280)])
def test_chunking_does_not_change_the_bits(W, F, monkeypatch):
    _, sd, model = _model(W, F, seed=6)
    ids, types, am, video, vm = _inputs(sd, 9, W, 8, F, seed=7, video_dtype=torch.float64)
    with torch.no_grad():
        one_t = retrieval.embed_texts(model, ids, am, types)
        one_v = retrieval.embed_videos(model, video, vm)
        for budget in (1, 37, W + 1):
            monkeypatch.setattr(modeling, "EMBED_TOKENS", budget)
            assert _same_bits(retrieval.embed_texts(model, ids, am, types), one_t), budget
            assert _same_bits(retrieval.embed_videos(model, video, vm), one_v), budget
        rt.reserve_sms(40)
        try:
            assert _same_bits(retrieval.embed_texts(model, ids, am, types), one_t)
            assert _same_bits(retrieval.embed_videos(model, video, vm), one_v)
        finally:
            rt.reserve_sms(0)


def test_fp64_and_strided_video_copy_only_the_valid_frames(monkeypatch):
    """A chunk holds at most EMBED_TOKENS valid frames, however many rows without one it spans: its fp32 copy of a
    fp64 or strided video, and its peak, stay bounded by the budget.  fp64, strided fp32 and contiguous fp32 (read in
    place) give the same bits."""
    _, sd, model = _model(16, 64, seed=10)
    Nv, F, D, budget = 600, 64, synth.VIDEO_DIM, 64
    g = _g(11)
    vm = torch.zeros((Nv, F), dtype=torch.long)
    vm[::5, 3] = 1  # one valid frame in every fifth clip, the others empty
    vm[0] = 1
    vm = vm.to(DEV)
    fp64 = torch.randn((Nv, F, D), generator=g, dtype=torch.float64).to(DEV)
    strided = torch.empty((Nv, F, 2 * D), dtype=torch.float32, device=DEV)[..., :D]
    strided.copy_(fp64)  # the same rounding to fp32 as fp64.float()
    assert not strided.is_contiguous()
    monkeypatch.setattr(modeling, "EMBED_TOKENS", budget)
    with torch.no_grad():
        ref = retrieval.embed_videos(model, fp64.float().contiguous(), vm)
        for video in (fp64, strided):
            retrieval.embed_videos(model, video, vm)  # warm-up: the weight arena, the allocator
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            got = retrieval.embed_videos(model, video, vm)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            assert _same_bits(got, ref), video.dtype
            # the budget alone lets a chunk span ~320 clips, whose frames in fp32 are 84 MB; the row bound keeps it
            # to 8, and only their valid frames are copied.  The fp32 result [600, 768] itself is 1.8 MB.
            print("%s: peak %.2f MiB" % (video.dtype, peak / 2 ** 20))
            assert peak < 6 * 2 ** 20, peak


def test_the_encoders_run_alone_and_only_in_evaluation(monkeypatch):
    _, sd, model = _model(16, 12, seed=8)
    ids, types, am, video, vm = _inputs(sd, 4, 16, 3, 12, seed=9)
    calls = []
    monkeypatch.setattr(model.bert, "encode", lambda *a, **k: calls.append("text"))
    monkeypatch.setattr(model.visual, "encode", lambda *a, **k: calls.append("visual"))
    monkeypatch.setattr(model.normalize_video, "forward", lambda *a, **k: calls.append("norm"))
    with torch.no_grad():
        retrieval.embed_texts(model, ids, am)
        retrieval.embed_videos(model, video, vm)
        assert calls == []
        # token_type_ids=None is type 0 everywhere
        assert _same_bits(retrieval.embed_texts(model, ids, am), retrieval.embed_texts(model, ids, am, ids * 0))
        # a mask of another dtype selects the same tokens
        assert _same_bits(retrieval.embed_videos(model, video, vm.bool()), retrieval.embed_videos(model, video, vm))
    with pytest.raises(RuntimeError):
        retrieval.embed_texts(model, ids, am)  # gradients enabled
    model.train()
    with torch.no_grad(), pytest.raises(RuntimeError):
        retrieval.embed_videos(model, video, vm)
    model.eval()
    with torch.no_grad(), pytest.raises(RuntimeError):
        retrieval.embed_texts(model, ids.cpu(), am.cpu())
    with pytest.raises(RuntimeError):
        retrieval.topk(torch.zeros(2, 8), torch.zeros(3, 8), 1)
