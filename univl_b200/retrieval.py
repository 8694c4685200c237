"""Retrieval over galleries too large for the dense Nt x Nv evaluation: shortlist with the mean-pooled (dual-encoder)
similarity, re-rank the shortlisted pairs with a cross encoder.

  topk_similarity  the k best videos per text by UniVL._mean_pool_similarity (reference modeling.py:327-339, :385-389),
                   exactly: the scores carry the similarity matrix's bits, the order is score descending then video
                   index ascending, and the [Nt, Nv] matrix is never formed (csrc/retrieval.cu).
  score_pairs      the cross-encoder logit of listed (text, video) pairs only, equal bit for bit to the same entries of
                   the dense evaluation's get_similarity_logits under the same UNIVL_EVAL_LAYOUT / UNIVL_EVAL_PRECISION.
  search           the two composed: top k_shortlist by the first model, re-ranked by the second.

Inputs are what get_sequence_visual_output returns: sequence_output [Nt, W, H], visual_output [Nv, F, H] and the int64
masks attention_mask [Nt, W], video_mask [Nv, F].

A gallery can also be indexed as one pooled vector per row, encoded once and searched later:

  embed_texts / embed_videos  the text and video vectors _mean_pool_similarity multiplies, fp32 [N, H], from the
                              text (or visual) encoder alone, run on each row's valid tokens only
  topk                        the exact top k of stored query vectors against stored gallery vectors, in either
                              direction (text-to-video or video-to-text)

and scored against ground truth at gallery scale, without the similarity matrix:

  ranks                       each query's exact rank of its first positive (labels: many positives per query)
  ranks_from_scores           the same rule on a dense score matrix the caller already has (cross encoders)
  rank_metrics                R@1/5/10, median and mean rank of those ranks
"""
import numpy as np
import torch

from . import ops
from . import runtime as rt
from .modules import modeling
from .modules.modeling import _flat, eval_layout, eval_precision
from .modules.transformer import _layer_params


def _inputs(model, sequence_output, visual_output, attention_mask, video_mask):
    seq2d = sequence_output.to(torch.bfloat16).reshape(-1, sequence_output.shape[-1]).contiguous()
    vis2d = visual_output.to(torch.bfloat16).reshape(-1, visual_output.shape[-1]).contiguous()
    return seq2d, vis2d, _flat(attention_mask), _flat(video_mask)


def topk_similarity(model, sequence_output, visual_output, attention_mask, video_mask, k):
    """-> (scores fp32 [Nt, k], index int64 [Nt, k]): for each text row the k videos with the largest mean-pooled
    similarity (L2-normalised unless task_config.use_mil, as the model's own), score descending, ties by lower video
    index.  scores[i, j] has the bits of _mean_pool_similarity(...)[i, index[i, j]].  1 <= k <= min(256, Nv)."""
    with rt.use_model(model, model._device()), torch.no_grad():
        seq2d, vis2d, am, vm = _inputs(model, sequence_output, visual_output, attention_mask, video_mask)
        l2 = model.task_config.use_mil is False
        n_t, W = am.shape
        n_v, F = vm.shape
        text = ops.MeanPoolFn.apply(seq2d, am, n_t, W, True, False, l2)
        video = ops.MeanPoolFn.apply(vis2d, vm, n_v, F, False, True, l2)
        scores, index = ops.sim_topk(text, video, k)
        return scores, index.long()


def _host_index(x, n, name):
    """a 1-D integer index list (tensor or array-like) checked on the host against [0, n) -> int64 numpy"""
    if isinstance(x, torch.Tensor):
        if x.dtype not in (torch.int32, torch.int64):
            raise ValueError("%s must be int32 or int64, got %s" % (name, x.dtype))
        a = x.detach().cpu().numpy()
    else:
        a = np.asarray(x)
        if a.size and a.dtype.kind not in "iu":
            raise ValueError("%s must hold integers, got %s" % (name, a.dtype))
    if a.ndim != 1:
        raise ValueError("%s must be 1-D, got shape %s" % (name, tuple(a.shape)))
    a = a.astype(np.int64)
    if a.size and (a.min() < 0 or a.max() >= n):
        raise ValueError("%s has entries outside [0, %d)" % (name, n))
    return a


def _pair_chunks(cost, budget):
    """consecutive list ranges [a, b) of at most `budget` summed cost (at least one pair each)"""
    c = np.concatenate([[0], np.cumsum(cost)])
    out, a = [], 0
    while a < cost.size:
        b = int(np.searchsorted(c, c[a] + budget, side="right")) - 1
        b = min(cost.size, max(a + 1, b))
        out.append((a, b))
        a = b
    return out


def score_pairs(model, sequence_output, visual_output, attention_mask, video_mask, text_index, video_index):
    """-> fp32 [P]: the cross-encoder similarity logit of pair p = (text row text_index[p], video row video_index[p]),
    equal bit for bit to get_similarity_logits(...)[text_index[p], video_index[p]] of the dense evaluation with the
    same UNIVL_EVAL_LAYOUT and UNIVL_EVAL_PRECISION (read on every call), including its fallback to the padded layout
    when any text row's attention_mask[i, 0] is 0.  Lists may be unsorted, repeat pairs or be empty; indices are
    checked on the host (ValueError).  Evaluation only: model.eval() and no gradients (RuntimeError otherwise).
    Pairs are scored in tiles of at most EVAL_PAIR_TOKENS tokens."""
    if model.training or torch.is_grad_enabled():
        raise RuntimeError("score_pairs: call model.eval() and run under torch.no_grad()")
    if model.cross is None or not (model._stage_two or model.train_sim_after_cross):
        raise ValueError("score_pairs needs a cross-encoder model (stage two, or train_sim_after_cross)")
    (Nt, W), (Nv, F) = _flat(attention_mask).shape, _flat(video_mask).shape
    ti = _host_index(text_index, Nt, "text_index")
    vi = _host_index(video_index, Nv, "video_index")
    if ti.size != vi.size:
        raise ValueError("text_index and video_index differ in length (%d vs %d)" % (ti.size, vi.size))
    with rt.use_model(model, model._device()):
        seq2d, vis2d, am, vm = _inputs(model, sequence_output, visual_output, attention_mask, video_mask)
        out = torch.empty(ti.size, dtype=torch.float32, device=seq2d.device)
        if ti.size == 0:
            return out
        cross = model.cross
        fp8 = eval_precision() == "fp8" and len(cross.encoder.layer) > 1
        qw = cross.fp8_eval_weights() if fp8 else None
        packing = ops.PairPacking(am, vm) if eval_layout() == "packed" else None
        if packing is not None and not packing.token0_valid:
            packing = None
        x, qkv = cross.first_layer_source_rows(seq2d, vis2d, Nt, W, Nv, F)
        ti_d = torch.from_numpy(ti.astype(np.int32)).to(seq2d.device)
        vi_d = torch.from_numpy(vi.astype(np.int32)).to(seq2d.device)
        if packing is not None:
            cost = np.asarray(packing.len_t, dtype=np.int64)[ti] + np.asarray(packing.len_v, dtype=np.int64)[vi]
        else:
            cost = np.full(ti.size, W + F, dtype=np.int64)
        for a, b in _pair_chunks(cost, modeling.EVAL_PAIR_TOKENS):
            if packing is not None:
                seqs = packing.pairs(ti_d[a:b], vi_d[a:b])
                first = cross.encode_pairs_first_token_eval_packed(x, qkv, Nt * W, seqs, qw)
            else:
                first = cross.encode_pairs_first_token_eval_list(x, qkv, am, vm, ti_d[a:b], vi_d[a:b], qw)
            u = cross.pooler.pre_activation(first, b - a, 1)
            out[a:b] = ops.PoolerSimFn.apply(u, model.similarity_dense.weight, model.similarity_dense.bias)
        return out


def search(shortlist_model, rerank_model, sequence_output, visual_output, attention_mask, video_mask, k_shortlist, k,
           rerank_sequence_output=None, rerank_visual_output=None):
    """-> (scores fp32 [Nt, k], index int64 [Nt, k]): for each text row, the top k_shortlist videos by
    topk_similarity(shortlist_model, ...) re-scored by score_pairs(rerank_model, ...), the k best by that score, ties
    kept in shortlist order.  The two models may be one object.  rerank_sequence_output / rerank_visual_output: the
    re-ranking model's own encoder outputs when its encoders differ from the shortlist model's (the masks are shared);
    by default both stages read sequence_output / visual_output.  1 <= k <= k_shortlist."""
    if not 1 <= k <= k_shortlist:
        raise ValueError("search: need 1 <= k <= k_shortlist, got k=%r k_shortlist=%r" % (k, k_shortlist))
    _, short = topk_similarity(shortlist_model, sequence_output, visual_output, attention_mask, video_mask, k_shortlist)
    Nt = short.shape[0]
    ti = torch.arange(Nt, device=short.device).repeat_interleave(k_shortlist)
    seq = sequence_output if rerank_sequence_output is None else rerank_sequence_output
    vis = visual_output if rerank_visual_output is None else rerank_visual_output
    with torch.no_grad():
        scores = score_pairs(rerank_model, seq, vis, attention_mask, video_mask, ti, short.reshape(-1))
    scores, order = torch.sort(scores.view(Nt, k_shortlist), dim=1, descending=True, stable=True)
    return scores[:, :k].contiguous(), short.gather(1, order[:, :k])


def _check_eval(model, what):
    if model.training or torch.is_grad_enabled():
        raise RuntimeError("%s: call model.eval() and run under torch.no_grad()" % what)


def _check_cuda(what, *tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("univl_b200: %s needs CUDA tensors (no CPU path)" % what)


class RowPacking:
    """The valid tokens of the N rows of a [N, S] mask (any dtype; nonzero = valid, any pattern), cut into chunks of
    consecutive rows of at most `budget` valid tokens and at most ROW_SPAN * budget padded tokens each (at least one
    row per chunk).  The second bound caps the rows of a chunk, which the valid-token budget alone does not: rows
    without a valid token cost no budget, and chunk() builds per-padded-token index arrays (int32) over its rows.  At
    a packed fraction of 1 / ROW_SPAN or more, only the valid-token budget cuts.  One device-to-host copy: the per-row
    counts.
      counts   host int64 array [N]
      chunks   list of row ranges (a, b)
      max_len  the longest row of the whole call: every chunk passes it to the attention, so which attention kernel a
               row runs on does not depend on the chunking"""

    ROW_SPAN = 8

    def __init__(self, mask, budget):
        self.valid = mask.reshape(-1, mask.shape[-1]) != 0
        self.S = self.valid.shape[1]
        self.counts = self.valid.sum(1).cpu().numpy().astype(np.int64)
        cap = max(1, self.ROW_SPAN * budget // max(1, self.S))
        self.chunks = [(x, min(b, x + cap)) for a, b in _pair_chunks(self.counts, budget) for x in range(a, b, cap)]
        self.max_len = int(self.counts.max(initial=0))

    def chunk(self, a, b):
        """rows [a, b) -> (idx, cu, seqs): idx int32 the valid tokens (i - a) * S + s in row then position order, cu
        int32 [b - a + 1] the packed row offsets, seqs their ops.VarlenSeqs (packed addressing)"""
        valid = self.valid[a:b]
        idx = ops._valid_rows(valid, int(self.counts[a:b].sum()))
        cu = ops._exclusive_cumsum(valid.sum(1)).to(ops.I32)
        return idx, cu, ops.VarlenSeqs(cu, idx.numel(), self.max_len)


def _no_rows(like):
    return torch.empty((0, like.shape[1]), dtype=torch.bfloat16, device=like.device)


def _encode_packed(layers, x, seqs):
    for layer in layers:
        x = ops.encoder_layer_eval_packed(x, seqs, _layer_params(layer))
    return x


def embed_texts(model, input_ids, attention_mask, token_type_ids=None):
    """-> fp32 [Nt, H]: the text vectors of UniVL._mean_pool_similarity (reference modeling.py:327-339, :386-388):
    the text encoder's output mean-pooled over the valid tokens but token 0, L2-normalised unless
    task_config.use_mil.  The encoder runs on each row's valid tokens alone (attention_mask != 0, any pattern), each
    at its original position; no visual encoder runs.  A row without a pooled token gives what the padded pooling
    gives (0 / 0).  input_ids, attention_mask (and token_type_ids) are [Nt, W] (or [..., W], flattened as the model
    does) CUDA tensors.  Evaluation only: model.eval() under torch.no_grad() (RuntimeError otherwise).  Rows are
    encoded in chunks of at most modeling.EMBED_TOKENS valid tokens; a row's vector does not depend on the chunking."""
    _check_eval(model, "embed_texts")
    ids, am = _flat(input_ids), _flat(attention_mask)
    if ids.shape != am.shape:
        raise ValueError("embed_texts: input_ids %s and attention_mask %s differ in shape"
                         % (tuple(ids.shape), tuple(am.shape)))
    types = None if token_type_ids is None else _flat(token_type_ids)
    if types is not None and types.shape != ids.shape:
        raise ValueError("embed_texts: token_type_ids %s and input_ids %s differ in shape"
                         % (tuple(types.shape), tuple(ids.shape)))
    ids, types = ids.long().contiguous(), (None if types is None else types.long().contiguous())
    emb = model.bert.embeddings
    W = ids.shape[1]
    if not 0 < W <= emb.position_embeddings.weight.shape[0]:
        raise ValueError("embed_texts: %d tokens per row, the position table holds %d"
                         % (W, emb.position_embeddings.weight.shape[0]))
    _check_cuda("embed_texts", ids, am, types)
    l2 = model.task_config.use_mil is False
    with rt.use_model(model, model._device()):
        rows = RowPacking(am, modeling.EMBED_TOKENS)
        out = torch.empty((ids.shape[0], emb.word_embeddings.weight.shape[1]), dtype=torch.float32, device=ids.device)
        for a, b in rows.chunks:
            idx, cu, seqs = rows.chunk(a, b)
            if idx.numel() == 0:  # no valid token in the chunk: the pooling alone gives its rows' vectors
                out[a:b] = ops.meanpool_packed(_no_rows(out), cu, idx, W, True, False, l2)
                continue
            x = ops.embed_text_packed(ids[a:b], None if types is None else types[a:b], idx, W,
                                      emb.word_embeddings.weight, emb.position_embeddings.weight,
                                      emb.token_type_embeddings.weight, emb.LayerNorm.weight, emb.LayerNorm.bias)
            x = _encode_packed(model.bert.encoder.layer, x, seqs)
            out[a:b] = ops.meanpool_packed(x, cu, idx, W, True, False, l2)
        return out


def embed_videos(model, video, video_mask):
    """-> fp32 [Nv, H]: the video vectors of UniVL._mean_pool_similarity: NormalizeVideo, the visual encoder and the
    mean over the valid frames (video_mask != 0, any pattern; a row without one gives the zero vector), L2-normalised
    unless task_config.use_mil, computed on the valid frames alone, each at its original position; no text encoder
    runs.  video: fp32 or fp64 [Nv, F, video_dim] (or [..., F, video_dim]), video_mask [Nv, F], CUDA tensors.  A
    contiguous fp32 video is read in place; of any other only the valid frames of a chunk are copied (to fp32).
    Evaluation only, chunked, and independent of the chunking as embed_texts."""
    _check_eval(model, "embed_videos")
    if video.dtype not in (torch.float32, torch.float64):
        raise ValueError("embed_videos: video must be float32 or float64, got %s" % video.dtype)
    if video.dim() < 3:
        raise ValueError("embed_videos: video must be [N, F, video_dim], got shape %s" % (tuple(video.shape),))
    D = model.task_config.video_dim
    v = video.reshape(-1, video.shape[-2], video.shape[-1])
    vm = _flat(video_mask)
    if v.shape[-1] != D or tuple(v.shape[:2]) != tuple(vm.shape):
        raise ValueError("embed_videos: video %s does not match video_mask %s and video_dim %d"
                         % (tuple(video.shape), tuple(video_mask.shape), D))
    emb = model.visual.embeddings
    F = vm.shape[1]
    if not 0 < F <= emb.position_embeddings.weight.shape[0]:
        raise ValueError("embed_videos: %d frames per row, the position table holds %d"
                         % (F, emb.position_embeddings.weight.shape[0]))
    _check_cuda("embed_videos", video, video_mask)
    norm = model.normalize_video.visual_norm2d
    l2 = model.task_config.use_mil is False
    with rt.use_model(model, model._device()):
        rows = RowPacking(vm, modeling.EMBED_TOKENS)
        w16 = rt.current().bf16(emb.word_embeddings.weight)
        out = torch.empty((v.shape[0], w16.shape[0]), dtype=torch.float32, device=v.device)
        for a, b in rows.chunks:
            idx, cu, seqs = rows.chunk(a, b)
            if idx.numel() == 0:
                out[a:b] = ops.meanpool_packed(_no_rows(out), cu, idx, F, False, True, l2)
                continue
            if v.dtype == torch.float32 and v[a:b].is_contiguous():  # the kernel reads the valid frames in place
                rows2d, ridx = v[a:b].view(-1, D), idx
            else:  # copy the valid frames alone to fp32 (an exact conversion): at most EMBED_TOKENS rows
                li = idx.long()
                rows2d = v[a + li // F, li % F].float()
                ridx = torch.arange(idx.numel(), dtype=ops.I32, device=idx.device)
            x = ops.video_norm_rows(rows2d, ridx, norm.weight, norm.bias)
            del rows2d, ridx
            x = ops.linear_fwd(x, w16, emb.word_embeddings.bias)
            x = ops.embed_src_packed(x, idx, F, emb.position_embeddings.weight, emb.LayerNorm.weight,
                                     emb.LayerNorm.bias)
            x = _encode_packed(model.visual.encoder.layer, x, seqs)
            out[a:b] = ops.meanpool_packed(x, cu, idx, F, False, True, l2)
        return out


def _check_vectors(what, queries, gallery):
    """the stored-vector arguments of topk / ranks, checked on the host"""
    for t, name in ((queries, "queries"), (gallery, "gallery")):
        if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.dtype != torch.float32:
            raise ValueError("%s: %s must be a 2-D float32 tensor" % (what, name))
    if queries.shape[1] != gallery.shape[1] or queries.shape[1] % 4:
        raise ValueError("%s: queries %s and gallery %s need the same width, a multiple of 4"
                         % (what, tuple(queries.shape), tuple(gallery.shape)))
    if queries.device != gallery.device:
        raise ValueError("%s: queries on %s and gallery on %s: both must be on one device"
                         % (what, queries.device, gallery.device))


def topk(queries, gallery, k):
    """-> (scores fp32 [Nq, k], index int64 [Nq, k]): for each stored query vector the k gallery rows with the largest
    dot product, score descending, ties by lower gallery index (univl_sim_topk).  Text-to-video:
    topk(embed_texts(...), embed_videos(...), k); video-to-text: topk(embed_videos(...), embed_texts(...), k).  Every
    score has the bits of _mean_pool_similarity(...)[i, j] (text-to-video) or [j, i] (video-to-text) of the same
    vectors.  queries [Nq, H] and gallery [Ng, H]: fp32 CUDA tensors on one device, H a multiple of 4;
    1 <= k <= min(256, Ng)."""
    _check_vectors("topk", queries, gallery)
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(256, gallery.shape[0]):
        raise ValueError("topk: need 1 <= k <= min(256, %d gallery rows), got %r" % (gallery.shape[0], k))
    _check_cuda("topk", queries, gallery)
    if queries.shape[0] == 0:
        return (torch.empty((0, k), dtype=torch.float32, device=queries.device),
                torch.empty((0, k), dtype=torch.int64, device=queries.device))
    scores, index = ops.sim_topk(queries, gallery, k)
    return scores, index.long()


# Ground-truth ranks.  A query's gallery is ranked in topk's order (score descending, then gallery index ascending); its
# positives are the gallery rows that share its label, and its rank is the 0-based position of its first positive in
# that order: the number of gallery rows ranked above its best positive, every one of them a negative.


def _labels(what, query_labels, gallery_labels, Nq, Ng, device):
    """-> (query labels, gallery labels), int64 on `device`: each defaults to arange (query i's positive is gallery row
    i, which needs Nq <= Ng when neither is given); given labels are 1-D int32 / int64 tensors on `device`"""
    if query_labels is None and gallery_labels is None and Nq > Ng:
        raise ValueError("%s: without labels query i's positive is gallery row i, which needs Nq <= Ng (got %d > %d)"
                         % (what, Nq, Ng))
    out = []
    for x, n, name in ((query_labels, Nq, "query_labels"), (gallery_labels, Ng, "gallery_labels")):
        if x is None:
            out.append(torch.arange(n, device=device))
            continue
        if not isinstance(x, torch.Tensor) or x.dtype not in (torch.int32, torch.int64) or x.dim() != 1:
            raise ValueError("%s: %s must be a 1-D int32 or int64 tensor" % (what, name))
        if x.shape[0] != n:
            raise ValueError("%s: %s holds %d labels for %d rows" % (what, name, x.shape[0], n))
        if x.device != device:
            raise ValueError("%s: %s is on %s, the vectors on %s" % (what, name, x.device, device))
        out.append(x.long())
    return out


def _no_positive(what, missing):
    """one device-to-host read: the count of queries without a positive"""
    n = int(missing.sum())
    if n:
        raise ValueError("%s: %d queries have no positive (no gallery row shares their label)" % (what, n))


def _positive_ranges(what, query_labels, gallery_labels):
    """-> (perm, lo, hi): query i's positives are the gallery rows perm[lo[i]:hi[i]] (ascending), from a stable sort
    of the gallery labels and a search of it, on the labels' device; ValueError for a query without a positive"""
    sorted_labels, perm = torch.sort(gallery_labels, stable=True)
    lo = torch.searchsorted(sorted_labels, query_labels, side="left")
    hi = torch.searchsorted(sorted_labels, query_labels, side="right")
    _no_positive(what, lo == hi)
    return perm, lo, hi


def ranks(queries, gallery, query_labels=None, gallery_labels=None):
    """-> int64 [Nq]: each stored query's rank, the 0-based position of its best positive in topk's order, computed
    exactly on the device without the [Nq, Ng] matrix (univl_sim_best_positive, univl_sim_rank): rank < k exactly
    when a positive is in topk(queries, gallery, k), and the first one sits at position rank.  Every score compared has
    the bits of _mean_pool_similarity's entry for the same vectors.  Text-to-video: ranks(embed_texts(...),
    embed_videos(...)); video-to-text: the two swapped.  queries and gallery as topk takes them.  Labels: 1-D int32 /
    int64 tensors on the vectors' device, [Nq] and [Ng]; a query's positives are the gallery rows with its label, and
    a missing side defaults to arange (so with neither, query i's positive is gallery row i, which needs Nq <= Ng).  A
    query without a positive raises ValueError, after one device-to-host read of their count."""
    _check_vectors("ranks", queries, gallery)
    Nq, Ng = queries.shape[0], gallery.shape[0]
    ql, gl = _labels("ranks", query_labels, gallery_labels, Nq, Ng, queries.device)
    _check_cuda("ranks", queries, gallery)
    if Nq == 0:
        return torch.empty((0,), dtype=torch.int64, device=queries.device)
    perm, lo, hi = _positive_ranges("ranks", ql, gl)
    best_s, best_i = ops.sim_best_positive(queries, gallery, perm.to(ops.I32), lo.to(ops.I32), hi.to(ops.I32))
    return ops.sim_rank(queries, gallery, best_s, best_i)


def ranks_from_scores(scores, query_labels=None, gallery_labels=None):
    """-> int64 [Nq]: ranks' rule on a dense fp32 [Nq, Ng] CUDA matrix the caller already has (a cross encoder's
    get_similarity_logits, or ops.SimMatmulFn of stored vectors), with torch ops on the device.  Labels and errors as
    ranks."""
    if not isinstance(scores, torch.Tensor) or scores.dim() != 2 or scores.dtype != torch.float32:
        raise ValueError("ranks_from_scores: scores must be a 2-D float32 tensor")
    Nq, Ng = scores.shape
    ql, gl = _labels("ranks_from_scores", query_labels, gallery_labels, Nq, Ng, scores.device)
    _check_cuda("ranks_from_scores", scores)
    pos = ql[:, None] == gl[None, :]
    _no_positive("ranks_from_scores", ~pos.any(1))
    best_s = torch.where(pos, scores, float("-inf")).amax(1, keepdim=True)
    best_i = (pos & (scores == best_s)).int().argmax(1, keepdim=True)  # the first positive with the best score
    j = torch.arange(Ng, device=scores.device)[None, :]
    return ((scores > best_s) | ((scores == best_s) & (j < best_i))).sum(1)


def rank_metrics(ranks):
    """-> {"R1", "R5", "R10", "MR", "MeanR"} of 0-based ranks (a 1-D tensor or array-like, not empty), as the
    reference's compute_metrics defines them: R@K the fraction of ranks below K, MR = median + 1 (numpy's median, the
    mean of the two middle ranks for an even count) and MeanR = mean + 1."""
    r = ranks.detach().cpu().numpy() if isinstance(ranks, torch.Tensor) else np.asarray(ranks)
    if r.ndim != 1 or r.size == 0:
        raise ValueError("rank_metrics: ranks must be 1-D and not empty, got shape %s" % (r.shape,))
    out = {"R%d" % k: float(np.mean(r < k)) for k in (1, 5, 10)}
    out["MR"] = float(np.median(r)) + 1
    out["MeanR"] = float(np.mean(r)) + 1
    return out
