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
"""
import numpy as np
import torch

from . import ops
from . import runtime as rt
from .modules import modeling
from .modules.modeling import _flat, eval_layout, eval_precision


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
