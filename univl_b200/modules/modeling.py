"""UniVL orchestrator — the drop-in surface of the reference's modules/modeling.py (UniVLPreTrainedModel :39-81,
NormalizeVideo :83-92, UniVL :109-428) driving the fused sm_90a kernels.

Same constructor, `from_pretrained`, `forward` (a scalar loss in train mode, None in eval), `get_sequence_visual_output`,
`get_similarity_logits`, `decoder_caption`, sub-module names, parameter names / tying and stage flags, so the reference
drivers (main_task_retrieval.py / main_task_caption.py / main_pretrain.py) load it unchanged.  Differences a caller can
observe: hidden states are bf16 (the kernels' activation type); everything needs a CUDA device; there is no CPU path.
"""
import logging
import math
import os

import numpy as np
import torch
from torch import nn

from .. import ops
from .. import runtime as rt
from ..caption import PrefixDecodeCache, decode_cache_mode
from .module_bert import BertConfig, BertModel, BertOnlyMLMHead
from .module_cross import CrossConfig, CrossModel
from .module_decoder import DecoderConfig, DecoderModel
from .module_visual import VisualConfig, VisualModel, VisualOnlyMLMHead
from .until_module import CrossEn, LayerNorm, MaxMarginRankingLoss, MILNCELoss, PreTrainedModel

logger = logging.getLogger(__name__)

# Pair tokens (pairs x (W + F)) per tile of the cross-encoder similarity in evaluation (UniVL._cross_similarity_eval).
# A tile's memory grows linearly with it.  At this value, W = F = 48 and two cross layers, a tile's peak was 5.2 GiB of
# torch allocations (measured on an H100 80GB HBM3 at a 400 W power limit, scripts/bench_retrieval_eval.py); the eval
# path draws no stream-ordered kernel scratch.
EVAL_PAIR_TOKENS = 1 << 18

# Valid tokens per chunk of the gallery encoders (univl_b200.retrieval.embed_texts / embed_videos).  A chunk's memory
# grows linearly with it: the packed rows of one encoder layer, the fp32 copy of its valid frames when the video is
# not contiguous fp32, and index arrays over at most retrieval.RowPacking.ROW_SPAN times as many padded tokens.  A
# row's vector does not depend on it.  At this value the peak of torch allocations was 2.73 GiB, for the text and the
# visual encoder alike (measured on an H100 80GB HBM3 at a 700 W power limit, scripts/bench_gallery_index.py).
EMBED_TOKENS = 1 << 17

EVAL_PRECISIONS = ("bf16", "fp8")


def eval_precision():
    """UNIVL_EVAL_PRECISION, read on every tiled evaluation call: "bf16" (default) or "fp8", which runs the cross
    layers' dense GEMMs over the pair tokens as block-scaled e4m3 GEMMs (CrossModel.encode_pairs_first_token_eval_fp8).
    An environment variable, so that evaluation drivers pick it up unchanged."""
    value = os.environ.get("UNIVL_EVAL_PRECISION", "bf16")
    if value not in EVAL_PRECISIONS:
        raise ValueError("UNIVL_EVAL_PRECISION must be one of %s, got %r" % ("/".join(EVAL_PRECISIONS), value))
    return value


EVAL_LAYOUTS = ("padded", "packed")


def eval_layout():
    """UNIVL_EVAL_LAYOUT, read on every tiled evaluation call: "padded" (default) computes every pair at W + F tokens;
    "packed" computes pair (i, j) on text i's and video j's valid tokens alone (CrossModel.
    encode_pairs_first_token_eval_packed), under either UNIVL_EVAL_PRECISION.  Training, calls with gradients and
    micro-batched calls never read it."""
    value = os.environ.get("UNIVL_EVAL_LAYOUT", "padded")
    if value not in EVAL_LAYOUTS:
        raise ValueError("UNIVL_EVAL_LAYOUT must be one of %s, got %r" % ("/".join(EVAL_LAYOUTS), value))
    return value


class UniVLPreTrainedModel(PreTrainedModel, nn.Module):
    def __init__(self, bert_config, visual_config, cross_config, decoder_config, *inputs, **kwargs):
        super(UniVLPreTrainedModel, self).__init__(bert_config)
        self.bert_config = bert_config
        self.visual_config = visual_config
        self.cross_config = cross_config
        self.decoder_config = decoder_config
        self.bert = None
        self.visual = None
        self.cross = None
        self.decoder = None

    @classmethod
    def from_pretrained(cls, pretrained_bert_name, visual_model_name, cross_model_name, decoder_model_name,
                        state_dict=None, cache_dir=None, type_vocab_size=2, *inputs, **kwargs):
        task_config = kwargs.get("task_config")
        if task_config is not None:
            if not hasattr(task_config, "local_rank"):
                task_config.__dict__["local_rank"] = 0
            elif task_config.local_rank == -1:
                task_config.local_rank = 0
        bert_config, state_dict = BertConfig.get_config(pretrained_bert_name, cache_dir, type_vocab_size, state_dict,
                                                        task_config=task_config)
        visual_config, _ = VisualConfig.get_config(visual_model_name, cache_dir, type_vocab_size, state_dict=None,
                                                   task_config=task_config)
        cross_config, _ = CrossConfig.get_config(cross_model_name, cache_dir, type_vocab_size, state_dict=None,
                                                 task_config=task_config)
        decoder_config, _ = DecoderConfig.get_config(decoder_model_name, cache_dir, type_vocab_size, state_dict=None,
                                                     task_config=task_config)
        model = cls(bert_config, visual_config, cross_config, decoder_config, *inputs, **kwargs)
        assert model.bert is not None
        assert model.visual is not None
        if state_dict is not None:
            model = cls.init_preweight(model, state_dict, task_config=task_config)
        return model


class NormalizeVideo(nn.Module):
    """LayerNorm over the video feature dimension on fp32 (or fp64) dataloader output (reference :83-92)."""

    def __init__(self, task_config):
        super(NormalizeVideo, self).__init__()
        self.visual_norm2d = LayerNorm(task_config.video_dim)

    def forward(self, video):
        video = torch.as_tensor(video)
        if not video.is_cuda:
            raise RuntimeError("univl_b200: NormalizeVideo needs a CUDA tensor (no CPU path)")
        video = video.float().contiguous()
        video = video.view(-1, video.shape[-2], video.shape[-1])
        return ops.VideoNormFn.apply(video, self.visual_norm2d.weight, self.visual_norm2d.bias)


def show_log(task_config, info):
    if task_config is None or task_config.local_rank == 0:
        logger.warning(info)


def update_attr(target_name, target_config, target_attr_name, source_config, source_attr_name, default_value=None):
    if hasattr(source_config, source_attr_name):
        value = getattr(source_config, source_attr_name)
        if default_value is None or value != default_value:
            setattr(target_config, target_attr_name, value)
            show_log(source_config, "Set {}.{}: {}.".format(target_name, target_attr_name, value))
    return target_config


def check_attr(target_name, task_config):
    return hasattr(task_config, target_name) and task_config.__dict__[target_name]


def _flat(t):
    return t.reshape(-1, t.shape[-1]).contiguous()


def _eval_tile(Nt, Nv, S, budget):
    """(text rows, video rows) of one tile of the eval similarity: about square, at most `budget` pair tokens (at
    least one pair)"""
    pairs = max(1, budget // S)
    bv = min(Nv, max(1, math.isqrt(pairs)))
    bt = min(Nt, max(1, pairs // bv))
    return bt, min(Nv, max(1, pairs // bt))


def _packed_eval_tiles(len_t, len_v, budget):
    """Tiles (t0, t1, v0, v1) of the packed eval similarity, each at most `budget` packed pair tokens (at least one
    pair).  len_t / len_v: valid tokens of every text / video row.  Video blocks have _eval_tile's width at the mean
    pair length, capped so that one text row against a whole block fits; each block's text rows are then cut greedily,
    a tile of text rows [t0, t1) costing (v1 - v0) * sum(len_t[t0:t1]) + (t1 - t0) * sum(len_v[v0:v1]) tokens."""
    lt = np.asarray(len_t, dtype=np.int64)
    lv = np.asarray(len_v, dtype=np.int64)
    Nt, Nv = lt.size, lv.size
    if Nt == 0 or Nv == 0:
        return []
    mean = max(1, math.ceil(lt.mean() + lv.mean()))
    longest = max(1, int(lt.max() + lv.max()))
    bv = max(1, min(_eval_tile(Nt, Nv, mean, budget)[1], budget // longest))
    ct = np.concatenate([[0], np.cumsum(lt)])
    tiles = []
    for v0 in range(0, Nv, bv):
        v1 = min(Nv, v0 + bv)
        cost = (v1 - v0) * ct + int(lv[v0:v1].sum()) * np.arange(Nt + 1)  # tokens of text rows [0, t)
        t0 = 0
        while t0 < Nt:
            t1 = int(np.searchsorted(cost, cost[t0] + budget, side="right")) - 1
            t1 = min(Nt, max(t0 + 1, t1))
            tiles.append((t0, t1, v0, v1))
            t0 = t1
    return tiles


class UniVL(UniVLPreTrainedModel):
    def __init__(self, bert_config, visual_config, cross_config, decoder_config, task_config):
        super(UniVL, self).__init__(bert_config, visual_config, cross_config, decoder_config)
        self.task_config = task_config
        self.ignore_video_index = -1

        assert task_config.max_words <= bert_config.max_position_embeddings
        assert task_config.max_words <= decoder_config.max_target_embeddings
        assert task_config.max_frames <= visual_config.max_position_embeddings
        assert task_config.max_words + task_config.max_frames <= cross_config.max_position_embeddings

        self._stage_one = True
        self._stage_two = False
        if check_attr("stage_two", task_config):
            self._stage_one = False
            self._stage_two = task_config.stage_two
        show_log(task_config, "Stage-One:{}, Stage-Two:{}".format(self._stage_one, self._stage_two))

        self.train_sim_after_cross = False
        if self._stage_one and check_attr("train_sim_after_cross", task_config):
            self.train_sim_after_cross = True
            show_log(task_config, "Test retrieval after cross encoder.")

        bert_config = update_attr("bert_config", bert_config, "num_hidden_layers", task_config,
                                  "text_num_hidden_layers")
        self.bert = BertModel(bert_config)
        word_table = self.bert.embeddings.word_embeddings.weight
        position_table = self.bert.embeddings.position_embeddings.weight

        visual_config = update_attr("visual_config", visual_config, "num_hidden_layers", task_config,
                                    "visual_num_hidden_layers")
        self.visual = VisualModel(visual_config)
        visual_in_proj = self.visual.embeddings.word_embeddings.weight

        if self._stage_one is False or self.train_sim_after_cross:
            cross_config = update_attr("cross_config", cross_config, "num_hidden_layers", task_config,
                                       "cross_num_hidden_layers")
            self.cross = CrossModel(cross_config)
            if self.train_sim_after_cross is False:
                decoder_config = update_attr("decoder_config", decoder_config, "num_decoder_layers", task_config,
                                             "decoder_num_hidden_layers")
                self.decoder = DecoderModel(decoder_config, word_table, position_table)
            if task_config.do_pretrain:
                self.cls = BertOnlyMLMHead(bert_config, word_table)
                self.cls_visual = VisualOnlyMLMHead(visual_config, visual_in_proj)
            self.similarity_dense = nn.Linear(bert_config.hidden_size, 1)

        self.normalize_video = NormalizeVideo(task_config)

        local_bs = task_config.batch_size // task_config.n_gpu
        mil = MILNCELoss(batch_size=local_bs, n_pair=task_config.n_pair)
        margin = MaxMarginRankingLoss(margin=task_config.margin, negative_weighting=task_config.negative_weighting,
                                      batch_size=local_bs, n_pair=task_config.n_pair,
                                      hard_negative_rate=task_config.hard_negative_rate)
        if task_config.use_mil:
            self.loss_fct = CrossEn() if self._stage_two else mil
            self._pretrain_sim_loss_fct = mil
        else:
            self.loss_fct = CrossEn() if self._stage_two else margin
            self._pretrain_sim_loss_fct = margin

        self.apply(self.init_weights)

    def train(self, mode=True):
        """nn.Module.train; back in training mode the caption decoding cache (PrefixDecodeCache) is released"""
        if mode:
            PrefixDecodeCache.release(self)
        return super(UniVL, self).train(mode)

    # ------------------------------------------------------------------------------------------------------
    # internals work on 2-D bf16 [rows, H] tensors plus the int64 masks
    # ------------------------------------------------------------------------------------------------------
    def _device(self):
        return self.bert.embeddings.word_embeddings.weight.device

    def _encode(self, input_ids, token_type_ids, attention_mask, video_norm, video_mask):
        """reference :299-313 (inputs already flattened / normalised).  The text and the visual stacks are independent
        until the similarity / cross encoder, and at M = B*W = 1536 rows each of their kernels fills a fraction of the
        132 SMs: the visual stack runs on a side stream forked from (and joined back into) the current one, so the two
        stacks' sub-wave kernels share the machine — forward here, and backward too, because autograd replays every
        node on the stream its forward ran on.  Captured as two parallel branches under CUDA-graph capture."""
        side = rt.side_stream(self._device())
        if side is None:
            seq = self.bert.encode(input_ids, token_type_ids, attention_mask)
            vis = self.visual.encode(video_norm, video_mask)
            return seq, vis
        cur = torch.cuda.current_stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            vis = self.visual.encode(video_norm, video_mask)
        seq = self.bert.encode(input_ids, token_type_ids, attention_mask)
        cur.wait_stream(side)
        return seq, vis

    def _cross_pairs(self, seq2d, vis2d, attention_mask, video_mask, all_pairs):
        """reference :315-325 (+ the pairing of :355-370) -> (hidden2d, n_seq, S)"""
        return self.cross.encode_pairs(seq2d, vis2d, attention_mask, video_mask, all_pairs)

    def _cross_similarity(self, seq2d, vis2d, attention_mask, video_mask, groups=1):
        """reference :341-375: every (text i, video j) pair through the cross encoder -> pooled -> similarity_dense.
        The reference walks text rows in chunks of 5 and `repeat`s both sides; here all B_t x B_v sequences go
        through the layer kernels in one batch and the embedding kernel reads the un-repeated sources, except in
        evaluation without gradients, which scores them in bounded tiles (_cross_similarity_eval).  groups > 1:
        only the pairs inside each micro-batch, G * Bg^2 sequences -> [G, Bg, Bg]."""
        if groups == 1 and not self.training and not torch.is_grad_enabled():
            return self._cross_similarity_eval(seq2d, vis2d, attention_mask, video_mask)
        return self._cross_similarity_all_pairs(seq2d, vis2d, attention_mask, video_mask, groups)

    def _cross_similarity_all_pairs(self, seq2d, vis2d, attention_mask, video_mask, groups=1):
        """_cross_similarity as one batch of all the pair sequences (training, and any call with gradients)"""
        bt, bv = attention_mask.shape[0], video_mask.shape[0]
        # only token 0 of the last cross layer feeds the pooler: the last layer computes just those rows
        first, n_seq = self.cross.encode_pairs_first_token(seq2d, vis2d, attention_mask, video_mask, groups)
        u = self.cross.pooler.pre_activation(first, n_seq, 1)
        logits = ops.PoolerSimFn.apply(u, self.similarity_dense.weight, self.similarity_dense.bias)
        if groups > 1:
            return logits.view(groups, bt // groups, bv // groups)
        return logits.view(bt, bv)

    def _cross_similarity_eval(self, seq2d, vis2d, attention_mask, video_mask):
        """_cross_similarity in evaluation (model.eval() under torch.no_grad(), as the reference's eval_epoch calls
        it), in memory bounded by EVAL_PAIR_TOKENS whatever the batch: the Nt x Nv pairs are scored in tiles of
        (text block x video block) into one fp32 [Nt, Nv] result.  With dropout off, the first cross layer's Q/K/V
        projections of a pair's token depend on its text or video row alone, so they are computed once per source row
        (CrossModel.first_layer_source_qkv) and every tile reads them in place.  Every other stage is row- or
        sequence-local, so a pair's logit does not depend on the tiling.  UNIVL_EVAL_PRECISION=fp8 (eval_precision)
        runs the cross layers' dense GEMMs over the pair tokens in FP8, with weights quantized once per call.
        UNIVL_EVAL_LAYOUT=packed (eval_layout) scores the pairs on their valid tokens alone
        (_cross_similarity_eval_packed).  Token 0 is the one the pooler reads, and it must be a real key of every pair:
        a packed call with any text row whose attention_mask[i, 0] == 0 takes the padded path as a whole."""
        Nt, W = attention_mask.shape
        Nv, F = video_mask.shape
        fp8 = eval_precision() == "fp8" and len(self.cross.encoder.layer) > 1
        qw = self.cross.fp8_eval_weights() if fp8 else None
        if eval_layout() == "packed":
            packing = ops.PairPacking(attention_mask, video_mask)
            if packing.token0_valid:
                return self._cross_similarity_eval_packed(seq2d, vis2d, packing, qw)
        qkv = self.cross.first_layer_source_qkv(seq2d, vis2d, Nt, W, Nv, F)
        qkv_t, qkv_v = qkv[:Nt * W], qkv[Nt * W:]
        logits = torch.empty((Nt, Nv), dtype=torch.float32, device=seq2d.device)
        bt, bv = _eval_tile(Nt, Nv, W + F, EVAL_PAIR_TOKENS)
        for t0 in range(0, Nt, bt):
            t1 = min(Nt, t0 + bt)
            for v0 in range(0, Nv, bv):
                v1 = min(Nv, v0 + bv)
                tile_args = (seq2d[t0 * W:t1 * W], vis2d[v0 * F:v1 * F], attention_mask[t0:t1], video_mask[v0:v1],
                             qkv_t[t0 * W:t1 * W], qkv_v[v0 * F:v1 * F])
                if fp8:
                    first = self.cross.encode_pairs_first_token_eval_fp8(*tile_args, qw)
                else:
                    first = self.cross.encode_pairs_first_token_eval(*tile_args)
                u = self.cross.pooler.pre_activation(first, (t1 - t0) * (v1 - v0), 1)
                tile = ops.PoolerSimFn.apply(u, self.similarity_dense.weight, self.similarity_dense.bias)
                logits[t0:t1, v0:v1] = tile.view(t1 - t0, v1 - v0)
        return logits

    def _cross_similarity_eval_packed(self, seq2d, vis2d, packing, qw):
        """_cross_similarity_eval on the packed layout: pair (i, j) is computed on text i's and video j's valid tokens
        alone, each at its original position.  A padded key adds -10000 to its score, so next to a real key its
        exp(s - max) is exactly 0 in fp32, and every other stage acts on each row alone: a real row's result does not
        depend on the padded rows, and the logits equal the padded path's up to the order of the fp32 sums inside
        attention.  Tiles hold at most EVAL_PAIR_TOKENS packed tokens (_packed_eval_tiles); a pair's logit does not
        depend on the tiling.  packing: the call's ops.PairPacking; qw: fp8_eval_weights() or None (bf16)."""
        (Nt, W), (Nv, F) = packing.text_shape, packing.video_shape
        x, qkv = self.cross.first_layer_source_rows(seq2d, vis2d, Nt, W, Nv, F)
        logits = torch.empty((Nt, Nv), dtype=torch.float32, device=seq2d.device)
        for t0, t1, v0, v1 in _packed_eval_tiles(packing.len_t, packing.len_v, EVAL_PAIR_TOKENS):
            seqs = packing.tile(t0, t1, v0, v1)
            first = self.cross.encode_pairs_first_token_eval_packed(x, qkv, Nt * W, seqs, qw)
            u = self.cross.pooler.pre_activation(first, seqs.n_seq, 1)
            tile = ops.PoolerSimFn.apply(u, self.similarity_dense.weight, self.similarity_dense.bias)
            logits[t0:t1, v0:v1] = tile.view(t1 - t0, v1 - v0)
        return logits

    def _mean_pool_similarity(self, seq2d, vis2d, attention_mask, video_mask, groups=1):
        """reference :327-339 and :385-389; groups > 1: the block diagonal [G, Bg, Bg]"""
        l2 = self.task_config.use_mil is False
        n_t, W = attention_mask.shape
        n_v, F = video_mask.shape
        text = ops.MeanPoolFn.apply(seq2d, attention_mask, n_t, W, True, False, l2)
        video = ops.MeanPoolFn.apply(vis2d, video_mask, n_v, F, False, True, l2)
        return ops.SimMatmulFn.apply(text, video, groups)

    def _similarity(self, seq2d, vis2d, attention_mask, video_mask, _pretrain_joint=False, groups=1):
        if (self._stage_two and _pretrain_joint is False) or self.train_sim_after_cross:
            return self._cross_similarity(seq2d, vis2d, attention_mask, video_mask, groups)
        return self._mean_pool_similarity(seq2d, vis2d, attention_mask, video_mask, groups)

    def _calculate_mlm_loss(self, cross2d, n_seq, S, W, token_labels, groups=1):
        """reference :273-276 on the text half of the cross output"""
        text_rows = cross2d.view(n_seq, S, -1)[:, :W].reshape(n_seq * W, -1)
        return self.cls.loss(text_rows, token_labels, groups=groups)

    def _calculate_mfm_loss(self, cross2d, n_seq, S, W, video_norm, video_mask, video_labels_index, groups=1):
        """reference :278-297: NCE of every masked frame against all frames of the rank (of its micro-batch)"""
        F = S - W
        vis_rows = cross2d.view(n_seq, S, -1)[:, W:].reshape(n_seq * F, -1)
        scores = self.cls_visual.scores(vis_rows)
        frames = video_norm.reshape(n_seq * F, -1)
        return ops.ProjXentFn.apply(scores, frames, None, video_labels_index.reshape(-1).contiguous(),
                                    video_mask.reshape(-1).contiguous(), 1, False, False, groups)

    def _decoder_hidden(self, seq2d, vis2d, attention_mask, video_mask, input_caption_ids, decoder_mask):
        """reference :393-407 up to the classifier"""
        cross2d, n_seq, S = self._cross_pairs(seq2d, vis2d, attention_mask, video_mask, False)
        return self.decoder.decode(input_caption_ids, cross2d, decoder_mask, attention_mask, video_mask)

    # ------------------------------------------------------------------------------------------------------
    # public surface
    # ------------------------------------------------------------------------------------------------------
    def forward(self, input_ids, token_type_ids, attention_mask, video, video_mask=None,
                pairs_masked_text=None, pairs_token_labels=None, masked_video=None, video_labels_index=None,
                input_caption_ids=None, decoder_mask=None, output_caption_ids=None, micro_batches=1):
        """micro_batches = G > 1: the batch holds G consecutive micro-batches (rows [g b, (g+1) b) of the leading
        dimension) of a gradient-accumulation window, run as one batch.  Returns (1/G) * sum_g L_g, L_g being the loss
        of micro-batch g alone (its own similarity matrix, contrastive negatives, MLM / MFM / caption means), so one
        backward() gives the window's accumulated gradient.  G = 1 is the plain call."""
        G = micro_batches
        if isinstance(G, bool) or not isinstance(G, int) or G < 1:
            raise ValueError("micro_batches must be an integer >= 1, got %r" % (micro_batches,))
        if G > 1 and input_ids.shape[0] % G:
            raise ValueError("micro_batches=%d does not divide the batch of %d rows" % (G, input_ids.shape[0]))
        with rt.use_model(self, self._device()):
            input_ids, token_type_ids = _flat(input_ids), _flat(token_type_ids)
            attention_mask, video_mask = _flat(attention_mask), _flat(video_mask)
            video = self.normalize_video(video)
            if input_caption_ids is not None:
                input_caption_ids, decoder_mask = _flat(input_caption_ids), _flat(decoder_mask)
            seq, vis = self._encode(input_ids, token_type_ids, attention_mask, video, video_mask)
            if not self.training:
                return None
            cfg = self.task_config
            loss = 0.
            if self._stage_one:
                sim = self._similarity(seq, vis, attention_mask, video_mask, groups=G)
                loss = loss + self.loss_fct(sim)
            if self._stage_two:
                seq_a, vis_a = seq, vis
                if cfg.do_pretrain:
                    masked_ids, token_labels = _flat(pairs_masked_text), _flat(pairs_token_labels)
                    masked_video = self.normalize_video(masked_video)
                    video_labels_index = _flat(video_labels_index)
                    seq_a, vis_a = self._encode(masked_ids, token_type_ids, attention_mask, masked_video, video_mask)
                    cross2d, n_seq, S = self._cross_pairs(seq_a, vis_a, attention_mask, video_mask, False)
                    W = attention_mask.shape[-1]
                    loss = loss + self._calculate_mlm_loss(cross2d, n_seq, S, W, token_labels, G)
                    loss = loss + self._calculate_mfm_loss(cross2d, n_seq, S, W, video, video_mask,
                                                           video_labels_index, G)
                    joint = self._similarity(seq, vis, attention_mask, video_mask, _pretrain_joint=True, groups=G)
                    loss = loss + self._pretrain_sim_loss_fct(joint)
                if input_caption_ids is not None and (cfg.do_pretrain or cfg.task_type == "caption"):
                    hidden = self._decoder_hidden(seq_a, vis_a, attention_mask, video_mask, input_caption_ids,
                                                  decoder_mask)
                    loss = loss + self.decoder.classifier.cls.loss(hidden, _flat(output_caption_ids), groups=G)
                if cfg.do_pretrain or cfg.task_type == "retrieval":
                    sim = self._similarity(seq_a, vis_a, attention_mask, video_mask, groups=G)
                    loss = loss + self.loss_fct(sim)
            return loss

    def get_sequence_visual_output(self, input_ids, token_type_ids, attention_mask, video, video_mask, shaped=False):
        with rt.use_model(self, self._device()):
            if shaped is False:
                input_ids, token_type_ids = _flat(input_ids), _flat(token_type_ids)
                attention_mask, video_mask = _flat(attention_mask), _flat(video_mask)
                video = self.normalize_video(video)
            seq, vis = self._encode(input_ids, token_type_ids, attention_mask, video, video_mask)
            n, W = input_ids.shape
            return seq.view(n, W, -1), vis.view(video_mask.shape[0], video_mask.shape[1], -1)

    def get_similarity_logits(self, sequence_output, visual_output, attention_mask, video_mask, shaped=False,
                              _pretrain_joint=False):
        with rt.use_model(self, self._device()):
            if shaped is False:
                attention_mask, video_mask = _flat(attention_mask), _flat(video_mask)
            seq2d = sequence_output.to(torch.bfloat16).reshape(-1, sequence_output.shape[-1]).contiguous()
            vis2d = visual_output.to(torch.bfloat16).reshape(-1, visual_output.shape[-1]).contiguous()
            return self._similarity(seq2d, vis2d, attention_mask.contiguous(), video_mask.contiguous(),
                                    _pretrain_joint=_pretrain_joint)

    def _get_decoder_score(self, sequence_output, visual_output, input_ids, attention_mask, video_mask,
                           input_caption_ids, decoder_mask, shaped=False):
        with rt.use_model(self, self._device()):
            if shaped is False:
                attention_mask, video_mask = _flat(attention_mask), _flat(video_mask)
                input_caption_ids, decoder_mask = _flat(input_caption_ids), _flat(decoder_mask)
            seq2d = sequence_output.to(torch.bfloat16).reshape(-1, sequence_output.shape[-1]).contiguous()
            vis2d = visual_output.to(torch.bfloat16).reshape(-1, visual_output.shape[-1]).contiguous()
            hidden = self._decoder_hidden(seq2d, vis2d, attention_mask.contiguous(), video_mask.contiguous(),
                                          input_caption_ids.contiguous(), decoder_mask.contiguous())
            n, L = input_caption_ids.shape
            return self.decoder.classifier.cls.logits(hidden).reshape(n, L, -1), ()

    def decoder_caption(self, sequence_output, visual_output, input_ids, attention_mask, video_mask,
                        input_caption_ids, decoder_mask, shaped=False, get_logits=False):
        """UNIVL_DECODE_CACHE=prefix (caption.decode_cache_mode) serves the calls of a token-by-token decoding loop
        incrementally through the model's caption.PrefixDecodeCache; the result is the same either way."""
        if decode_cache_mode() == "prefix":
            scores = PrefixDecodeCache.of(self).logits(sequence_output, visual_output, attention_mask, video_mask,
                                                       input_caption_ids, decoder_mask, shaped=shaped)
        else:
            scores, _ = self._get_decoder_score(sequence_output, visual_output, input_ids, attention_mask, video_mask,
                                                input_caption_ids, decoder_mask, shaped=shaped)
        if get_logits:
            return scores
        return torch.max(scores, -1)[1]
