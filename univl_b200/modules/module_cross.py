"""Cross-modal encoder — surface of the reference's modules/module_cross.py (CrossConfig :44-107, CrossModel
:355-394) over the fused sm_90a layer kernels."""
import logging

import torch
from torch import nn

from .. import ops
from .. import runtime as rt
from .transformer import EncoderStack, Pooler, _layer_params, check_config, hidden_list
from .until_config import PretrainedConfig
from .until_module import LayerNorm, PreTrainedModel

logger = logging.getLogger(__name__)

PRETRAINED_MODEL_ARCHIVE_MAP = {}
CONFIG_NAME = "cross_config.json"
WEIGHTS_NAME = "cross_pytorch_model.bin"


class CrossConfig(PretrainedConfig):
    pretrained_model_archive_map = PRETRAINED_MODEL_ARCHIVE_MAP
    config_name = CONFIG_NAME
    weights_name = WEIGHTS_NAME

    def __init__(self, vocab_size_or_config_json_file, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1,
                 attention_probs_dropout_prob=0.1, max_position_embeddings=512, type_vocab_size=2,
                 initializer_range=0.02):
        self._init_from(vocab_size_or_config_json_file, dict(
            hidden_size=hidden_size, num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
            hidden_act=hidden_act, intermediate_size=intermediate_size, hidden_dropout_prob=hidden_dropout_prob,
            attention_probs_dropout_prob=attention_probs_dropout_prob,
            max_position_embeddings=max_position_embeddings, type_vocab_size=type_vocab_size,
            initializer_range=initializer_range))


class CrossEmbeddings(nn.Module):
    """position + type tables added to already-hidden-size inputs, LayerNorm, dropout (reference :109-138)."""

    def __init__(self, config):
        super(CrossEmbeddings, self).__init__()
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def run(self, text2d, video2d, Nt, W, Nv, F, all_pairs):
        return ops.EmbedSrcFn.apply(text2d, video2d, Nt, W, Nv, F, all_pairs, self.position_embeddings.weight,
                                    self.token_type_embeddings.weight, self.LayerNorm.weight, self.LayerNorm.bias,
                                    self.dropout.p, self.training)


def _n_seq(Nt, Nv, groups):
    """sequences of a pairing over `groups` groups (0 / False: aligned)"""
    groups = int(groups)
    if groups and (Nt % groups or Nv % groups):
        raise ValueError("cross pairing: %d groups must divide %d text and %d video rows" % (groups, Nt, Nv))
    return Nt * Nv // groups if groups else Nt


class CrossModel(PreTrainedModel):
    """embeddings -> N fused encoder layers -> pooler (reference :355-394)."""

    def __init__(self, config):
        super(CrossModel, self).__init__(config)
        check_config(config)
        self.embeddings = CrossEmbeddings(config)
        self.encoder = EncoderStack(config)
        self.pooler = Pooler(config)
        self.apply(self.init_weights)

    def encode_pairs(self, text2d, video2d, text_mask, video_mask, all_pairs, keep_all=False):
        """text2d [Nt*W, H], video2d [Nv*F, H]; sequence p = concat(text_i, video_j) with (i, j) = (p, p) or, if
        all_pairs, (p / Nv, p % Nv) — the B x B pairing of reference modeling.py:341-375 without `repeat` copies.
        all_pairs = G > 1 pairs within G micro-batches only: G groups of (Nt/G) x (Nv/G) sequences, group after group.
        -> (hidden [n_seq*(W+F), H], n_seq, W+F)"""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        n_seq = _n_seq(Nt, Nv, all_pairs)
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, all_pairs)
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=all_pairs)
        return self.encoder.run(x, n_seq, W + F, mask, keep_all=keep_all), n_seq, W + F

    def encode_pairs_first_token(self, text2d, video2d, text_mask, video_mask, all_pairs):
        """as encode_pairs, but only token 0 of every sequence of the LAST layer is produced: [n_seq, H].  The pooled
        similarity head (reference modeling.py:371-373) reads nothing else, so the last layer skips the query side of
        the other W+F-1 tokens."""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        n_seq = _n_seq(Nt, Nv, all_pairs)
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, all_pairs)
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=all_pairs)
        return self.encoder.run_first_token(x, n_seq, W + F, mask), n_seq

    def first_layer_source_qkv(self, text2d, video2d, Nt, W, Nv, F):
        """Evaluation only: the first layer's Q/K/V projections of every text row and every video row, once per source
        row -> [Nt*W + Nv*F, 3H], text rows first.  With dropout off, a pair's first-layer input row is the embedding
        LayerNorm of its text or video row alone (position and type rows are the same for every pair), so these are
        the projections every pair sequence would compute for itself."""
        return self.first_layer_source_rows(text2d, video2d, Nt, W, Nv, F)[1]

    def first_layer_source_rows(self, text2d, video2d, Nt, W, Nv, F):
        """first_layer_source_qkv and the embedding-LayerNorm rows it projects, the first layer's residual input
        -> (x [Nt*W + Nv*F, H], qkv [Nt*W + Nv*F, 3H]), text rows first"""
        emb = self.embeddings
        pos, typ = emb.position_embeddings.weight, emb.token_type_embeddings.weight
        gamma, beta = emb.LayerNorm.weight, emb.LayerNorm.bias
        rows_t = Nt * W
        x = torch.empty((rows_t + Nv * F, text2d.shape[1]), dtype=torch.bfloat16, device=text2d.device)
        ops.embed_src_rows_eval(text2d, Nt, W, pos, typ, gamma, beta, x[:rows_t])
        ops.embed_src_rows_eval(video2d, Nv, F, pos[W:], typ[1:], gamma, beta, x[rows_t:])  # video rows: s >= W, type 1
        a = self.encoder.layer[0].attention.self
        wqkv = rt.current().bf16_qkv(a.query.weight, a.key.weight, a.value.weight)
        return x, ops.linear_fwd(x, wqkv, rt.packed_bias(a.query.bias, a.key.bias, a.value.bias))

    def encode_pairs_first_token_eval(self, text2d, video2d, text_mask, video_mask, qkv_t, qkv_v):
        """encode_pairs_first_token over all Nt x Nv pairs in evaluation, with the first layer's Q/K/V projections read
        from qkv_t [Nt*W, 3H] and qkv_v [Nv*F, 3H] (rows of first_layer_source_qkv) -> [Nt*Nv, H]"""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        S = W + F
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, 1)  # the first layer's residual input
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=1)
        layers = self.encoder.layer
        x = ops.pair_layer_eval(x, qkv_t, qkv_v, Nt, Nv, S, mask, _layer_params(layers[0]), len(layers) == 1)
        if len(layers) == 1:
            return x
        return self.encoder.run_first_token(x, Nt * Nv, S, mask, start=1)

    def fp8_eval_weights(self):
        """Per layer, the e4m3 weights encode_pairs_first_token_eval_fp8 reads, quantized now from the fp32 parameters
        (nothing is cached, so in-place weight edits and replicas are always current).  Needs >= 2 layers."""
        layers = self.encoder.layer
        out = []
        for i, layer in enumerate(layers):
            names = ("kv",) if i == len(layers) - 1 else ("o", "w1", "w2") if i == 0 else ("qkv", "o", "w1", "w2")
            out.append(ops.fp8_layer_weights(_layer_params(layer), names))
        return out

    def encode_pairs_first_token_eval_fp8(self, text2d, video2d, text_mask, video_mask, qkv_t, qkv_v, qw):
        """encode_pairs_first_token_eval with the dense GEMMs over the pair tokens in FP8 (qw = fp8_eval_weights()):
        the first layer's attention output and FFN, the middle layers' Q/K/V projection, attention output and FFN, and
        the last layer's K/V projection.  Needs >= 2 layers (with one, only token-0 rows remain, which stay bf16)."""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        S = W + F
        n_seq = Nt * Nv
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, 1)
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=1)
        layers = self.encoder.layer
        x = ops.pair_layer_eval_fp8(x, qkv_t, qkv_v, Nt, Nv, S, mask, _layer_params(layers[0]), qw[0])
        for i in range(1, len(layers) - 1):
            x = ops.encoder_layer_eval_fp8(x, n_seq, S, mask, _layer_params(layers[i]), qw[i])
        return ops.cls_layer_eval_fp8(x, n_seq, S, mask, _layer_params(layers[-1]), qw[-1])

    def encode_pairs_first_token_eval_list(self, x, qkv, text_mask, video_mask, text_index, video_index, qw=None):
        """encode_pairs_first_token_eval (qw None) or _fp8 (qw = fp8_eval_weights()) on a list of pairs instead of a
        grid, each pair at all W + F tokens: sequence p = (text row text_index[p], video row video_index[p]) (int32
        device tensors).  x, qkv: first_layer_source_rows of the call.  The first layer reads Q/K/V from qkv through
        the list (ops.attention_pair_fwd), its residual rows are gathered from x, and every layer reads the listed
        pairs' own mask rows, so a pair's result equals the grid's -> [P, H]"""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        S, P, rows_t = W + F, text_index.numel(), Nt * W
        pairs = (text_index, video_index)
        mask = ops.MaskSpec(text_mask.index_select(0, text_index.long()),
                            video_mask.index_select(0, video_index.long()), all_pairs=0)
        h = ops.gather_rows_varlen(x[:rows_t], x[rows_t:], ops.padded_pair_seqs(text_index, video_index, Nt, W, Nv, F),
                                   False)
        layers = self.encoder.layer
        if qw is not None:
            h = ops.pair_layer_eval_fp8(h, qkv[:rows_t], qkv[rows_t:], P, 1, S, mask, _layer_params(layers[0]), qw[0],
                                        pairs)
            for i in range(1, len(layers) - 1):
                h = ops.encoder_layer_eval_fp8(h, P, S, mask, _layer_params(layers[i]), qw[i])
            return ops.cls_layer_eval_fp8(h, P, S, mask, _layer_params(layers[-1]), qw[-1])
        h = ops.pair_layer_eval(h, qkv[:rows_t], qkv[rows_t:], P, 1, S, mask, _layer_params(layers[0]),
                                len(layers) == 1, pairs)
        if len(layers) == 1:
            return h
        return self.encoder.run_first_token(h, P, S, mask, start=1)

    def encode_pairs_first_token_eval_packed(self, x, qkv, rows_t, seqs, qw=None):
        """encode_pairs_first_token_eval (qw None) or _fp8 (qw = fp8_eval_weights()) on the packed layout: every pair
        of one tile on its valid tokens alone.  x, qkv: first_layer_source_rows of the call, whose first rows_t rows are
        the text rows; seqs: the tile's ops.VarlenSeqs (PairPacking.tile) -> [seqs.n_seq, H]"""
        layers = self.encoder.layer
        h = ops.pair_layer_eval_packed(x[:rows_t], x[rows_t:], qkv[:rows_t], qkv[rows_t:], seqs,
                                       _layer_params(layers[0]), len(layers) == 1, qw[0] if qw else None)
        if len(layers) == 1:
            return h
        for i in range(1, len(layers) - 1):
            h = ops.encoder_layer_eval_packed(h, seqs, _layer_params(layers[i]), qw[i] if qw else None)
        return ops.cls_layer_eval_packed(h, seqs, _layer_params(layers[-1]), qw[-1] if qw else None)

    def forward(self, concat_input, concat_type=None, attention_mask=None, output_all_encoded_layers=True):
        """API-parity entry: `concat_type` must be the reference's layout (0s for the text part then 1s)."""
        N, S, _ = concat_input.shape
        if attention_mask is None:
            attention_mask = torch.ones(N, S, dtype=torch.long, device=concat_input.device)
        if concat_type is None:
            concat_type = torch.zeros_like(attention_mask)
        W = int((concat_type[0] == 0).sum().item())
        if not bool((concat_type[:, :W] == 0).all()) or not bool((concat_type[:, W:] == 1).all()):
            raise ValueError("CrossModel.forward: concat_type must be [0]*W + [1]*F for every row")
        with rt.use_model(self, concat_input.device):
            x = concat_input.to(torch.bfloat16)
            text = x[:, :W].contiguous().view(N * W, -1)
            video = x[:, W:].contiguous().view(N * (S - W), -1) if S > W else None
            am = attention_mask.long()
            outs, n_seq, S2 = self.encode_pairs(text, video, am[:, :W].contiguous(),
                                                am[:, W:].contiguous() if S > W else am[:, :0], False, keep_all=True)
            pooled = self.pooler.run(outs[-1], n_seq, S2)
            layers = hidden_list(outs, n_seq, S2)
            return (layers if output_all_encoded_layers else layers[-1]), pooled
