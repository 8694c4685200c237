"""Cross-modal encoder — surface of the reference's modules/module_cross.py (CrossConfig :44-107, CrossModel
:355-394) over the fused sm_90a layer kernels."""
import logging

import torch
from torch import nn

from .. import ops
from .. import runtime as rt
from .transformer import EncoderStack, Pooler, check_config, hidden_list
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
        -> (hidden [n_seq*(W+F), H], n_seq, W+F)"""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        n_seq = Nt * Nv if all_pairs else Nt
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, all_pairs)
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=all_pairs)
        return self.encoder.run(x, n_seq, W + F, mask, keep_all=keep_all), n_seq, W + F

    def encode_pairs_first_token(self, text2d, video2d, text_mask, video_mask, all_pairs):
        """as encode_pairs, but only token 0 of every sequence of the LAST layer is produced: [n_seq, H].  The pooled
        similarity head (reference modeling.py:371-373) reads nothing else, so the last layer skips the query side of
        the other W+F-1 tokens."""
        Nt, W = text_mask.shape
        Nv, F = video_mask.shape
        n_seq = Nt * Nv if all_pairs else Nt
        x = self.embeddings.run(text2d, video2d, Nt, W, Nv, F, all_pairs)
        mask = ops.MaskSpec(text_mask, video_mask, all_pairs=all_pairs)
        return self.encoder.run_first_token(x, n_seq, W + F, mask), n_seq

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
