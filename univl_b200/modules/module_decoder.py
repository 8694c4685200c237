"""Caption decoder — surface of the reference's modules/module_decoder.py (DecoderConfig :45-109, DecoderModel
:351-406) over the fused sm_90a layer kernels."""
import logging

import torch
from torch import nn

from .. import ops
from .. import runtime as rt
from .module_bert import BertOnlyMLMHead
from .transformer import (DenseNormParams, IntermediateParams, SelfAttentionParams, attention_param_list,
                          check_config, ffn_param_list)
from .until_config import PretrainedConfig
from .until_module import LayerNorm, PreTrainedModel

logger = logging.getLogger(__name__)

PRETRAINED_MODEL_ARCHIVE_MAP = {}
CONFIG_NAME = "decoder_config.json"
WEIGHTS_NAME = "decoder_pytorch_model.bin"


class DecoderConfig(PretrainedConfig):
    pretrained_model_archive_map = PRETRAINED_MODEL_ARCHIVE_MAP
    config_name = CONFIG_NAME
    weights_name = WEIGHTS_NAME

    def __init__(self, vocab_size_or_config_json_file, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1,
                 attention_probs_dropout_prob=0.1, type_vocab_size=2, initializer_range=0.02,
                 max_target_embeddings=128, num_decoder_layers=1):
        self._init_from(vocab_size_or_config_json_file, dict(
            hidden_size=hidden_size, num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
            hidden_act=hidden_act, intermediate_size=intermediate_size, hidden_dropout_prob=hidden_dropout_prob,
            attention_probs_dropout_prob=attention_probs_dropout_prob, type_vocab_size=type_vocab_size,
            initializer_range=initializer_range, max_target_embeddings=max_target_embeddings,
            num_decoder_layers=num_decoder_layers))


class DecoderAttention(nn.Module):
    """`att.{query,key,value}` + `output.{dense,LayerNorm}` (reference :195-213, :268-277)."""

    def __init__(self, config):
        super(DecoderAttention, self).__init__()
        self.att = SelfAttentionParams(config)
        self.output = DenseNormParams(config.hidden_size, config)


class DecoderLayer(nn.Module):
    """causal self-attention, encoder attention, FFN (reference :279-292) — one fused autograd node."""

    def __init__(self, config):
        super(DecoderLayer, self).__init__()
        self.slf_attn = DecoderAttention(config)
        self.enc_attn = DecoderAttention(config)
        self.intermediate = IntermediateParams(config)
        self.output = DenseNormParams(config.intermediate_size, config)

    def run(self, x2d, enc2d, n_seq, L, Se, slf_mask, enc_mask):
        params = attention_param_list(self.slf_attn.att, self.slf_attn.output) + \
            attention_param_list(self.enc_attn.att, self.enc_attn.output) + \
            ffn_param_list(self.intermediate, self.output)
        return ops.DecoderLayerFn.apply(x2d, enc2d, n_seq, L, Se, slf_mask, enc_mask, self.output.dropout.p,
                                        self.slf_attn.att.dropout.p, self.training, *params)


class DecoderEmbeddings(nn.Module):
    """word + position tables tied to the text encoder's, LayerNorm, dropout (reference :294-320)."""

    def __init__(self, config, decoder_word_embeddings_weight, decoder_position_embeddings_weight):
        super(DecoderEmbeddings, self).__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_target_embeddings, config.hidden_size)
        self.word_embeddings.weight = decoder_word_embeddings_weight
        self.position_embeddings.weight = decoder_position_embeddings_weight
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def run(self, input_ids):
        return ops.EmbedTextFn.apply(input_ids, None, self.word_embeddings.weight, self.position_embeddings.weight,
                                     None, self.LayerNorm.weight, self.LayerNorm.bias, self.dropout.p, self.training)


class Decoder(nn.Module):
    def __init__(self, config):
        super(Decoder, self).__init__()
        self.layer = nn.ModuleList([DecoderLayer(config) for _ in range(config.num_decoder_layers)])


class DecoderClassifier(nn.Module):
    def __init__(self, config, embedding_weights):
        super(DecoderClassifier, self).__init__()
        self.cls = BertOnlyMLMHead(config, embedding_weights)


class DecoderModel(PreTrainedModel):
    """embeddings -> N decoder layers -> tied vocabulary classifier (reference :351-406)."""

    def __init__(self, config, decoder_word_embeddings_weight, decoder_position_embeddings_weight):
        super(DecoderModel, self).__init__(config)
        check_config(config)
        self.config = config
        self.max_target_length = config.max_target_embeddings
        self.embeddings = DecoderEmbeddings(config, decoder_word_embeddings_weight,
                                            decoder_position_embeddings_weight)
        self.decoder = Decoder(config)
        self.classifier = DecoderClassifier(config, decoder_word_embeddings_weight)
        self.apply(self.init_weights)

    def decode(self, input_ids, enc2d, answer_mask, enc_mask_a, enc_mask_b):
        """-> hidden bf16 [N*L, H].  Self-attention mask = (answer padded OR future) -> -10000 once (:389-396);
        encoder mask = concat(enc_mask_a, enc_mask_b) (:385-387)."""
        n_seq, L = input_ids.shape
        Se = enc_mask_a.shape[1] + (enc_mask_b.shape[1] if enc_mask_b is not None else 0)
        x = self.embeddings.run(input_ids)
        slf = ops.MaskSpec(answer_mask, causal=True)
        enc = ops.MaskSpec(enc_mask_a, enc_mask_b)
        for layer in self.decoder.layer:
            x = layer.run(x, enc2d, n_seq, L, Se, slf, enc)
        return x

    def forward(self, input_ids, encoder_outs=None, answer_mask=None, encoder_mask=None):
        """-> logits [N, L, vocab] fp32"""
        with rt.use_model(self, input_ids.device):
            n_seq, L = input_ids.shape
            enc2d = encoder_outs.to(torch.bfloat16).contiguous().view(-1, encoder_outs.shape[-1])
            h = self.decode(input_ids.contiguous(), enc2d, answer_mask.long().contiguous(),
                            encoder_mask.long().contiguous(), None)
            return self.classifier.cls.logits(h).reshape(n_seq, L, -1)
