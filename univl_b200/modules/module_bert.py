"""Text encoder — surface of the reference's modules/module_bert.py (BertConfig :44-116, BertModel :364-447,
BertOnlyMLMHead :333-340) over the fused sm_90a layer kernels."""
import logging

import torch
from torch import nn

from .. import ops
from .. import runtime as rt
from .transformer import EncoderStack, HeadTransform, Pooler, check_config, hidden_list
from .until_config import PretrainedConfig
from .until_module import LayerNorm, PreTrainedModel

logger = logging.getLogger(__name__)

PRETRAINED_MODEL_ARCHIVE_MAP = {}
CONFIG_NAME = "bert_config.json"
WEIGHTS_NAME = "pytorch_model.bin"


class BertConfig(PretrainedConfig):
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


class BertEmbeddings(nn.Module):
    """word + position + token-type tables, LayerNorm, dropout (reference :118-146)."""

    def __init__(self, config):
        super(BertEmbeddings, self).__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def run(self, input_ids, token_type_ids):
        return ops.EmbedTextFn.apply(input_ids, token_type_ids, self.word_embeddings.weight,
                                     self.position_embeddings.weight, self.token_type_embeddings.weight,
                                     self.LayerNorm.weight, self.LayerNorm.bias, self.dropout.p, self.training)


class BertLMPredictionHead(nn.Module):
    """transform + tied vocabulary projection + bias (reference :314-330)."""

    def __init__(self, config, bert_model_embedding_weights):
        super(BertLMPredictionHead, self).__init__()
        self.transform = HeadTransform(config)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1), bert_model_embedding_weights.size(0),
                                 bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))


class BertOnlyMLMHead(nn.Module):
    def __init__(self, config, bert_model_embedding_weights):
        super(BertOnlyMLMHead, self).__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)

    def loss(self, hidden2d, labels, return_logits=False):
        """CrossEntropy(ignore_index=-1) of the tied projection, fused (reference modeling.py:273-276)."""
        t = self.predictions.transform.run(hidden2d)
        return ops.ProjXentFn.apply(t, self.predictions.decoder.weight, self.predictions.bias, labels.reshape(-1),
                                    None, 0, True, return_logits)

    def logits(self, hidden2d):
        """[T, vocab] fp32 scores (inference: decoder_caption)."""
        t = self.predictions.transform.run(hidden2d)
        w16 = rt.current().bf16(self.predictions.decoder.weight)
        V = w16.shape[0]
        out = torch.empty((t.shape[0], ops._ld_pad(V)), dtype=torch.float32, device=t.device)[:, :V]
        return ops.gemm(t, w16, t.shape[0], V, t.shape[1], out, epi=ops.EPI_F32, bias=self.predictions.bias)

    def forward(self, sequence_output):
        with rt.use_model(self, sequence_output.device):
            shape = sequence_output.shape
            x = sequence_output.to(torch.bfloat16).contiguous().view(-1, shape[-1])
            return self.logits(x).reshape(*shape[:-1], -1)


class BertModel(PreTrainedModel):
    """embeddings -> N fused encoder layers -> pooler (reference :364-447)."""

    def __init__(self, config):
        super(BertModel, self).__init__(config)
        check_config(config)
        self.embeddings = BertEmbeddings(config)
        self.encoder = EncoderStack(config)
        self.pooler = Pooler(config)
        self.apply(self.init_weights)

    def encode(self, input_ids, token_type_ids, attention_mask, keep_all=False):
        """-> bf16 [N*S, H] (or the list over layers)"""
        n_seq, S = input_ids.shape
        mask = ops.MaskSpec(attention_mask)
        x = self.embeddings.run(input_ids, token_type_ids)
        return self.encoder.run(x, n_seq, S, mask, keep_all=keep_all)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, output_all_encoded_layers=True):
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        with rt.use_model(self, input_ids.device):
            n_seq, S = input_ids.shape
            outs = self.encode(input_ids, token_type_ids, attention_mask, keep_all=True)
            pooled = self.pooler.run(outs[-1], n_seq, S)
            layers = hidden_list(outs, n_seq, S)
            return (layers if output_all_encoded_layers else layers[-1]), pooled
