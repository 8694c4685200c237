"""Visual (S3D feature) encoder — surface of the reference's modules/module_visual.py (VisualConfig :44-102,
VisualModel :364-425, VisualOnlyMLMHead :314-321) over the fused sm_90a layer kernels."""
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
CONFIG_NAME = "visual_config.json"
WEIGHTS_NAME = "visual_pytorch_model.bin"


class VisualConfig(PretrainedConfig):
    pretrained_model_archive_map = PRETRAINED_MODEL_ARCHIVE_MAP
    config_name = CONFIG_NAME
    weights_name = WEIGHTS_NAME

    def __init__(self, vocab_size_or_config_json_file=4096, hidden_size=768, num_hidden_layers=3,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1,
                 attention_probs_dropout_prob=0.1, max_position_embeddings=512, initializer_range=0.02):
        self._init_from(vocab_size_or_config_json_file, dict(
            hidden_size=hidden_size, num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
            hidden_act=hidden_act, intermediate_size=intermediate_size, hidden_dropout_prob=hidden_dropout_prob,
            attention_probs_dropout_prob=attention_probs_dropout_prob,
            max_position_embeddings=max_position_embeddings, initializer_range=initializer_range))


class VisualEmbeddings(nn.Module):
    """Linear(video_dim -> hidden) + position table + LayerNorm + dropout (reference :104-131)."""

    def __init__(self, config):
        super(VisualEmbeddings, self).__init__()
        self.word_embeddings = nn.Linear(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def run(self, video2d, n_seq, F):
        proj = ops.LinearFn.apply(video2d, self.word_embeddings.weight, self.word_embeddings.bias, False,
                                  video2d.requires_grad)
        return ops.EmbedSrcFn.apply(proj, None, n_seq, F, 0, 0, False, self.position_embeddings.weight, None,
                                    self.LayerNorm.weight, self.LayerNorm.bias, self.dropout.p, self.training)


class VisualLMPredictionHead(nn.Module):
    """transform, then multiply by the UN-transposed tied input projection [hidden, video_dim] (reference :298-311)."""

    def __init__(self, config, visual_model_embedding_weights):
        super(VisualLMPredictionHead, self).__init__()
        self.transform = HeadTransform(config)
        self.weight = visual_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(visual_model_embedding_weights.size(1)))


class VisualOnlyMLMHead(nn.Module):
    def __init__(self, config, visual_model_embedding_weights):
        super(VisualOnlyMLMHead, self).__init__()
        self.predictions = VisualLMPredictionHead(config, visual_model_embedding_weights)

    def scores(self, hidden2d):
        """[T, video_dim] bf16 = transform(h) @ W + bias with W stored [hidden, video_dim] (an MN-major B operand)."""
        t = self.predictions.transform.run(hidden2d)
        return ops.LinearTFn.apply(t, self.predictions.weight, self.predictions.bias)

    def forward(self, sequence_output):
        with rt.use_model(self, sequence_output.device):
            shape = sequence_output.shape
            x = sequence_output.to(torch.bfloat16).contiguous().view(-1, shape[-1])
            return self.scores(x).view(*shape[:-1], -1)


class VisualModel(PreTrainedModel):
    """embeddings -> N fused encoder layers -> pooler (reference :364-425).  `video`: [N, F, video_dim]."""

    def __init__(self, config):
        super(VisualModel, self).__init__(config)
        check_config(config)
        self.embeddings = VisualEmbeddings(config)
        self.encoder = EncoderStack(config)
        self.pooler = Pooler(config)
        self.apply(self.init_weights)

    def encode(self, video, video_mask, keep_all=False):
        n_seq, F = video.shape[0], video.shape[1]
        x = self.embeddings.run(video.to(torch.bfloat16).contiguous().view(n_seq * F, -1), n_seq, F)
        return self.encoder.run(x, n_seq, F, ops.MaskSpec(video_mask), keep_all=keep_all)

    def forward(self, video, attention_mask=None, output_all_encoded_layers=True):
        if attention_mask is None:
            attention_mask = torch.ones(video.size(0), video.size(1), dtype=torch.long, device=video.device)
        with rt.use_model(self, video.device):
            n_seq, F = video.shape[0], video.shape[1]
            outs = self.encode(video, attention_mask, keep_all=True)
            pooled = self.pooler.run(outs[-1], n_seq, F)
            layers = hidden_list(outs, n_seq, F)
            return (layers if output_all_encoded_layers else layers[-1]), pooled
