"""Primitives, the PreTrainedModel base and the similarity losses — the surface of the reference's
modules/until_module.py (LayerNorm :40-53, gelu :28-33, PreTrainedModel :55-177, CrossEn :182-191, MILNCELoss
:193-221, MaxMarginRankingLoss :223-251) on top of the sm_90a kernels.  No CPU path: every forward here requires CUDA
tensors and raises otherwise.
"""
import logging

import torch
from torch import nn

from .. import ops
from ..runtime import call
from .until_config import PretrainedConfig

logger = logging.getLogger(__name__)


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError("univl_b200: %s needs CUDA tensors (sm_90a kernels only, no CPU fallback)" % what)


def gelu(x):
    """erf-GELU, x * 0.5 * (1 + erf(x / sqrt(2))) — evaluated by the fused GEMM epilogue on the hot path; this
    standalone form exists for API parity and runs the same device function via gelu'(x) integration-free path."""
    _require_cuda(x, "gelu")
    xb = x.to(torch.bfloat16).contiguous()
    out = torch.empty_like(xb)
    call("univl_gelu_fwd_bf16", xb.data_ptr(), out.data_ptr(), xb.numel())
    return out.to(x.dtype)


def swish(x):
    raise NotImplementedError("univl_b200 implements the hot path only: hidden_act must be 'gelu'")


ACT2FN = {"gelu": gelu}


class LayerNorm(nn.Module):
    """TF-style LayerNorm (epsilon inside the square root), fp32 parameters `weight` / `bias`."""

    def __init__(self, hidden_size, eps=1e-12):
        super(LayerNorm, self).__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        _require_cuda(x, "LayerNorm")
        shape = x.shape
        y = ops.LayerNormFn.apply(x.reshape(-1, shape[-1]).to(torch.bfloat16).contiguous(), self.weight, self.bias)
        return y.view(shape)


class PreTrainedModel(nn.Module):
    """Weight initialisation + non-strict, key-renaming checkpoint loading (reference :55-177)."""

    def __init__(self, config, *inputs, **kwargs):
        super(PreTrainedModel, self).__init__()
        if not isinstance(config, PretrainedConfig):
            raise ValueError(
                "Parameter config in `{}(config)` should be an instance of class `PretrainedConfig`. "
                "To create a model from a Google pretrained model use "
                "`model = {}.from_pretrained(PRETRAINED_MODEL_NAME)`".format(
                    self.__class__.__name__, self.__class__.__name__))
        self.config = config

    def init_weights(self, module):
        """N(0, initializer_range) for Linear/Embedding weights, zeros for Linear biases, (1, 0) for LayerNorm."""
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    def resize_token_embeddings(self, new_num_tokens=None):
        raise NotImplementedError

    @classmethod
    def init_preweight(cls, model, state_dict, prefix=None, task_config=None):
        """Load `state_dict` by key name; `gamma`/`beta` are renamed to `weight`/`bias`; missing and unexpected keys
        are logged, never raised (reference :91-146)."""
        renamed = {}
        for key in list(state_dict.keys()):
            new_key = key
            if "gamma" in new_key:
                new_key = new_key.replace("gamma", "weight")
            if "beta" in new_key:
                new_key = new_key.replace("beta", "bias")
            if prefix is not None:
                new_key = prefix + new_key
            renamed[new_key] = state_dict[key]
        metadata = getattr(state_dict, "_metadata", None)
        missing, unexpected, errors = [], [], []

        def visit(module, path):
            meta = {} if metadata is None else metadata.get(path[:-1], {})
            module._load_from_state_dict(renamed, path, meta, True, missing, unexpected, errors)
            for name, child in module._modules.items():
                if child is not None:
                    visit(child, path + name + ".")

        visit(model, "")
        if prefix is None and (task_config is None or task_config.local_rank == 0):
            logger.info("-" * 20)
            if missing:
                logger.info("Weights of {} not initialized from pretrained model: {}".format(
                    model.__class__.__name__, "\n   " + "\n   ".join(missing)))
            if unexpected:
                logger.info("Weights from pretrained model not used in {}: {}".format(
                    model.__class__.__name__, "\n   " + "\n   ".join(unexpected)))
            if errors:
                logger.error("Weights from pretrained model cause errors in {}: {}".format(
                    model.__class__.__name__, "\n   " + "\n   ".join(errors)))
        arena = model.__dict__.get("_univl_arena")
        if arena is not None:
            arena.fresh = False
        return model

    @property
    def dtype(self):
        try:
            return next(self.parameters()).dtype
        except StopIteration:
            return torch.float32

    @classmethod
    def from_pretrained(cls, config, state_dict=None, *inputs, **kwargs):
        model = cls(config, *inputs, **kwargs)
        if state_dict is None:
            return model
        return cls.init_preweight(model, state_dict)


# ---------------------------------------------------------------------------------------------------------
# losses on the [B, B] similarity matrix, or on a [G, B, B] stack of one matrix per micro-batch: the mean over the G
# group losses, each the reference loss of its own matrix (UniVL.forward(micro_batches=G))
# ---------------------------------------------------------------------------------------------------------
def _sim_input(sim_matrix, what, group_size=None):
    _require_cuda(sim_matrix, what)
    if sim_matrix.dim() == 3 and sim_matrix.shape[-1] != sim_matrix.shape[-2]:
        raise ValueError("%s: expected [G, B, B] micro-batch similarity matrices, got %s"
                         % (what, tuple(sim_matrix.shape)))
    if sim_matrix.dim() == 3 and group_size is not None and sim_matrix.shape[-1] != group_size:
        raise ValueError("%s: micro-batch similarity is %dx%d but the loss was built for batch_size * n_pair = %d"
                         % (what, sim_matrix.shape[-1], sim_matrix.shape[-1], group_size))
    return sim_matrix.float()


class CrossEn(nn.Module):
    def forward(self, sim_matrix):
        return ops.SimLossFn.apply(_sim_input(sim_matrix, "CrossEn"), "crossen", None)


class MILNCELoss(nn.Module):
    def __init__(self, batch_size=1, n_pair=1):
        super(MILNCELoss, self).__init__()
        self.batch_size = batch_size
        self.n_pair = n_pair

    def forward(self, sim_matrix):
        sim = _sim_input(sim_matrix, "MILNCELoss", self.batch_size * self.n_pair)
        return ops.SimLossFn.apply(sim, "milnce", (self.batch_size, self.n_pair))


class MaxMarginRankingLoss(nn.Module):
    def __init__(self, margin=1.0, negative_weighting=False, batch_size=1, n_pair=1, hard_negative_rate=0.5):
        super(MaxMarginRankingLoss, self).__init__()
        self.margin = margin
        self.n_pair = n_pair
        self.batch_size = batch_size
        self.easy_negative_rate = 1 - hard_negative_rate
        self.negative_weighting = negative_weighting
        # block weights of the reference's mm_mask (:238-243): same-video block vs other blocks
        self.w_same = self.w_diff = 1.0
        self.weighted = bool(negative_weighting) and n_pair > 1 and batch_size > 1
        if n_pair > 1 and batch_size > 1:
            easy = self.easy_negative_rate
            alpha = easy / ((batch_size - 1) * (1 - easy))
            scale = batch_size * (1 - easy)
            self.w_same, self.w_diff = 1.0 * scale, alpha * scale

    def forward(self, x):
        x = _sim_input(x, "MaxMarginRankingLoss", self.batch_size * self.n_pair)
        args = (self.margin, self.n_pair if self.weighted else 0, self.w_same, self.w_diff)
        return ops.SimLossFn.apply(x, "maxmargin", args)
