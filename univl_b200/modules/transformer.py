"""Shared transformer building blocks for the four UniVL sub-models.

The reference has four copy-pasted BERT stacks (module_bert.py / module_visual.py / module_cross.py /
module_decoder.py); here ONE set of parameter-holder modules reproduces their attribute paths (and therefore their
`state_dict` keys, SURVEY.md Appendix A) while the arithmetic of a whole layer is a single fused autograd node
(univl_b200/ops.py: EncoderLayerFn / DecoderLayerFn) over the sm_90a kernels.  The nn.Linear / nn.Embedding children
only own parameters — their stock forwards are never called.
"""
import torch
from torch import nn

from .. import ops
from .until_module import LayerNorm


def check_config(config):
    if config.hidden_size != 768 or config.num_attention_heads != 12 or config.intermediate_size % 256 != 0:
        raise ValueError("univl_b200 kernels are specialised for hidden_size 768 / 12 heads of 64 (got %d / %d)"
                         % (config.hidden_size, config.num_attention_heads))
    if config.hidden_size % config.num_attention_heads != 0:
        raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                         % (config.hidden_size, config.num_attention_heads))
    act = config.hidden_act
    if not (isinstance(act, str) and act == "gelu"):
        raise ValueError("univl_b200 fuses erf-GELU into the FFN GEMM: hidden_act must be 'gelu' (got %r)" % (act,))


class SelfAttentionParams(nn.Module):
    """query / key / value projections (reference modules/module_bert.py:149-164)."""

    def __init__(self, config):
        super(SelfAttentionParams, self).__init__()
        check_config(config)
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = config.hidden_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)

    def _qkv_modules(self):  # read by runtime.WeightArena: these three weights are laid out adjacently
        return self.query, self.key, self.value


class DenseNormParams(nn.Module):
    """dense + dropout + LayerNorm(residual) holder (reference modules/module_bert.py:200-211, :239-250)."""

    def __init__(self, in_features, config):
        super(DenseNormParams, self).__init__()
        self.dense = nn.Linear(in_features, config.hidden_size)
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class IntermediateParams(nn.Module):
    """dense(H -> I) + erf-GELU holder (reference modules/module_bert.py:226-236)."""

    def __init__(self, config):
        super(IntermediateParams, self).__init__()
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)


class AttentionParams(nn.Module):
    """`attention.self.*` + `attention.output.*` (reference modules/module_bert.py:213-224)."""

    def __init__(self, config):
        super(AttentionParams, self).__init__()
        self.self = SelfAttentionParams(config)
        self.output = DenseNormParams(config.hidden_size, config)


def attention_param_list(self_mod, out_mod):
    """parameter tuple in ops.ATT_KEYS order"""
    return (self_mod.query.weight, self_mod.query.bias, self_mod.key.weight, self_mod.key.bias,
            self_mod.value.weight, self_mod.value.bias, out_mod.dense.weight, out_mod.dense.bias,
            out_mod.LayerNorm.weight, out_mod.LayerNorm.bias)


def ffn_param_list(intermediate, output):
    """parameter tuple in ops.FFN_KEYS order"""
    return (intermediate.dense.weight, intermediate.dense.bias, output.dense.weight, output.dense.bias,
            output.LayerNorm.weight, output.LayerNorm.bias)


class EncoderLayer(nn.Module):
    """BertLayer / VisualLayer / CrossLayer (reference modules/module_bert.py:253-264)."""

    def __init__(self, config):
        super(EncoderLayer, self).__init__()
        self.attention = AttentionParams(config)
        self.intermediate = IntermediateParams(config)
        self.output = DenseNormParams(config.intermediate_size, config)
        self.p_hidden = config.hidden_dropout_prob
        self.p_attn = config.attention_probs_dropout_prob

    def run(self, x2d, n_seq, S, mask):
        params = attention_param_list(self.attention.self, self.attention.output) + \
            ffn_param_list(self.intermediate, self.output)
        # dropout probabilities follow the nn.Dropout children so `m.p = 0` (parity tests) is honoured
        return ops.EncoderLayerFn.apply(x2d, n_seq, S, mask, self.attention.output.dropout.p,
                                        self.attention.self.dropout.p, self.training, *params)


def _layer_params(layer):
    return attention_param_list(layer.attention.self, layer.attention.output) + \
        ffn_param_list(layer.intermediate, layer.output)


class EncoderStack(nn.Module):
    """`encoder.layer.N` (reference modules/module_bert.py:267-281)."""

    def __init__(self, config):
        super(EncoderStack, self).__init__()
        self.layer = nn.ModuleList([EncoderLayer(config) for _ in range(config.num_hidden_layers)])

    def run(self, x2d, n_seq, S, mask, keep_all=False):
        outs = []
        cuts = self.__dict__.get("_cut_layers")   # univl_b200.ddp.PhasedBackward: cut the autograd graph at these layers
        for i, layer in enumerate(self.layer):
            if cuts and i in cuts and x2d.requires_grad:
                leaf = x2d.detach().requires_grad_(True)
                self.__dict__.setdefault("_cut_pairs", []).append((i, x2d, leaf))
                x2d = leaf
            x2d = layer.run(x2d, n_seq, S, mask)
            if keep_all:
                outs.append(x2d)
        return outs if keep_all else x2d

    def run_first_token(self, x2d, n_seq, S, mask, start=0):
        """-> [n_seq, H]: token 0 of the last layer's output, for consumers that read nothing else (pooler).  All layers
        but the last run in full; the last one computes only what token 0 needs (ops.EncoderLayerClsFn).  start: x2d
        is the output of layer start - 1 (the layers before it ran elsewhere)."""
        for layer in self.layer[start:-1]:
            x2d = layer.run(x2d, n_seq, S, mask)
        last = self.layer[-1]
        return ops.EncoderLayerClsFn.apply(x2d, n_seq, S, mask, last.attention.output.dropout.p,
                                           last.attention.self.dropout.p, last.training, *_layer_params(last))


class Pooler(nn.Module):
    """tanh(dense(h[:, 0])) (reference modules/module_bert.py:284-296)."""

    def __init__(self, config):
        super(Pooler, self).__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.activation = nn.Tanh()

    def pre_activation(self, h2d, n_seq, S):
        first = h2d.view(n_seq, S, -1)[:, 0]  # strided rows, read in place by TMA
        return ops.LinearFn.apply(first, self.dense.weight, self.dense.bias, False, True)

    def run(self, h2d, n_seq, S):
        return ops.TanhFn.apply(self.pre_activation(h2d, n_seq, S))


class HeadTransform(nn.Module):
    """LN(gelu(dense(x))) (reference modules/module_bert.py:298-312)."""

    def __init__(self, config):
        super(HeadTransform, self).__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = LayerNorm(config.hidden_size, eps=1e-12)

    def run(self, x2d):
        t = ops.LinearFn.apply(x2d, self.dense.weight, self.dense.bias, True, True)
        return ops.LayerNormFn.apply(t, self.LayerNorm.weight, self.LayerNorm.bias)


def as_rows(t3d):
    """[N, S, H] -> contiguous bf16 [N*S, H]"""
    n, s, h = t3d.shape
    return t3d.to(torch.bfloat16).contiguous().view(n * s, h)


def hidden_list(outs, n_seq, S):
    return [o.view(n_seq, S, -1) for o in outs]
