"""torch.autograd bindings of the C-ABI kernels (include/univl_b200.h).

Everything here is plumbing: allocate outputs with torch, hand raw device pointers to the library on the current
stream, keep what backward needs.  No arithmetic on the hot path is done by torch ops; the forward/backward
orchestration of a whole transformer block lives in ONE autograd.Function so a layer costs one autograd node and the
saved activations are exactly the tensors the backward kernels read.
"""
import math
import os

import torch

from . import lib
from . import runtime as rt
from .runtime import call, ptr

BF16 = torch.bfloat16
F32 = torch.float32
LN_EPS = 1e-12
HEADS = 12
LD_VOCAB_ALIGN = 64

EPI_BIAS, EPI_GELU, EPI_GELU_BWD, EPI_ADD, EPI_F32, EPI_ATOMIC = 0, 1, 2, 3, 4, 5


def _empty(shape, dtype, like):
    return torch.empty(shape, dtype=dtype, device=like.device)


def _zeros(shape, dtype, like):
    return torch.zeros(shape, dtype=dtype, device=like.device)


def _check2d(t, name):
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError("univl_b200: %s must be a row-major 2-D tensor (got shape %s strides %s)"
                           % (name, tuple(t.shape), t.stride()))


class GradSink:
    """Where parameter gradients are accumulated.  With a flat-gradient registration (univl_b200.optim.flatten) the
    backward kernels add straight into the flat fp32 views and autograd receives None for those parameters; otherwise
    each gradient is a fresh zero tensor returned through autograd (the reference's DistributedDataParallel wrapping
    keeps working).  Captured at forward time because backward runs outside the model context."""

    def __init__(self):
        self.flat = rt.current_sink()

    def one(self, param):
        """-> (fp32 accumulation tensor, value to return to autograd)"""
        if param is None:
            return None, None
        if self.flat is not None and self.flat.has(param):
            return self.flat.grad_view(param), None
        t = torch.zeros(param.shape, dtype=F32, device=param.device)
        return t, t

    def packed(self, params):
        """adjacent tensors (q/k/v) as one buffer -> (buffer, [values to return to autograd])"""
        if self.flat is not None and all(self.flat.has(p) for p in params):
            v = self.flat.grad_view_packed(params)
            if v is not None:
                return v, [None] * len(params)
        rows = sum(p.shape[0] for p in params)
        t = torch.zeros((rows,) + tuple(params[0].shape[1:]), dtype=F32, device=params[0].device)
        outs, r = [], 0
        for p in params:
            outs.append(t[r:r + p.shape[0]])
            r += p.shape[0]
        return t, outs


# ---------------------------------------------------------------------------------------------------------
# raw kernels
# ---------------------------------------------------------------------------------------------------------
def gemm(a, b, M, N, K, out, epi=EPI_BIAS, bias=None, aux_in=None, aux_out=None, a_mn=False, b_mn=False, alpha=1.0,
         block_n=0, split_k=0):
    _check2d(a, "gemm A"); _check2d(b, "gemm B"); _check2d(out, "gemm out")
    call("univl_gemm_bf16", a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn), M, N, K,
         out.data_ptr(), out.stride(0), epi, ptr(bias), ptr(aux_in), aux_in.stride(0) if aux_in is not None else 0,
         ptr(aux_out), aux_out.stride(0) if aux_out is not None else 0, float(alpha), block_n, split_k)
    return out


def linear_fwd(x, w16, bias, epi=EPI_BIAS, aux_out=None, out_dtype=BF16, ld_out=None):
    """y[T,N] = x[T,K] w16[N,K]^T + bias"""
    T, K = x.shape
    N = w16.shape[0]
    if ld_out is None:
        out = _empty((T, N), out_dtype, x)
    else:
        out = _empty((T, ld_out), out_dtype, x)[:, :N]
    return gemm(x, w16, T, N, K, out, epi=epi, bias=bias, aux_out=aux_out)


def linear_dgrad(dy, w16, epi=EPI_BIAS, aux_in=None):
    """dx[T,K] = dy[T,N] w16[N,K]  (+ fused epilogue)"""
    T, N = dy.shape
    K = w16.shape[1]
    out = _empty((T, K), BF16, dy)
    return gemm(dy, w16, T, K, N, out, epi=epi, aux_in=aux_in, b_mn=True)


def linear_wgrad(dy, x, dw=None):
    """dW[N,K] (+)= dy[T,N]^T x[T,K]   fp32, accumulated atomically (split-K)"""
    T, N = dy.shape
    K = x.shape[1]
    if dw is None:
        dw = _zeros((N, K), F32, dy)
    return gemm(dy, x, N, K, T, dw, epi=EPI_ATOMIC, a_mn=True, b_mn=True)


def colsum(x, out=None):
    rows, cols = x.shape
    if out is None:
        out = _zeros((cols,), F32, x)
    call("univl_colsum_bf16", x.data_ptr(), x.stride(0), out.data_ptr(), rows, cols)
    return out


def layernorm_fwd(x, res, gamma, beta, p=0.0, mode=0, seed=0, stream=0):
    rows, cols = x.shape
    y = _empty((rows, cols), BF16, x)
    mean = _empty((rows,), F32, x)
    rstd = _empty((rows,), F32, x)
    call("univl_layernorm_fwd", x.data_ptr(), ptr(res), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
         mean.data_ptr(), rstd.data_ptr(), rows, cols, LN_EPS, float(p), mode, seed, stream)
    return y, mean, rstd


def layernorm_bwd(dy, dy2, x, res, gamma, mean, rstd, p=0.0, mode=0, seed=0, stream=0, want_dbias=True,
                  want_dx=True, dgamma=None, dbeta=None, dbias=None):
    rows, cols = x.shape
    dx_res = _empty((rows, cols), BF16, x) if want_dx else None
    dx_dense = _empty((rows, cols), BF16, x) if (want_dx and p > 0.0 and mode == 1) else dx_res
    dgamma = _zeros((cols,), F32, x) if dgamma is None else dgamma
    dbeta = _zeros((cols,), F32, x) if dbeta is None else dbeta
    if dbias is None and want_dbias:
        dbias = _zeros((cols,), F32, x)
    call("univl_layernorm_bwd", dy.data_ptr(), ptr(dy2), x.data_ptr(), ptr(res), gamma.data_ptr(), mean.data_ptr(),
         rstd.data_ptr(), ptr(dx_res), ptr(dx_dense), dgamma.data_ptr(), dbeta.data_ptr(), ptr(dbias), rows, cols,
         float(p), mode, seed, stream)
    return dx_res, dx_dense, dgamma, dbeta, dbias


class MaskSpec:
    """Key-padding description for attention: concat(mask_a[i, :Wa], mask_b[j, :Fb]); (i, j) per sequence.
    all_pairs: number of pairing groups (include/univl_b200.h): 0 / False = aligned (i = j = sequence), 1 / True = every
    (i, j) pair, G = G micro-batches each pairing its own Na/G x Nb/G rows."""

    def __init__(self, mask_a=None, mask_b=None, all_pairs=False, causal=False):
        self.a = mask_a.contiguous() if mask_a is not None else None
        self.b = mask_b.contiguous() if mask_b is not None else None
        self.all_pairs = int(all_pairs)
        self.causal = bool(causal)
        for m in (self.a, self.b):
            if m is not None and m.dtype != torch.int64:
                raise RuntimeError("univl_b200: masks must be int64 (as the reference dataloaders emit them)")

    @property
    def Wa(self):
        return self.a.shape[1] if self.a is not None else 0

    @property
    def Fb(self):
        return self.b.shape[1] if self.b is not None else 0

    @property
    def Nb(self):
        return self.b.shape[0] if self.b is not None else 0


SHORT_ATTN_MAX_S = 256  # csrc/attention.cu keeps a head's whole K/V in shared memory up to this length


def _attention_entry(kind, Sq, Sk):
    """univl_attention_<kind> up to 256 tokens, the key-tiled univl_attention_long_<kind> (csrc/attention_long.cu,
    <= 1024 tokens) beyond"""
    if Sq > SHORT_ATTN_MAX_S or Sk > SHORT_ATTN_MAX_S:
        return "univl_attention_long_" + kind
    return "univl_attention_" + kind


def attention_fwd(q, k, v, n_seq, Sq, Sk, mask, p=0.0, seed=0, stream=0):
    """q/k/v: 2-D views whose columns [h*64, h*64+64) hold head h (row stride arbitrary)."""
    o = _empty((n_seq * Sq, HEADS * 64), BF16, q)
    lse = _empty((n_seq * HEADS * Sq,), F32, q)
    call(_attention_entry("fwd", Sq, Sk), q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
         v.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr(), ptr(mask.a), ptr(mask.b), mask.Wa, mask.Fb, mask.Nb,
         int(mask.all_pairs), n_seq, HEADS, Sq, Sk, int(mask.causal), 1.0 / math.sqrt(64.0), float(p), seed, stream)
    return o, lse


def fused_attention_supported(n_seq, S, H):
    """self-attention shapes the fused QKV-projection + attention kernel (csrc/fused_attn.cu) takes"""
    if os.environ.get("UNIVL_FUSED_ATTN", "1") == "0":
        return False
    from . import lib
    return bool(lib.load().univl_fused_qkv_attention_supported(int(n_seq), HEADS, int(S), int(H)))


def fused_qkv_attention_fwd(x, wqkv, bqkv, n_seq, S, mask, p=0.0, seed=0, stream=0, save_qkv=True):
    """ctx, lse, qkv = fused QKV projection + self-attention of x[T, H] (one wgmma kernel; q/k/v only reach HBM when
    `save_qkv` — the copy the backward pass reads)."""
    T, H = x.shape
    _check2d(x, "fused attention x"); _check2d(wqkv, "fused attention wqkv")
    o = _empty((T, H), BF16, x)
    lse = _empty((n_seq * HEADS * S,), F32, x)
    qkv = _empty((T, 3 * H), BF16, x) if save_qkv else None
    call("univl_fused_qkv_attention_fwd", x.data_ptr(), x.stride(0), wqkv.data_ptr(), wqkv.stride(0), bqkv.data_ptr(),
         ptr(qkv), 3 * H, o.data_ptr(), o.stride(0), lse.data_ptr(), ptr(mask.a), ptr(mask.b), mask.Wa, mask.Fb,
         mask.Nb, int(mask.all_pairs), n_seq, HEADS, S, int(mask.causal), 1.0 / math.sqrt(64.0), float(p), seed, stream)
    return o, lse, qkv


def fused_attention_bwd(qkv, o, lse, d_o, dqkv, n_seq, S, mask, p=0.0, seed=0, stream=0, dbias=None):
    """dqkv[T, 3H] = backward of the attention core on wgmma (csrc/fused_attn.cu) for the shapes the fused forward
    takes; dbias: optional contiguous fp32 [3H] the column sums are added to."""
    call("univl_fused_attention_bwd", qkv.data_ptr(), qkv.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr(),
         d_o.data_ptr(), d_o.stride(0), dqkv.data_ptr(), dqkv.stride(0), ptr(dbias), ptr(mask.a), ptr(mask.b), mask.Wa,
         mask.Fb, mask.Nb, int(mask.all_pairs), n_seq, HEADS, S, int(mask.causal), 1.0 / math.sqrt(64.0), float(p), seed,
         stream)


def attention_bwd(q, k, v, o, lse, d_o, dq, dk, dv, n_seq, Sq, Sk, mask, p=0.0, seed=0, stream=0, dbias=None,
                  rng_layout=0):
    """dbias: optional (dbq, dbk, dbv) fp32 [H] tensors; the kernel adds the column sums of dq / dk / dv (the projection
    bias gradients) to them, which saves the separate column-sum pass over the [T, 3H] gradient.
    rng_layout 1: the forward was the fused kernel (row-major dropout layout)."""
    dbq, dbk, dbv = dbias if dbias is not None else (None, None, None)
    entry = _attention_entry("bwd", Sq, Sk)
    # the fused forward (the only source of rng_layout 1) runs at S <= 128 only
    assert rng_layout == 0 or entry == "univl_attention_bwd", (rng_layout, Sq, Sk)
    call(entry, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
         o.data_ptr(), o.stride(0), lse.data_ptr(), d_o.data_ptr(), d_o.stride(0), dq.data_ptr(), dq.stride(0),
         dk.data_ptr(), dk.stride(0), dv.data_ptr(), dv.stride(0), ptr(mask.a), ptr(mask.b), mask.Wa, mask.Fb,
         mask.Nb, int(mask.all_pairs), n_seq, HEADS, Sq, Sk, int(mask.causal), 1.0 / math.sqrt(64.0), float(p), seed,
         stream, int(rng_layout), ptr(dbq), ptr(dbk), ptr(dbv))


def attention_pair_fwd(qkv_a, qkv_b, Na, Nb, Sq, mask, pairs=None):
    """Attention core of the Na x Nb sequences concat(a_i, b_j), p = i * Nb + j, reading Q/K/V from per-source
    projections (csrc/attention_pair.cu): qkv_a [Na*Wa, 3H] and qkv_b [Nb*Fb, 3H] hold q | k | v of every source row.
    Sq = Wa + Fb, or 1 for token 0 only.  No dropout.  -> ctx [Na*Nb*Sq, H].
    pairs: (text_index, video_index) int32 [P] on the device — the listed sequences p = (text_index[p], video_index[p])
    instead of the grid (univl_attention_pair_list_fwd), with mask holding the listed pairs' own rows -> [P*Sq, H]"""
    H = HEADS * 64
    if pairs is not None:
        ti, vi = pairs
        o = _empty((ti.numel() * Sq, H), BF16, qkv_a)
        call("univl_attention_pair_list_fwd", qkv_a.data_ptr(), qkv_a.stride(0), qkv_a[:, H:].data_ptr(),
             qkv_a.stride(0), qkv_a[:, 2 * H:].data_ptr(), qkv_a.stride(0), qkv_b.data_ptr(), qkv_b.stride(0),
             qkv_b[:, H:].data_ptr(), qkv_b.stride(0), qkv_b[:, 2 * H:].data_ptr(), qkv_b.stride(0), o.data_ptr(),
             o.stride(0), None, ti.data_ptr(), vi.data_ptr(), ptr(mask.a), ptr(mask.b), ti.numel(), mask.Wa, mask.Fb,
             HEADS, Sq, 1.0 / math.sqrt(64.0))
        return o
    o = _empty((Na * Nb * Sq, H), BF16, qkv_a)
    call("univl_attention_pair_fwd", qkv_a.data_ptr(), qkv_a.stride(0), qkv_a[:, H:].data_ptr(), qkv_a.stride(0),
         qkv_a[:, 2 * H:].data_ptr(), qkv_a.stride(0), qkv_b.data_ptr(), qkv_b.stride(0), qkv_b[:, H:].data_ptr(),
         qkv_b.stride(0), qkv_b[:, 2 * H:].data_ptr(), qkv_b.stride(0), o.data_ptr(), o.stride(0), None, ptr(mask.a),
         ptr(mask.b), Na, mask.Wa, Nb, mask.Fb, HEADS, Sq, 1.0 / math.sqrt(64.0))
    return o


def embed_src_rows_eval(a, N, W, pos, type_w, gamma, beta, out):
    """LayerNorm(a + pos[s] + type[0]) of every row of one source alone (aligned univl_embed_src_fwd, no dropout) into
    out [N*W, H].  With pos / type_w offset by the rows that precede the source in the pair sequence, these are exactly
    the source's rows of the all-pairs embedding, since that LayerNorm reads the row alone."""
    mean = _empty((N * W,), F32, a)
    rstd = _empty((N * W,), F32, a)
    call("univl_embed_src_fwd", a.data_ptr(), None, pos.data_ptr(), type_w.data_ptr(), gamma.data_ptr(),
         beta.data_ptr(), out.data_ptr(), mean.data_ptr(), rstd.data_ptr(), N, W, 0, 0, 0, a.shape[1], LN_EPS, 0.0,
         None, 0)
    return out


def pair_layer_eval(x, qkv_a, qkv_b, Na, Nb, S, mask, params, first_token, pairs=None):
    """An encoder layer over the Na x Nb pair sequences in evaluation (no dropout, no autograd) whose Q/K/V
    projections are given per source row, computed once per text row and once per video row instead of once per pair.
    x: the pair inputs [Na*Nb*S, H] (the residual of the attention block); params as EncoderLayerFn.  first_token: the
    layer is the stack's last and produces token 0 of every sequence only, as EncoderLayerClsFn -> [Na*Nb, H].
    Same arithmetic as EncoderLayerFn / EncoderLayerClsFn on the QKV-GEMM + attention-core path.  pairs: the listed
    sequences of attention_pair_fwd instead of the grid (x then holds their P*S rows)."""
    arena = rt.current()
    wa = dict(zip(ATT_KEYS, params[:10]))
    wf = dict(zip(FFN_KEYS, params[10:16]))
    drop = _Drop(0.0, 0.0, False)
    n_seq = pairs[0].numel() if pairs is not None else Na * Nb
    ctx = attention_pair_fwd(qkv_a, qkv_b, Na, Nb, 1 if first_token else S, mask, pairs)
    xq = x.view(n_seq, S, -1)[:, 0].contiguous() if first_token else x
    ao = linear_fwd(ctx, arena.bf16(wa["o"]), wa["bo"])
    y, _, _ = layernorm_fwd(ao, xq, wa["gamma"], wa["beta"], 0.0, 1, drop.seed, drop.stream())
    return ffn_block_fwd(y, wf, drop)[0]


# ---------------------------------------------------------------------------------------------------------
# FP8 evaluation (include/univl_b200.h: e4m3 codes with power-of-two block scales, forward only)
# ---------------------------------------------------------------------------------------------------------
E4M3 = torch.float8_e4m3fn
FP8_EPI_BIAS, FP8_EPI_GELU = 0, 1


def quantize_e4m3_rows(x):
    """bf16 [M, K] -> (e4m3 [M, K], fp32 scales [K/128, M]), one scale per (row, 128-column block)"""
    _check2d(x, "quantize_e4m3_rows x")
    M, K = x.shape
    q = _empty((M, K), E4M3, x)
    s = _empty((K // 128, M), F32, x)
    call("univl_quantize_e4m3_rows", x.data_ptr(), x.stride(0), q.data_ptr(), q.stride(0), s.data_ptr(), M, K)
    return q, s


def quantize_e4m3_blocks(w, q=None, s=None):
    """fp32 [N, K] -> (e4m3 [N, K], fp32 scales [N/128, K/128]), one scale per 128 x 128 block; q / s: optional
    outputs (row slices of larger buffers)"""
    _check2d(w, "quantize_e4m3_blocks w")
    N, K = w.shape
    q = _empty((N, K), E4M3, w) if q is None else q
    s = _empty((N // 128, K // 128), F32, w) if s is None else s
    call("univl_quantize_e4m3_blocks", w.data_ptr(), w.stride(0), q.data_ptr(), q.stride(0), s.data_ptr(), N, K)
    return q, s


def gemm_fp8(a, a_scale, b, b_scale, bias, gelu=False):
    """a e4m3 [M, K] with a_scale [K/128, M], b e4m3 [N, K] with b_scale [N/128, K/128] ->
    bf16 [M, N] = a b^T + bias, or with gelu (e4m3 [M, N], scales [N/128, M]) of gelu_erf(a b^T + bias)"""
    _check2d(a, "gemm_fp8 A"); _check2d(b, "gemm_fp8 B")
    M, K = a.shape
    N = b.shape[0]
    if gelu:
        out = _empty((M, N), E4M3, a)
        out_s = _empty((N // 128, M), F32, a)
    else:
        out = _empty((M, N), BF16, a)
        out_s = None
    call("univl_gemm_fp8", a.data_ptr(), a.stride(0), a_scale.data_ptr(), b.data_ptr(), b.stride(0),
         b_scale.data_ptr(), M, N, K, FP8_EPI_GELU if gelu else FP8_EPI_BIAS, bias.data_ptr(), out.data_ptr(),
         out.stride(0), ptr(out_s))
    return (out, out_s) if gelu else out


def fp8_layer_weights(params, names):
    """The e4m3 weights (with their block scales) of one encoder layer's FP8 GEMMs, quantized from the fp32 parameters
    (params as EncoderLayerFn) -> {name: (codes, scales)} for the names asked for: "qkv" (Q/K/V projection), "kv" (the
    last layer's K/V projection), "o" (attention output), "w1", "w2" (FFN)."""
    wa = dict(zip(ATT_KEYS, params[:10]))
    wf = dict(zip(FFN_KEYS, params[10:16]))
    H = wa["q"].shape[1]

    def stacked(ws):
        q = _empty((len(ws) * H, H), E4M3, ws[0])
        s = _empty((len(ws) * H // 128, H // 128), F32, ws[0])
        for i, w in enumerate(ws):
            quantize_e4m3_blocks(w, q[i * H:(i + 1) * H], s[i * H // 128:(i + 1) * H // 128])
        return q, s

    make = {"qkv": lambda: stacked((wa["q"], wa["k"], wa["v"])), "kv": lambda: stacked((wa["k"], wa["v"])),
            "o": lambda: quantize_e4m3_blocks(wa["o"]), "w1": lambda: quantize_e4m3_blocks(wf["w1"]),
            "w2": lambda: quantize_e4m3_blocks(wf["w2"])}
    return {n: make[n]() for n in names}


def _fp8_layer_tail(ctx, x, params, qw):
    """attention output dense + LayerNorm(x) and the FFN block of an encoder layer in evaluation, the three dense GEMMs
    in FP8: ctx the attention context [T, H], x the layer input (the attention block's residual)"""
    wa = dict(zip(ATT_KEYS, params[:10]))
    wf = dict(zip(FFN_KEYS, params[10:16]))
    drop = _Drop(0.0, 0.0, False)
    ao = gemm_fp8(*quantize_e4m3_rows(ctx), *qw["o"], wa["bo"])
    y, _, _ = layernorm_fwd(ao, x, wa["gamma"], wa["beta"], 0.0, 1, drop.seed, drop.stream())
    h, hs = gemm_fp8(*quantize_e4m3_rows(y), *qw["w1"], wf["b1"], gelu=True)
    fo = gemm_fp8(h, hs, *qw["w2"], wf["b2"])
    out, _, _ = layernorm_fwd(fo, y, wf["gamma"], wf["beta"], 0.0, 1, drop.seed, drop.stream())
    return out


def pair_layer_eval_fp8(x, qkv_a, qkv_b, Na, Nb, S, mask, params, qw, pairs=None):
    """pair_layer_eval for a layer that is not the stack's last, its dense GEMMs over the pair tokens in FP8
    (qw holds "o", "w1", "w2" of fp8_layer_weights).  The attention core and the LayerNorms stay bf16."""
    ctx = attention_pair_fwd(qkv_a, qkv_b, Na, Nb, S, mask, pairs)
    return _fp8_layer_tail(ctx, x, params, qw)


def encoder_layer_eval_fp8(x, n_seq, S, mask, params, qw):
    """EncoderLayerFn in evaluation with the Q/K/V projection, attention output and FFN GEMMs in FP8 (qw holds "qkv",
    "o", "w1", "w2" of fp8_layer_weights)"""
    wa = dict(zip(ATT_KEYS, params[:10]))
    H = x.shape[1]
    qkv = gemm_fp8(*quantize_e4m3_rows(x), *qw["qkv"], rt.packed_bias(wa["bq"], wa["bk"], wa["bv"]))
    drop = _Drop(0.0, 0.0, False)
    ctx, _ = attention_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], n_seq, S, S, mask, 0.0, drop.seed,
                           drop.stream())
    return _fp8_layer_tail(ctx, x, params, qw)


def cls_layer_eval_fp8(x, n_seq, S, mask, params, qw):
    """EncoderLayerClsFn in evaluation with the K/V projection of all n_seq * S rows in FP8 (qw holds "kv" of
    fp8_layer_weights); everything on the n_seq token-0 rows (Q, attention output, FFN) stays bf16
    -> [n_seq, H]"""
    arena = rt.current()
    wa = dict(zip(ATT_KEYS, params[:10]))
    wf = dict(zip(FFN_KEYS, params[10:16]))
    drop = _Drop(0.0, 0.0, False)
    H = x.shape[1]
    x0 = x.view(n_seq, S, H)[:, 0].contiguous()
    kv = gemm_fp8(*quantize_e4m3_rows(x), *qw["kv"], rt.packed_bias(wa["bk"], wa["bv"]))
    q = linear_fwd(x0, arena.bf16_qkv(wa["q"], wa["k"], wa["v"])[:H], wa["bq"])
    ctx, _ = attention_fwd(q, kv[:, :H], kv[:, H:], n_seq, 1, S, mask, 0.0, drop.seed, drop.stream())
    ao = linear_fwd(ctx, arena.bf16(wa["o"]), wa["bo"])
    y, _, _ = layernorm_fwd(ao, x0, wa["gamma"], wa["beta"], 0.0, 1, drop.seed, drop.stream())
    return ffn_block_fwd(y, wf, drop)[0]


# ---------------------------------------------------------------------------------------------------------
# packed evaluation: the pair sequences on their valid tokens alone (include/univl_b200.h univl_attention_varlen_fwd)
# ---------------------------------------------------------------------------------------------------------
I32 = torch.int32


def _exclusive_cumsum(n):
    out = torch.zeros(n.numel() + 1, dtype=torch.int64, device=n.device)
    torch.cumsum(n, 0, out=out[1:])
    return out


class VarlenSeqs:
    """Variable-length sequences of univl_attention_varlen_fwd / univl_gather_rows_varlen: cu int32 [n_seq + 1] (sequence
    p is rows [cu[p], cu[p + 1]) of the packed layout), `total` = cu[-1] and `max_sk` (host ints, max_sk >= every
    sequence's length); under pair addressing also the int32 index lists idx_a / idx_b and the per-sequence start_a /
    start_b / len_a (all None: packed addressing)."""

    def __init__(self, cu, total, max_sk, idx_a=None, idx_b=None, start_a=None, start_b=None, len_a=None):
        self.cu, self.total, self.max_sk = cu, int(total), int(max_sk)
        self.idx_a, self.idx_b, self.start_a, self.start_b, self.len_a = idx_a, idx_b, start_a, start_b, len_a
        self.n_seq = cu.numel() - 1

    def packed(self):
        """the same sequences under packed addressing: their rows stored back to back"""
        return VarlenSeqs(self.cu, self.total, self.max_sk)

    def index_args(self):
        return (ptr(self.idx_a), ptr(self.idx_b), ptr(self.start_a), ptr(self.start_b), ptr(self.len_a),
                self.cu.data_ptr())


def _valid_rows(m, n):
    """int32 indices of the n nonzero entries of the flat bool m, ascending, with no device-to-host sync (unlike
    nonzero(), which must learn n first): entry k goes to slot cumsum(m)[k] - 1, the others to a spare slot n"""
    flat = m.reshape(-1)
    slot = torch.where(flat, torch.cumsum(flat, 0) - 1, n)
    out = torch.empty(n + 1, dtype=I32, device=m.device)
    out.scatter_(0, slot, torch.arange(flat.numel(), dtype=I32, device=m.device))
    return out[:n]


class PairPacking:
    """The packed layout of the (text i, video j) pair sequences of one evaluation call: pair (i, j) is text i's valid
    tokens then video j's, each at its original row (so its original position), and nothing else.  Built from the int64
    masks text_mask [Nt, W] and video_mask [Nv, F] with torch ops on their device and one device-to-host copy: the
    per-row counts (len_t / len_v below), which choose the tiles, and the token-0 flag.
      token0_valid    every text row's token 0 is valid (the packed layout needs it: the pooler reads token 0)
      idx_t / idx_v   int32: the valid rows i * W + s of the text source and j * F + s of the video source, ascending
      start_t / start_v  int32 [Nt] / [Nv]: where row i's (j's) entries begin in idx_t (idx_v)
      len_t / len_v   host lists of the valid-token counts
      max_sk          longest pair of the call (max len_t + max len_v).  Every tile passes this one value, so which
                      attention kernel a pair runs on does not depend on the tiling."""

    def __init__(self, text_mask, video_mask):
        tm, vm = text_mask != 0, video_mask != 0
        self.text_shape, self.video_shape = tuple(tm.shape), tuple(vm.shape)
        nt, nv = tm.sum(1), vm.sum(1)
        token0 = tm[:, 0].all().view(1) if tm.shape[1] else torch.zeros(1, dtype=torch.bool, device=tm.device)
        host = torch.cat([nt, nv, token0.long()]).cpu().tolist()  # the one device-to-host copy
        Nt = tm.shape[0]
        self.len_t, self.len_v = host[:Nt], host[Nt:-1]
        self.token0_valid = bool(host[-1])
        self.idx_t = _valid_rows(tm, sum(self.len_t))
        self.idx_v = _valid_rows(vm, sum(self.len_v))
        self.start_t = _exclusive_cumsum(nt)[:-1].to(I32)
        self.start_v = _exclusive_cumsum(nv)[:-1].to(I32)
        self.n_t, self.n_v = nt.to(I32), nv.to(I32)
        self.max_sk = max(self.len_t, default=0) + max(self.len_v, default=0)

    def tokens(self, t0, t1, v0, v1):
        """packed rows of the tile of text rows [t0, t1) x video rows [v0, v1)"""
        return (v1 - v0) * sum(self.len_t[t0:t1]) + (t1 - t0) * sum(self.len_v[v0:v1])

    def tile(self, t0, t1, v0, v1):
        """VarlenSeqs (pair addressing) of the pairs p = (i - t0) * (v1 - v0) + (j - v0) of that tile"""
        nt, nv = t1 - t0, v1 - v0
        len_a = self.n_t[t0:t1].repeat_interleave(nv)
        len_b = self.n_v[v0:v1].repeat(nt)
        cu = _exclusive_cumsum(len_a.long() + len_b.long()).to(I32)
        return VarlenSeqs(cu, self.tokens(t0, t1, v0, v1), self.max_sk, self.idx_t, self.idx_v,
                          self.start_t[t0:t1].repeat_interleave(nv), self.start_v[v0:v1].repeat(nt), len_a)

    def pairs(self, text_index, video_index):
        """VarlenSeqs (pair addressing) of the listed pairs p = (text_index[p], video_index[p]) (int64 or int32
        tensors on the masks' device, in range), in list order.  max_sk stays the call's, so each pair runs on the
        attention kernel the grid would run it on.  `total` costs one device-to-host copy."""
        ti, vi = text_index.long(), video_index.long()
        len_a = self.n_t[ti]
        cu = _exclusive_cumsum(len_a.long() + self.n_v[vi].long())
        return VarlenSeqs(cu.to(I32), int(cu[-1]), self.max_sk, self.idx_t, self.idx_v, self.start_t[ti],
                          self.start_v[vi], len_a)


def embed_text_packed(ids, type_ids, idx, S, word, pos, type_w, gamma, beta):
    """EmbedTextFn in evaluation on packed rows: row r is token idx[r] (int32, = i * S + s) of the [n, S] ids /
    type_ids (type_ids None: type 0) -> bf16 [idx.numel(), H]"""
    y = _empty((idx.numel(), word.shape[1]), BF16, word)
    call("univl_embed_text_packed_fwd", ids.data_ptr(), ptr(type_ids), idx.data_ptr(), idx.numel(), S,
         word.data_ptr(), pos.data_ptr(), ptr(type_w), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
         word.shape[1], word.shape[0], LN_EPS)
    return y


def video_norm_rows(video2d, idx, gamma, beta):
    """VideoNormFn's forward on the fp32 rows idx (int32) of video2d [rows, video_dim] -> bf16 [idx.numel(), video_dim]"""
    y = _empty((idx.numel(), video2d.shape[1]), BF16, video2d)
    call("univl_layernorm_f32_rows_fwd", video2d.data_ptr(), idx.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
         y.data_ptr(), idx.numel(), video2d.shape[1], LN_EPS)
    return y


def embed_src_packed(x, idx, S, pos, gamma, beta):
    """EmbedSrcFn in evaluation (one aligned source, the visual embeddings) on packed rows: x [T, H] holds token idx[r]
    (= j * S + s) -> bf16 LN(x[r] + pos[s]) [T, H]"""
    y = _empty(x.shape, BF16, x)
    call("univl_embed_src_packed_fwd", x.data_ptr(), idx.data_ptr(), x.shape[0], S, pos.data_ptr(), gamma.data_ptr(),
         beta.data_ptr(), y.data_ptr(), x.shape[1], LN_EPS)
    return y


def meanpool_packed(x, cu, idx, S, skip_first, guard_zero, l2norm):
    """MeanPoolFn's forward on packed rows: sequence n is rows [cu[n], cu[n + 1]) of x (int32 cu), row r at position
    idx[r] mod S -> fp32 [cu.numel() - 1, H], equal bit for bit to MeanPoolFn on the padded layout's rows"""
    N, H = cu.numel() - 1, x.shape[1]
    out = _empty((N, H), F32, cu)
    call("univl_meanpool_packed_fwd", x.data_ptr(), cu.data_ptr(), idx.data_ptr(), out.data_ptr(), N, S, H,
         int(skip_first), int(guard_zero), int(l2norm))
    return out


def padded_pair_seqs(text_index, video_index, Nt, W, Nv, F):
    """VarlenSeqs (pair addressing) of the listed pairs at all W + F tokens, over the rows of the per-source sources
    [Nt*W, *] (text) and [Nv*F, *] (video): pair p's rows are text rows text_index[p] * W + [0, W) then video rows
    video_index[p] * F + [0, F) — the padded layout's pair sequence, for gather_rows_varlen"""
    dev = text_index.device
    P, S = text_index.numel(), W + F
    cu = torch.arange(P + 1, dtype=I32, device=dev) * S
    idx_a = torch.arange(Nt * W, dtype=I32, device=dev)
    idx_b = torch.arange(Nv * F, dtype=I32, device=dev)
    return VarlenSeqs(cu, P * S, S, idx_a, idx_b, (text_index.long() * W).to(I32), (video_index.long() * F).to(I32),
                      torch.full((P,), W, dtype=I32, device=dev))


def attention_varlen_fwd(q, k, v, seqs, q_first, qb=None, kb=None, vb=None):
    """Attention core of the variable-length sequences `seqs` (csrc/attention_varlen.cu), no mask, no dropout.  q/k/v
    (and qb/kb/vb, the second source under pair addressing): 2-D views whose columns [h*64, h*64+64) hold head h.
    q_first: token 0 only (under packed addressing q holds one row per sequence) -> ctx [n_seq, H]; else
    [seqs.total, H] in packed order"""
    o = _empty((seqs.n_seq if q_first else seqs.total, HEADS * 64), BF16, q)
    if o.shape[0] == 0:
        return o
    b = (qb, kb, vb) if seqs.idx_a is not None else (None, None, None)
    call("univl_attention_varlen_fwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
         v.stride(0), ptr(b[0]), b[0].stride(0) if b[0] is not None else 0, ptr(b[1]),
         b[1].stride(0) if b[1] is not None else 0, ptr(b[2]), b[2].stride(0) if b[2] is not None else 0,
         *seqs.index_args(), seqs.n_seq, seqs.max_sk, HEADS, int(q_first), o.data_ptr(), o.stride(0), None,
         1.0 / math.sqrt(64.0))
    return o


def gather_rows_varlen(a, b, seqs, q_first):
    """the rows of `seqs` (a, and b under pair addressing) in packed order -> [seqs.total, cols], or with q_first row 0
    of every sequence -> [n_seq, cols]"""
    _check2d(a, "gather_rows_varlen a")
    out = _empty((seqs.n_seq if q_first else seqs.total, a.shape[1]), BF16, a)
    if out.shape[0] == 0:
        return out
    call("univl_gather_rows_varlen", a.data_ptr(), a.stride(0), ptr(b), b.stride(0) if b is not None else 0,
         *seqs.index_args(), seqs.n_seq, int(q_first), a.shape[1], out.data_ptr(), out.stride(0))
    return out


def attention_decode_fwd(q, kv, key_rows, n_keys, list_of_query=None, out=None, lse=None):
    """Single-token attention over indexed key rows (csrc/attention_decode.cu), no mask, no dropout.  q [n_q, 768];
    kv [*, >= 1536] with k | v in its first 1536 columns; key_rows int32 [n_lists, >= max keys] (row-major, any row
    stride); n_keys int32 [n_lists]; list_of_query int32 [n_q] or None (query r reads list r).  -> ctx [n_q, 768]
    (into `out` when given); lse: optional fp32 [n_q, 12]"""
    _check2d(q, "attention_decode q"); _check2d(kv, "attention_decode kv"); _check2d(key_rows, "attention_decode key_rows")
    for t, name in ((key_rows, "key_rows"), (n_keys, "n_keys"), (list_of_query, "list_of_query")):
        if t is not None and t.dtype != I32:
            raise RuntimeError("univl_b200: attention_decode %s must be int32" % name)
    o = _empty((q.shape[0], HEADS * 64), BF16, q) if out is None else out
    _check2d(o, "attention_decode out")
    call("univl_attention_decode_fwd", q.data_ptr(), q.stride(0), kv.data_ptr(), kv.stride(0), key_rows.data_ptr(),
         key_rows.stride(0), n_keys.data_ptr(), ptr(list_of_query), q.shape[0], HEADS, o.data_ptr(), o.stride(0),
         ptr(lse), 1.0 / math.sqrt(64.0))
    return o


def _split_qkv(qkv):
    H = qkv.shape[1] // 3
    return qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]


def _attn_out(ctx, x, params):
    """LayerNorm(ctx Wo^T + bo + x): the attention block's output in evaluation, bf16 (as pair_layer_eval)"""
    wa = dict(zip(ATT_KEYS, params[:10]))
    drop = _Drop(0.0, 0.0, False)
    ao = linear_fwd(ctx, rt.current().bf16(wa["o"]), wa["bo"])
    return layernorm_fwd(ao, x, wa["gamma"], wa["beta"], 0.0, 1, drop.seed, drop.stream())[0]


def _ffn(y, params):
    return ffn_block_fwd(y, dict(zip(FFN_KEYS, params[10:16])), _Drop(0.0, 0.0, False))[0]


# The packed layer functions below free the attention context (and the Q/K/V rows, and the gathered residual) before
# the FFN, which keeps a packed tile's peak below a padded tile's of the same token count by more than the per-source
# embedding rows the packed layout keeps for the whole call.
def pair_layer_eval_packed(x_a, x_b, qkv_a, qkv_b, seqs, params, first_token, qw=None):
    """pair_layer_eval on the packed layout: the first cross layer of the tile's pairs `seqs` (pair addressing), its
    Q/K/V read by index from the per-source projections qkv_a / qkv_b and its residual rows gathered from the
    per-source embedding rows x_a / x_b.  first_token: token 0 only -> [n_seq, H]; else [seqs.total, H].
    qw: the FP8 weights "o", "w1", "w2" (pair_layer_eval_fp8), or None for bf16."""
    xq = gather_rows_varlen(x_a, x_b, seqs, first_token)
    ctx = attention_varlen_fwd(*_split_qkv(qkv_a), seqs, first_token, *_split_qkv(qkv_b))
    if qw is not None:
        return _fp8_layer_tail(ctx, xq, params, qw)
    y = _attn_out(ctx, xq, params)
    del ctx, xq
    return _ffn(y, params)


def encoder_layer_eval_packed(x, seqs, params, qw=None):
    """a middle encoder layer in evaluation on the packed rows x [seqs.total, H]: QKV GEMM, varlen self-attention of
    every sequence, tail.  qw: the FP8 weights "qkv", "o", "w1", "w2" (encoder_layer_eval_fp8), or None for bf16."""
    wa = dict(zip(ATT_KEYS, params[:10]))
    bias = rt.packed_bias(wa["bq"], wa["bk"], wa["bv"])
    if qw is None:
        qkv = linear_fwd(x, rt.current().bf16_qkv(wa["q"], wa["k"], wa["v"]), bias)
    else:
        qkv = gemm_fp8(*quantize_e4m3_rows(x), *qw["qkv"], bias)
    ctx = attention_varlen_fwd(*_split_qkv(qkv), seqs.packed(), False)
    del qkv
    if qw is not None:
        return _fp8_layer_tail(ctx, x, params, qw)
    y = _attn_out(ctx, x, params)
    del ctx
    return _ffn(y, params)


def cls_layer_eval_packed(x, seqs, params, qw=None):
    """the last encoder layer in evaluation on the packed rows x [seqs.total, H], token 0 of every sequence only
    (EncoderLayerClsFn / cls_layer_eval_fp8): K/V GEMM on every packed row (FP8 with qw's "kv"), the Q projection,
    attention and tail on the n_seq token-0 rows, bf16 -> [n_seq, H]"""
    arena = rt.current()
    wa = dict(zip(ATT_KEYS, params[:10]))
    H = x.shape[1]
    wqkv = arena.bf16_qkv(wa["q"], wa["k"], wa["v"])
    bias = rt.packed_bias(wa["bk"], wa["bv"])
    if qw is None:
        kv = linear_fwd(x, wqkv[H:], bias)
    else:
        kv = gemm_fp8(*quantize_e4m3_rows(x), *qw["kv"], bias)
    packed = seqs.packed()
    x0 = gather_rows_varlen(x, None, packed, True)
    q = linear_fwd(x0, wqkv[:H], wa["bq"])
    ctx = attention_varlen_fwd(q, kv[:, :H], kv[:, H:], packed, True)
    del kv
    return _ffn(_attn_out(ctx, x0, params), params)


# ---------------------------------------------------------------------------------------------------------
# transformer blocks (forward keeps a dict of saved tensors; backward consumes it)
# ---------------------------------------------------------------------------------------------------------
class _Drop:
    """dropout bookkeeping of one block: probability, seed and a fresh Philox stream id per site"""

    def __init__(self, p_hidden, p_attn, training):
        arena = rt.current()
        self.ph = float(p_hidden) if training else 0.0
        self.pa = float(p_attn) if training else 0.0
        self.seed = arena.seed
        self.arena = arena
        self.epoch = arena.epoch_host

    def stream(self):
        return self.arena.next_stream()


def attn_block_fwd(xq, xkv, n_seq, Sq, Sk, mask, w, drop, need_bwd=True):
    """LayerNorm(dropout(dense(MHA(xq, xkv))) + xq)   (reference modules/module_bert.py:220-224).
    w: dict(q,k,v,o weights fp32 params; bq,bk,bv,bo; gamma,beta).
    Self-attention with S % 16 == 0, S <= 128 runs the fused QKV-projection + attention kernel (the [T,3H] projections
    reach HBM only when a backward pass will read them); other shapes use the QKV GEMM + attention-core pair."""
    arena = rt.current()
    H = xq.shape[1]
    self_attn = xkv is xq
    sv = {"self": self_attn, "fused": False}
    wqkv = arena.bf16_qkv(w["q"], w["k"], w["v"])
    ctx = None
    if self_attn and fused_attention_supported(n_seq, Sq, H):
        sa, sd = drop.stream(), drop.stream()
        ctx, lse, qkv = fused_qkv_attention_fwd(xq, wqkv, rt.packed_bias(w["bq"], w["bk"], w["bv"]), n_seq, Sq, mask,
                                                drop.pa, drop.seed, sa, save_qkv=need_bwd)
        sv["qkv"] = qkv
        sv["fused"] = True
    elif self_attn:
        qkv = linear_fwd(xq, wqkv, rt.packed_bias(w["bq"], w["bk"], w["bv"]))
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
        sv["qkv"] = qkv
    else:
        q = linear_fwd(xq, wqkv[:H], w["bq"])
        kv = linear_fwd(xkv, wqkv[H:], rt.packed_bias(w["bk"], w["bv"]))
        k, v = kv[:, :H], kv[:, H:]
        sv["q"], sv["kv"] = q, kv
    if ctx is None:
        sa, sd = drop.stream(), drop.stream()
        ctx, lse = attention_fwd(q, k, v, n_seq, Sq, Sk, mask, drop.pa, drop.seed, sa)
    ao = linear_fwd(ctx, arena.bf16(w["o"]), w["bo"])
    y, mean, rstd = layernorm_fwd(ao, xq, w["gamma"], w["beta"], drop.ph, 1, drop.seed, sd)
    sv.update(xq=xq, xkv=xkv, ctx=ctx, lse=lse, ao=ao, mean=mean, rstd=rstd, sa=sa, sd=sd, n_seq=n_seq, Sq=Sq, Sk=Sk,
              mask=mask, pa=drop.pa, ph=drop.ph, seed=drop.seed, wqkv=wqkv, wo=arena.bf16(w["o"]),
              gamma=w["gamma"], w=w, sink=GradSink(), arena=arena, epoch=drop.epoch)
    return y, sv


def attn_block_bwd(dy, dy2, sv, need_dxkv=True):
    """returns dxq, dxkv (None for self-attention: folded into dxq) and the autograd return values per ATT_KEYS"""
    H = sv["xq"].shape[1]
    sv["arena"].check_epoch(sv["epoch"], max(sv["pa"], sv["ph"]))
    w, sink = sv["w"], sv["sink"]
    dgamma, r_gamma = sink.one(w["gamma"])
    dbeta, r_beta = sink.one(w["beta"])
    dbo, r_bo = sink.one(w["bo"])
    g, gd, _, _, _ = layernorm_bwd(dy, dy2, sv["ao"], sv["xq"], sv["gamma"], sv["mean"], sv["rstd"], sv["ph"], 1,
                                   sv["seed"], sv["sd"], dgamma=dgamma, dbeta=dbeta, dbias=dbo)
    dwo, r_o = sink.one(w["o"])
    linear_wgrad(gd, sv["ctx"], dwo)
    dctx = linear_dgrad(gd, sv["wo"])
    T, Tk = sv["xq"].shape[0], sv["xkv"].shape[0]
    dwqkv, r_w = sink.packed((w["q"], w["k"], w["v"]))
    dbqkv, r_b = sink.packed((w["bq"], w["bk"], w["bv"]))
    if sv["self"]:
        qkv = sv["qkv"]
        dqkv = _empty((T, 3 * H), BF16, dy)
        if sv["fused"] and os.environ.get("UNIVL_FUSED_ATTN_BWD", "1") != "0":
            fused_attention_bwd(qkv, sv["ctx"], sv["lse"], dctx, dqkv, sv["n_seq"], sv["Sq"], sv["mask"], sv["pa"],
                                sv["seed"], sv["sa"], dbias=dbqkv)
        else:
            attention_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], sv["ctx"], sv["lse"], dctx, dqkv[:, :H],
                          dqkv[:, H:2 * H], dqkv[:, 2 * H:], sv["n_seq"], sv["Sq"], sv["Sk"], sv["mask"], sv["pa"],
                          sv["seed"], sv["sa"], dbias=(dbqkv[:H], dbqkv[H:2 * H], dbqkv[2 * H:]),
                          rng_layout=1 if sv["fused"] else 0)
        linear_wgrad(dqkv, sv["xq"], dwqkv)
        dxq = linear_dgrad(dqkv, sv["wqkv"], epi=EPI_ADD, aux_in=g)
        dxkv = None
    else:
        q, kv = sv["q"], sv["kv"]
        dq = _empty((T, H), BF16, dy)
        dkv = _empty((Tk, 2 * H), BF16, dy)
        attention_bwd(q, kv[:, :H], kv[:, H:], sv["ctx"], sv["lse"], dctx, dq, dkv[:, :H], dkv[:, H:], sv["n_seq"],
                      sv["Sq"], sv["Sk"], sv["mask"], sv["pa"], sv["seed"], sv["sa"],
                      dbias=(dbqkv[:H], dbqkv[H:2 * H], dbqkv[2 * H:]))
        linear_wgrad(dq, sv["xq"], dwqkv[:H])
        linear_wgrad(dkv, sv["xkv"], dwqkv[H:])
        dxq = linear_dgrad(dq, sv["wqkv"][:H], epi=EPI_ADD, aux_in=g)
        dxkv = linear_dgrad(dkv, sv["wqkv"][H:]) if need_dxkv else None
    rets = {"q": r_w[0], "k": r_w[1], "v": r_w[2], "bq": r_b[0], "bk": r_b[1], "bv": r_b[2], "o": r_o, "bo": r_bo,
            "gamma": r_gamma, "beta": r_beta}
    return dxq, dxkv, rets


def ffn_block_fwd(x, w, drop):
    """LayerNorm(dropout(dense2(gelu(dense1(x)))) + x)   (reference modules/module_bert.py:233-236, :246-250)"""
    arena = rt.current()
    w1, w2 = arena.bf16(w["w1"]), arena.bf16(w["w2"])
    T = x.shape[0]
    pre = _empty((T, w1.shape[0]), BF16, x)
    h = linear_fwd(x, w1, w["b1"], epi=EPI_GELU, aux_out=pre)
    fo = linear_fwd(h, w2, w["b2"])
    sd = drop.stream()
    y, mean, rstd = layernorm_fwd(fo, x, w["gamma"], w["beta"], drop.ph, 1, drop.seed, sd)
    sv = dict(x=x, pre=pre, h=h, fo=fo, mean=mean, rstd=rstd, sd=sd, ph=drop.ph, seed=drop.seed, w1=w1, w2=w2,
              gamma=w["gamma"], w=w, sink=GradSink(), arena=arena, epoch=drop.epoch)
    return y, sv


def ffn_block_bwd(dy, sv):
    """returns (g_residual, d_x_from_dense) — the caller sums them inside the next LayerNorm backward — and the
    autograd return values per FFN_KEYS"""
    w, sink = sv["w"], sv["sink"]
    sv["arena"].check_epoch(sv["epoch"], sv["ph"])
    dgamma, r_gamma = sink.one(w["gamma"])
    dbeta, r_beta = sink.one(w["beta"])
    db2, r_b2 = sink.one(w["b2"])
    g, gd, _, _, _ = layernorm_bwd(dy, None, sv["fo"], sv["x"], sv["gamma"], sv["mean"], sv["rstd"], sv["ph"], 1,
                                   sv["seed"], sv["sd"], dgamma=dgamma, dbeta=dbeta, dbias=db2)
    dw2, r_w2 = sink.one(w["w2"])
    linear_wgrad(gd, sv["h"], dw2)
    dpre = linear_dgrad(gd, sv["w2"], epi=EPI_GELU_BWD, aux_in=sv["pre"])
    db1, r_b1 = sink.one(w["b1"])
    colsum(dpre, db1)
    dw1, r_w1 = sink.one(w["w1"])
    linear_wgrad(dpre, sv["x"], dw1)
    dx = linear_dgrad(dpre, sv["w1"])
    return g, dx, {"w1": r_w1, "b1": r_b1, "w2": r_w2, "b2": r_b2, "gamma": r_gamma, "beta": r_beta}


ATT_KEYS = ("q", "bq", "k", "bk", "v", "bv", "o", "bo", "gamma", "beta")
FFN_KEYS = ("w1", "b1", "w2", "b2", "gamma", "beta")


class EncoderLayerFn(torch.autograd.Function):
    """One BertLayer / VisualLayer / CrossLayer (reference modules/module_bert.py:253-264) as a single autograd node.
    args: x[T,H] bf16, then 10 attention params (ATT_KEYS order), then 6 FFN params (FFN_KEYS order)."""

    @staticmethod
    def forward(ctx, x, n_seq, S, mask, p_hidden, p_attn, training, *params):
        wa = dict(zip(ATT_KEYS, params[:10]))
        wf = dict(zip(FFN_KEYS, params[10:16]))
        drop = _Drop(p_hidden, p_attn, training)
        y1, sva = attn_block_fwd(x, x, n_seq, S, S, mask, wa, drop, need_bwd=any(ctx.needs_input_grad))
        y2, svf = ffn_block_fwd(y1, wf, drop)
        ctx.sva, ctx.svf = sva, svf
        return y2

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        g2, dy1, gf = ffn_block_bwd(dy, ctx.svf)
        dx, _, ga = attn_block_bwd(dy1, g2, ctx.sva)
        ctx.sva = ctx.svf = None
        return (dx, None, None, None, None, None, None) + tuple(ga[k] for k in ATT_KEYS) + \
            tuple(gf[k] for k in FFN_KEYS)


class EncoderLayerClsFn(torch.autograd.Function):
    """The LAST layer of an encoder stack whose only consumer reads token 0 of every sequence (the cross encoder under
    `_cross_similarity`: pooler -> similarity_dense, reference modules/modeling.py:371-373 with module_cross.py:281-287).
    Token 0 of the layer output depends on the other tokens only through their keys and values, and the dense / FFN /
    LayerNorm stages are row-wise, so the query side (Q projection, softmax row, output projection, both LayerNorms, the
    FFN) runs on the n_seq first-token rows instead of all n_seq*S rows; K/V projections stay dense.  Same numbers for
    the rows that are used, same gradients (the unused rows receive exactly zero gradient in the dense form too).
    args as EncoderLayerFn; returns [n_seq, H]."""

    @staticmethod
    def forward(ctx, x, n_seq, S, mask, p_hidden, p_attn, training, *params):
        wa = dict(zip(ATT_KEYS, params[:10]))
        wf = dict(zip(FFN_KEYS, params[10:16]))
        drop = _Drop(p_hidden, p_attn, training)
        H = x.shape[1]
        xq = x.view(n_seq, S, H)[:, 0].contiguous()
        y1, sva = attn_block_fwd(xq, x, n_seq, 1, S, mask, wa, drop)
        y2, svf = ffn_block_fwd(y1, wf, drop)
        ctx.sva, ctx.svf = sva, svf
        ctx.shape = (n_seq, S, H)
        return y2

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        n_seq, S, H = ctx.shape
        g2, dy1, gf = ffn_block_bwd(dy, ctx.svf)
        dxq, dxkv, ga = attn_block_bwd(dy1, g2, ctx.sva)
        dxkv.view(n_seq, S, H)[:, 0].add_(dxq)  # the first-token rows are both a query source and a key/value source
        ctx.sva = ctx.svf = None
        return (dxkv, None, None, None, None, None, None) + tuple(ga[k] for k in ATT_KEYS) + \
            tuple(gf[k] for k in FFN_KEYS)


class DecoderLayerFn(torch.autograd.Function):
    """One DecoderLayer (reference modules/module_decoder.py:279-292): causal self-attention block, encoder-attention
    block, FFN block.  args: x[Td,H], enc[Te,H], then 10 + 10 + 6 params."""

    @staticmethod
    def forward(ctx, x, enc, n_seq, L, Se, slf_mask, enc_mask, p_hidden, p_attn, training, *params):
        ws = dict(zip(ATT_KEYS, params[:10]))
        we = dict(zip(ATT_KEYS, params[10:20]))
        wf = dict(zip(FFN_KEYS, params[20:26]))
        drop = _Drop(p_hidden, p_attn, training)
        s, svs = attn_block_fwd(x, x, n_seq, L, L, slf_mask, ws, drop, need_bwd=any(ctx.needs_input_grad))
        d, sve = attn_block_fwd(s, enc, n_seq, L, Se, enc_mask, we, drop)
        y, svf = ffn_block_fwd(d, wf, drop)
        ctx.svs, ctx.sve, ctx.svf = svs, sve, svf
        ctx.need_enc = enc.requires_grad
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        g3, dd, gf = ffn_block_bwd(dy, ctx.svf)
        ds, denc, ge = attn_block_bwd(dd, g3, ctx.sve, need_dxkv=ctx.need_enc)
        dx, _, gs = attn_block_bwd(ds, None, ctx.svs)
        ctx.svs = ctx.sve = ctx.svf = None
        return (dx, denc) + (None,) * 8 + tuple(gs[k] for k in ATT_KEYS) + tuple(ge[k] for k in ATT_KEYS) + \
            tuple(gf[k] for k in FFN_KEYS)


# ---------------------------------------------------------------------------------------------------------
# front-ends
# ---------------------------------------------------------------------------------------------------------
class VideoNormFn(torch.autograd.Function):
    """NormalizeVideo (reference modules/modeling.py:88-92): fp32 [N,F,1024] -> bf16 LayerNorm(1024)."""

    @staticmethod
    def forward(ctx, video, gamma, beta):
        x = video.reshape(-1, video.shape[-1])
        rows, cols = x.shape
        y = _empty((rows, cols), BF16, x)
        mean = _empty((rows,), F32, x)
        rstd = _empty((rows,), F32, x)
        call("univl_layernorm_f32_fwd", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
             mean.data_ptr(), rstd.data_ptr(), rows, cols, LN_EPS)
        ctx.save_for_backward(x, gamma, beta, mean, rstd)
        ctx.sink = GradSink()
        return y.view(video.shape)

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, mean, rstd = ctx.saved_tensors
        dy = dy.contiguous().view(x.shape)
        dgamma, r_g = ctx.sink.one(gamma)
        dbeta, r_b = ctx.sink.one(beta)
        call("univl_layernorm_f32_bwd", dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(),
             rstd.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), x.shape[0], x.shape[1])
        return None, r_g, r_b


class EmbedTextFn(torch.autograd.Function):
    """word + position (+ type) -> LayerNorm -> dropout (reference modules/module_bert.py:132-146)."""

    @staticmethod
    def forward(ctx, ids, type_ids, word, pos, type_w, gamma, beta, p, training):
        n_seq, S = ids.shape
        H = word.shape[1]
        arena = rt.current()
        p = float(p) if training else 0.0
        stream = arena.next_stream()
        ids = ids.contiguous()
        type_ids = type_ids.contiguous() if type_ids is not None else None
        y = _empty((n_seq * S, H), BF16, word)
        mean = _empty((n_seq * S,), F32, word)
        rstd = _empty((n_seq * S,), F32, word)
        call("univl_embed_text_fwd", ids.data_ptr(), ptr(type_ids), word.data_ptr(), pos.data_ptr(), ptr(type_w),
             gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), n_seq, S, H,
             word.shape[0], LN_EPS, p, arena.seed, stream)
        ctx.save_for_backward(ids, type_ids, word, pos, type_w, gamma, beta, mean, rstd)
        ctx.cfg = (n_seq, S, H, p, arena.seed, stream)
        ctx.sink = GradSink()
        return y

    @staticmethod
    def backward(ctx, dy):
        ids, type_ids, word, pos, type_w, gamma, beta, mean, rstd = ctx.saved_tensors
        n_seq, S, H, p, seed, stream = ctx.cfg
        dy = dy.contiguous()
        dword, r_word = ctx.sink.one(word)
        dpos, r_pos = ctx.sink.one(pos)
        dtype, r_type = ctx.sink.one(type_w)
        dgamma, r_g = ctx.sink.one(gamma)
        dbeta, r_b = ctx.sink.one(beta)
        call("univl_embed_text_bwd", dy.data_ptr(), ids.data_ptr(), ptr(type_ids), word.data_ptr(), pos.data_ptr(),
             ptr(type_w), gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(), dword.data_ptr(), dpos.data_ptr(),
             ptr(dtype), dgamma.data_ptr(), dbeta.data_ptr(), n_seq, S, H, word.shape[0], p, seed, stream)
        return None, None, r_word, r_pos, r_type, r_g, r_b, None, None


class EmbedSrcFn(torch.autograd.Function):
    """activation rows + position (+ type) -> LayerNorm -> dropout; visual (module_visual.py:118-131) and cross
    (module_cross.py:123-138) embeddings.  a: [Na*Wa, H] bf16, b: [Nb*Fb, H] bf16 or None.  all_pairs: pairing groups
    as in MaskSpec (Na * Nb / G sequences for G >= 1)."""

    @staticmethod
    def forward(ctx, a, b, Na, Wa, Nb, Fb, all_pairs, pos, type_w, gamma, beta, p, training):
        arena = rt.current()
        H = a.shape[1]
        p = float(p) if training else 0.0
        stream = arena.next_stream()
        all_pairs = int(all_pairs)
        n_seq = Na * Nb // all_pairs if (all_pairs and Fb > 0) else Na
        rows = n_seq * (Wa + Fb)
        y = _empty((rows, H), BF16, a)
        mean = _empty((rows,), F32, a)
        rstd = _empty((rows,), F32, a)
        call("univl_embed_src_fwd", a.data_ptr(), ptr(b), pos.data_ptr(), ptr(type_w), gamma.data_ptr(),
             beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), Na, Wa, Nb, Fb, all_pairs, H,
             LN_EPS, p, arena.seed, stream)
        ctx.save_for_backward(a, b, pos, type_w, gamma, beta, mean, rstd)
        ctx.cfg = (Na, Wa, Nb, Fb, all_pairs, H, p, arena.seed, stream)
        ctx.sink = GradSink()
        return y

    @staticmethod
    def backward(ctx, dy):
        a, b, pos, type_w, gamma, beta, mean, rstd = ctx.saved_tensors
        Na, Wa, Nb, Fb, all_pairs, H, p, seed, stream = ctx.cfg
        dy = dy.contiguous()
        da = _empty(a.shape, BF16, a)
        db = _empty(b.shape, BF16, a) if b is not None else None
        dpos, r_pos = ctx.sink.one(pos)
        dtype, r_type = ctx.sink.one(type_w)
        dgamma, r_g = ctx.sink.one(gamma)
        dbeta, r_b = ctx.sink.one(beta)
        call("univl_embed_src_bwd", dy.data_ptr(), a.data_ptr(), ptr(b), pos.data_ptr(), ptr(type_w),
             gamma.data_ptr(), mean.data_ptr(), rstd.data_ptr(), da.data_ptr(), ptr(db), dpos.data_ptr(),
             ptr(dtype), dgamma.data_ptr(), dbeta.data_ptr(), Na, Wa, Nb, Fb, all_pairs, H, p, seed, stream)
        return da, db, None, None, None, None, None, r_pos, r_type, r_g, r_b, None, None


class LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM (bf16 in/out, fp32 accumulate); optional fused erf-GELU.
    x may be a strided row view (e.g. the [CLS] rows h[:, 0]).  needs_dx=False skips the input gradient."""

    @staticmethod
    def forward(ctx, x, weight, bias, gelu, needs_dx):
        arena = rt.current()
        w16 = arena.bf16(weight)
        T = x.shape[0]
        pre = None
        if gelu:
            pre = _empty((T, w16.shape[0]), BF16, x)
            y = linear_fwd(x, w16, bias, epi=EPI_GELU, aux_out=pre)
        else:
            y = linear_fwd(x, w16, bias)
        ctx.save_for_backward(x, w16, pre, weight, bias)
        ctx.needs_dx = needs_dx
        ctx.sink = GradSink()
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w16, pre, weight, bias = ctx.saved_tensors
        dy = dy.contiguous()
        if pre is not None:
            dy = gelu_bwd(dy, pre)
        db, r_b = ctx.sink.one(bias)
        if db is not None:
            colsum(dy, db)
        dw, r_w = ctx.sink.one(weight)
        linear_wgrad(dy, x, dw)
        dx = linear_dgrad(dy, w16) if ctx.needs_dx else None
        return dx, r_w, r_b, None, None


class LinearTFn(torch.autograd.Function):
    """y = x W + b with W stored [K, N] (the MFM head multiplies by the UN-transposed tied visual input projection,
    reference modules/module_visual.py:308-311): W is an MN-major B operand, no transpose copy."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        w16 = rt.current().bf16(weight)
        T, K = x.shape
        N = w16.shape[1]
        y = _empty((T, N), BF16, x)
        gemm(x, w16, T, N, K, y, bias=bias, b_mn=True)
        ctx.save_for_backward(x, w16, weight, bias)
        ctx.sink = GradSink()
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w16, weight, bias = ctx.saved_tensors
        dy = dy.contiguous()
        T, K = x.shape
        N = w16.shape[1]
        dx = _empty((T, K), BF16, x)
        gemm(dy, w16, T, K, N, dx)                                       # dx = dy W^T : W[K,N] is K-major over N
        dw, r_w = ctx.sink.one(weight)
        gemm(x, dy, K, N, T, dw, epi=EPI_ATOMIC, a_mn=True, b_mn=True)   # dW = x^T dy
        db, r_b = ctx.sink.one(bias)
        colsum(dy, db)
        return dx, r_w, r_b


def gelu_bwd(dy, pre):
    """dpre = dy * gelu_erf'(pre) (prediction-head transforms, reference modules/module_bert.py:308-312)"""
    out = _empty(dy.shape, BF16, dy)
    call("univl_gelu_bwd_bf16", dy.data_ptr(), pre.data_ptr(), out.data_ptr(), dy.numel())
    return out


class TanhFn(torch.autograd.Function):
    """pooler activation (reference modules/module_bert.py:295)"""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        y = _empty(x.shape, BF16, x)
        call("univl_tanh_fwd_bf16", x.data_ptr(), y.data_ptr(), x.numel())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        out = _empty(y.shape, BF16, y)
        dy = dy.contiguous()
        call("univl_tanh_bwd_bf16", dy.data_ptr(), y.data_ptr(), out.data_ptr(), y.numel())
        return out


class LayerNormFn(torch.autograd.Function):
    """plain LayerNorm over bf16 rows (prediction-head transform LN, reference modules/module_bert.py:311)."""

    @staticmethod
    def forward(ctx, x, gamma, beta):
        y, mean, rstd = layernorm_fwd(x, None, gamma, beta)
        ctx.save_for_backward(x, gamma, beta, mean, rstd)
        ctx.sink = GradSink()
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, mean, rstd = ctx.saved_tensors
        dgamma, r_g = ctx.sink.one(gamma)
        dbeta, r_b = ctx.sink.one(beta)
        dx, _, _, _, _ = layernorm_bwd(dy.contiguous(), None, x, None, gamma, mean, rstd, want_dbias=False,
                                       dgamma=dgamma, dbeta=dbeta)
        return dx, r_g, r_b


# ---------------------------------------------------------------------------------------------------------
# heads and losses
# ---------------------------------------------------------------------------------------------------------
def _ld_pad(n):
    return (n + LD_VOCAB_ALIGN - 1) // LD_VOCAB_ALIGN * LD_VOCAB_ALIGN


VOCAB_LOSS_MODES = ("logits", "fused")


def vocab_loss_mode():
    """UNIVL_VOCAB_LOSS, read on every ProjXentFn call: "logits" (default) writes the fp32 logits and keeps them for
    backward; "fused" computes the vocabulary cross-entropy (target_mode 0, no pair mask, no logits returned) with
    univl_vocab_xent_fwd / _bwd, which never write logits, so nothing of size T x V lives from forward to backward.
    An environment variable, so that training drivers pick it up unchanged."""
    value = os.environ.get("UNIVL_VOCAB_LOSS", "logits")
    if value not in VOCAB_LOSS_MODES:
        raise ValueError("UNIVL_VOCAB_LOSS must be one of %s, got %r" % ("/".join(VOCAB_LOSS_MODES), value))
    return value


def vocab_xent_fwd(x, w16, bias, labels, groups):
    """-> (loss, lse [T], sum_count [2 G]) of CrossEntropy(x w16^T + bias, labels, ignore_index=-1), mean over `groups`
    consecutive row groups, without writing the logits"""
    _check2d(x, "vocab_xent x"); _check2d(w16, "vocab_xent W")
    T, K = x.shape
    V = w16.shape[0]
    nbytes = lib.load().univl_vocab_xent_workspace(T, V)
    if nbytes < 0:
        raise RuntimeError("univl_vocab_xent_workspace failed: %s" % lib.load().univl_last_error_string().decode())
    ws = _empty((nbytes,), torch.uint8, x)
    lse = _empty((T,), F32, x)
    sc = _empty((2 * groups,), F32, x)
    loss = _empty((), F32, x)
    call("univl_vocab_xent_fwd", x.data_ptr(), x.stride(0), w16.data_ptr(), w16.stride(0), ptr(bias),
         labels.data_ptr(), lse.data_ptr(), sc.data_ptr(), loss.data_ptr(), ws.data_ptr(), ws.numel(), T, V, K, groups)
    return loss, lse, sc


def vocab_xent_bwd(x, w16, bias, labels, lse, sc, g, groups):
    """-> dl bf16 [T, _ld_pad(V)]: the logits gradient univl_softmax_xent_bwd gives, from recomputed logits"""
    T, K = x.shape
    V = w16.shape[0]
    ld = _ld_pad(V)
    dl = _empty((T, ld), BF16, x)
    call("univl_vocab_xent_bwd", x.data_ptr(), x.stride(0), w16.data_ptr(), w16.stride(0), ptr(bias),
         labels.data_ptr(), lse.data_ptr(), sc.data_ptr(), ptr(g), dl.data_ptr(), ld, T, V, K, groups)
    return dl


BEAM_MAX = 8  # largest n_beam univl_vocab_beam_topk takes


def vocab_beam_topk_workspace(n_inst, n_beam, V, like):
    """uint8 workspace for vocab_beam_topk on like's device"""
    nbytes = lib.load().univl_vocab_beam_topk_workspace(int(n_inst), int(n_beam), int(V))
    if nbytes < 0:
        raise RuntimeError("univl_vocab_beam_topk_workspace failed: %s" % lib.load().univl_last_error_string().decode())
    return _empty((nbytes,), torch.uint8, like)


def vocab_beam_topk(x, w16, bias, score, n_live, n_beam, workspace=None, out=None):
    """One beam step's top n_beam per instance over the vocabulary, without logits (csrc/gemm_wgmma.cu): x bf16
    [n_inst * n_beam, K] (the head transform), w16 [V, K], bias fp32 [V], score fp32 [n_inst * n_beam], n_live int32
    [n_inst].  -> (lse fp32 [R], key fp32 [n_inst, n_beam], index int32 [n_inst, n_beam]); index = k * V + c for row k
    of the instance and word c, ordered by key descending then index ascending.  `out` = (lse, key, index) to write."""
    _check2d(x, "vocab_beam_topk x"); _check2d(w16, "vocab_beam_topk W")
    R, K = x.shape
    V = w16.shape[0]
    if not 1 <= n_beam <= BEAM_MAX or R % n_beam:
        raise ValueError("vocab_beam_topk: n_beam=%d must be in [1, %d] and divide the %d rows" % (n_beam, BEAM_MAX, R))
    n_inst = R // n_beam
    if workspace is None:
        workspace = vocab_beam_topk_workspace(n_inst, n_beam, V, x)
    if out is None:
        out = (_empty((R,), F32, x), _empty((n_inst, n_beam), F32, x), _empty((n_inst, n_beam), I32, x))
    lse, key, index = out
    call("univl_vocab_beam_topk", x.data_ptr(), x.stride(0), w16.data_ptr(), w16.stride(0), ptr(bias),
         score.data_ptr(), n_live.data_ptr(), n_inst, n_beam, V, K, lse.data_ptr(), key.data_ptr(), index.data_ptr(),
         workspace.data_ptr(), workspace.numel())
    return lse, key, index


def beam_advance(key, index, V, t, eos, score, done, prev_k, word, tokens, anc_in, anc_out):
    """The bookkeeping of beam step t (csrc/gemm_wgmma.cu, univl_beam_advance): in place on score fp32 [R], done int32
    [n_inst], the step tables prev_k / word int32 [max_words, n_inst, n_beam], tokens int64 [R] and anc_out int32
    [R, max_words] (row r's self-attention key slots for step t + 1, from anc_in)"""
    n_inst, n_beam = key.shape
    call("univl_beam_advance", key.data_ptr(), index.data_ptr(), n_inst, n_beam, int(V), int(t), prev_k.shape[0],
         int(eos), score.data_ptr(), done.data_ptr(), prev_k.data_ptr(), word.data_ptr(), tokens.data_ptr(),
         anc_in.data_ptr(), anc_out.data_ptr())


class ProjXentFn(torch.autograd.Function):
    """loss = CrossEntropy(x W^T + bias, labels) without ever exposing logits to autograd: tied vocab projection
    (reference modules/module_bert.py:327-330) + CrossEntropyLoss(ignore_index=-1) (modeling.py:253, :275), or the MFM
    NCE (modeling.py:278-297) when `pair_mask` is given (W = all frames of the rank, diagonal targets).
    w_is_param: W is an fp32 parameter [V, K] (bf16 copy from the arena); else W is a bf16 activation [V, K].
    groups: the T rows are `groups` consecutive micro-batches; the loss is the mean over groups of each group's mean.
    Grouped NCE (target_mode 1) scores each group's rows against that group's own T / groups frames only: one
    [T/G x T/G x K] logit GEMM per group, never the T x T matrix.
    UNIVL_VOCAB_LOSS=fused (vocab_loss_mode) computes the vocabulary cross-entropy (target_mode 0 without pair_mask or
    return_logits) without logits: forward saves x, W, labels, lse and sum_count only, and backward recomputes the
    logits tile by tile to form their gradient."""

    @staticmethod
    def forward(ctx, x, W, bias, labels, pair_mask, target_mode, w_is_param, return_logits, groups):
        arena = rt.current()
        w16 = arena.bf16(W) if w_is_param else W
        T, K = x.shape
        fused = vocab_loss_mode() == "fused" and target_mode == 0 and pair_mask is None and not return_logits
        if fused:
            labels = labels.contiguous()
            loss, lse, sc = vocab_xent_fwd(x, w16, bias, labels, groups)
            ctx.save_for_backward(x, w16, None, labels, None, lse, sc, W if w_is_param else None, bias)
            ctx.cfg = (target_mode, w_is_param, bias is not None, groups, False)
            ctx.sink = GradSink()
            return loss
        windowed = target_mode == 1 and groups > 1
        if windowed and (w_is_param or w16.shape[0] != T or T % groups):
            raise ValueError("grouped NCE needs one frame row per scored row and T divisible by the %d groups" % groups)
        V = T // groups if windowed else w16.shape[0]
        ld = _ld_pad(V)
        logits = _empty((T, ld), F32, x)[:, :V]
        if windowed:
            for g in range(groups):
                rows = slice(g * V, (g + 1) * V)
                gemm(x[rows], w16[rows], V, V, K, logits[rows], epi=EPI_F32, bias=bias)
        else:
            gemm(x, w16, T, V, K, logits, epi=EPI_F32, bias=bias)
        labels = labels.contiguous()
        lse = _empty((T,), F32, x)
        sc = _empty((2 * groups,), F32, x)
        loss = _empty((), F32, x)
        call("univl_softmax_xent_fwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), ptr(pair_mask),
             lse.data_ptr(), sc.data_ptr(), loss.data_ptr(), T, V, target_mode, -1, groups)
        ctx.save_for_backward(x, w16, logits, labels, pair_mask, lse, sc, W if w_is_param else None, bias)
        ctx.cfg = (target_mode, w_is_param, bias is not None, groups, windowed)
        ctx.sink = GradSink()
        if return_logits:
            return loss, logits
        return loss

    @staticmethod
    def backward(ctx, g, *unused):
        x, w16, logits, labels, pair_mask, lse, sc, W, bias = ctx.saved_tensors
        target_mode, w_is_param, has_bias, groups, windowed = ctx.cfg
        T, K = x.shape
        g = g.contiguous().to(F32)
        if logits is None:  # UNIVL_VOCAB_LOSS=fused
            V = w16.shape[0]
            dl = vocab_xent_bwd(x, w16, bias, labels, lse, sc, g, groups)
        else:
            V = logits.shape[1]
            ld = _ld_pad(V)
            dl = _empty((T, ld), BF16, x)
            call("univl_softmax_xent_bwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), ptr(pair_mask),
                 lse.data_ptr(), sc.data_ptr(), g.data_ptr(), dl.data_ptr(), ld, T, V, target_mode, -1, groups)
        dlv = dl[:, :V]
        dx = _empty((T, K), BF16, x)
        if windowed:
            dW = _empty((T, K), BF16, x)
            tmp = _zeros((T, K), F32, x)
            for gi in range(groups):
                rows = slice(gi * V, (gi + 1) * V)
                gemm(dlv[rows], w16[rows], V, K, V, dx[rows], b_mn=True)
                gemm(dl[rows], x[rows], V, K, V, tmp[rows], epi=EPI_ATOMIC, a_mn=True, b_mn=True)
            call("univl_cast_f32_to_bf16", tmp.data_ptr(), dW.data_ptr(), tmp.numel())
            db = None
            if has_bias:
                dbbuf, db = ctx.sink.one(bias)
                colsum(dlv, dbbuf)
            return dx, dW, db, None, None, None, None, None, None
        gemm(dlv, w16, T, K, V, dx, b_mn=True)
        if w_is_param:
            dWbuf, dW = ctx.sink.one(W)
            gemm(dl, x, V, K, T, dWbuf, epi=EPI_ATOMIC, a_mn=True, b_mn=True)
        else:
            dW = _empty((V, K), BF16, x)
            tmp = _zeros((V, K), F32, x)
            gemm(dl, x, V, K, T, tmp, epi=EPI_ATOMIC, a_mn=True, b_mn=True)
            call("univl_cast_f32_to_bf16", tmp.data_ptr(), dW.data_ptr(), tmp.numel())
        db = None
        if has_bias:
            dbbuf, db = ctx.sink.one(bias)
            colsum(dlv, dbbuf)
        return dx, dW, db, None, None, None, None, None, None


class MeanPoolFn(torch.autograd.Function):
    """masked mean over tokens (+ optional L2 normalise) (reference modules/modeling.py:327-339, :386-388)."""

    @staticmethod
    def forward(ctx, x, mask, N, S, skip_first, guard_zero, l2norm):
        H = x.shape[1]
        mask = mask.contiguous()
        out = _empty((N, H), F32, x)
        norm = _empty((N,), F32, x)
        call("univl_meanpool_fwd", x.data_ptr(), mask.data_ptr(), out.data_ptr(), norm.data_ptr(), N, S, H,
             int(skip_first), int(guard_zero), int(l2norm))
        ctx.save_for_backward(out, norm, mask)
        ctx.cfg = (N, S, H, int(skip_first), int(guard_zero), int(l2norm))
        return out

    @staticmethod
    def backward(ctx, dy):
        out, norm, mask = ctx.saved_tensors
        N, S, H, sf, gz, l2 = ctx.cfg
        dx = _empty((N * S, H), BF16, out)
        dy = dy.contiguous()
        call("univl_meanpool_bwd", dy.data_ptr(), out.data_ptr(), norm.data_ptr(), mask.data_ptr(), dx.data_ptr(), N,
             S, H, sf, gz, l2)
        return dx, None, None, None, None, None, None


class SimMatmulFn(torch.autograd.Function):
    """sim = T V^T (reference modules/modeling.py:389); groups > 1: the block diagonal [G, Bt/G, Bv/G], one similarity
    matrix per micro-batch."""

    @staticmethod
    def forward(ctx, t, v, groups):
        bt, bv = t.shape[0] // groups, v.shape[0] // groups
        sim = _empty((t.shape[0], v.shape[0]) if groups == 1 else (groups, bt, bv), F32, t)
        call("univl_sim_matmul_fwd", t.data_ptr(), v.data_ptr(), sim.data_ptr(), bt, bv, t.shape[1], groups)
        ctx.save_for_backward(t, v)
        ctx.groups = groups
        return sim

    @staticmethod
    def backward(ctx, ds):
        t, v = ctx.saved_tensors
        G = ctx.groups
        dt = _empty(t.shape, F32, t)
        dv = _empty(v.shape, F32, t)
        ds = ds.contiguous()
        call("univl_sim_matmul_bwd", ds.data_ptr(), t.data_ptr(), v.data_ptr(), dt.data_ptr(), dv.data_ptr(),
             t.shape[0] // G, v.shape[0] // G, t.shape[1], G)
        return dt, dv, None


def sim_topk(t, v, k):
    """Exact top-k of t v^T per row (csrc/retrieval.cu): t [Nt, H], v [Nv, H] fp32 -> (scores fp32 [Nt, k], index int32
    [Nt, k]), score descending then index ascending; each score has SimMatmulFn's bits.  1 <= k <= min(256, Nv)."""
    t, v = t.contiguous(), v.contiguous()
    _check2d(t, "sim_topk t"); _check2d(v, "sim_topk v")
    Nt, H = t.shape
    scores = _empty((Nt, max(int(k), 0)), F32, t)
    index = _empty((Nt, max(int(k), 0)), I32, t)
    call("univl_sim_topk", t.data_ptr(), v.data_ptr(), scores.data_ptr(), index.data_ptr(), Nt, v.shape[0], H, int(k))
    return scores, index


def sim_best_positive(t, v, perm, lo, hi):
    """For each row i of t [Nt, H], the best of the rows perm[lo[i]:hi[i]] of v [Nv, H] (int32 index tensors on the
    device) by score descending, then index ascending (csrc/retrieval.cu) -> (best_s fp32 [Nt], best_i int32 [Nt]);
    each score has SimMatmulFn's bits; (-inf, INT_MAX) for an empty range."""
    t, v = t.contiguous(), v.contiguous()
    _check2d(t, "sim_best_positive t"); _check2d(v, "sim_best_positive v")
    Nt, H = t.shape
    best_s, best_i = _empty((Nt,), F32, t), _empty((Nt,), I32, t)
    perm, lo, hi = perm.contiguous(), lo.contiguous(), hi.contiguous()
    call("univl_sim_best_positive", t.data_ptr(), v.data_ptr(), perm.data_ptr(), lo.data_ptr(), hi.data_ptr(),
         best_s.data_ptr(), best_i.data_ptr(), Nt, v.shape[0], H)
    return best_s, best_i


def sim_rank(t, v, best_s, best_i):
    """-> int64 [Nt]: for each row i of t, the number of rows of v that rank above (best_s[i], best_i[i]) in
    sim_topk's order, scored as sim_topk scores them (csrc/retrieval.cu).  No host synchronisation."""
    t, v = t.contiguous(), v.contiguous()
    _check2d(t, "sim_rank t"); _check2d(v, "sim_rank v")
    Nt, H = t.shape
    rank = _empty((Nt,), torch.int64, t)
    call("univl_sim_rank", t.data_ptr(), v.data_ptr(), best_s.contiguous().data_ptr(), best_i.contiguous().data_ptr(),
         rank.data_ptr(), Nt, v.shape[0], H)
    return rank


class SimLossFn(torch.autograd.Function):
    """scalar loss on a square similarity matrix [B, B], or the mean over groups of the loss of each matrix of a
    [G, B, B] stack; kind: 'maxmargin' | 'crossen' | 'milnce' (reference modules/until_module.py:182-251)."""

    @staticmethod
    def forward(ctx, sim, kind, args):
        sim = sim.contiguous()
        B = sim.shape[-1]
        G = sim.shape[0] if sim.dim() == 3 else 1
        loss = _empty((), F32, sim)
        dsim = _empty(sim.shape, F32, sim)
        if kind == "maxmargin":
            margin, n_pair, w_same, w_diff = args
            call("univl_maxmargin_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), B, float(margin), n_pair,
                 float(w_same), float(w_diff), G)
        elif kind == "crossen":
            call("univl_crossen_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), B, G)
        elif kind == "milnce":
            bs, n_pair = args
            if bs * n_pair != B:
                raise RuntimeError("MILNCELoss: sim matrix is %dx%d but batch_size*n_pair = %d" % (B, B, bs * n_pair))
            call("univl_milnce_loss", sim.data_ptr(), loss.data_ptr(), dsim.data_ptr(), bs, n_pair, G)
        else:
            raise ValueError(kind)
        ctx.save_for_backward(dsim)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dsim,) = ctx.saved_tensors
        out = _empty(dsim.shape, F32, dsim)
        g = g.contiguous().to(F32)
        call("univl_scale_f32", out.data_ptr(), dsim.data_ptr(), dsim.numel(), g.data_ptr())
        return out, None, None


class PoolerSimFn(torch.autograd.Function):
    """logit = similarity_dense(tanh(u)) for pooled cross outputs (reference modules/module_cross.py:286-287,
    modeling.py:371).  u: bf16 [N, H] (pooler dense output incl. bias)."""

    @staticmethod
    def forward(ctx, u, w, b):
        N, H = u.shape
        out = _empty((N,), F32, u)
        call("univl_pooler_sim_fwd", u.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), N, H)
        ctx.save_for_backward(u, w, b)
        ctx.sink = GradSink()
        return out

    @staticmethod
    def backward(ctx, dout):
        u, w, b = ctx.saved_tensors
        N, H = u.shape
        du = _empty((N, H), BF16, u)
        dw, r_w = ctx.sink.one(w)
        db, r_b = ctx.sink.one(b)
        dout = dout.contiguous()
        call("univl_pooler_sim_bwd", u.data_ptr(), w.data_ptr(), dout.data_ptr(), du.data_ptr(), dw.data_ptr(),
             db.data_ptr(), N, H)
        return du, r_w, r_b
