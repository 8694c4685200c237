"""fp64 stage-by-stage references of a whole transformer layer as univl_b200/ops.py composes it (attn_block_fwd /
attn_block_bwd, ffn_block_fwd / ffn_block_bwd, EncoderLayerFn, EncoderLayerClsFn, DecoderLayerFn), shared by
tests/test_gpu_layer_fp64.py and validated on CPU by tests/test_cpu_layer_check.py.

`Recorder` spies on the ops-level primitives the blocks call by module-global name and records every call: its
arguments, its outputs and the arena's dropout RNG state {seed, epoch}.  `check_layer` then walks the layer as the
reference states it (modules/module_bert.py:171-264, module_decoder.py:279-292, restated by oracle/univl_oracle.py) and
checks every stage's outputs per element, teacher-forced: each stage's fp64 reference is evaluated on the bf16 / fp32
tensors the kernels produced for the stages before it, so rounding does not pile up.  Which tensors, dropout masks and
residual gradients feed each stage is the reference formula's choice, never the code's: a stage fed the wrong tensor,
Philox stream or residual fails its bound.

The references and bounds are the kernels' own (tests/gemm_check.py, attn_check.py, row_check.py); the only new
compositions are the mode-1 LayerNorm backward's dense output dz keep / (1 - p), the bf16 add of the first-token
layer's query-row gradient into row 0 of its key/value gradient, and a parameter gradient summed over two backward
calls (`sum_refs`)."""
import inspect

import numpy as np
import torch

from tests import attn_check as ac
from tests import gemm_check as gc
from tests import row_check as rc
from tests.gemm_check import BF16_ROUND, U
from univl_b200 import ops
from univl_b200 import runtime as rt

H = 768
HEADS = 12
ROW_CHUNK = 8192           # rows per fp64 chunk of the row-wise stages
SCORE_CHUNK = 2 ** 24      # attention scores per fp64 chunk

PRIMITIVES = ("linear_fwd", "linear_dgrad", "linear_wgrad", "colsum", "layernorm_fwd", "layernorm_bwd",
              "attention_fwd", "attention_bwd", "fused_qkv_attention_fwd", "fused_attention_bwd")
# arguments a primitive accumulates into: their values before and after the call are copied
ACCUM = {"linear_wgrad": ("dw",), "colsum": ("out",), "layernorm_bwd": ("dgamma", "dbeta", "dbias"),
         "attention_bwd": ("dbias",), "fused_attention_bwd": ("dbias",)}
# primitives whose output the caller may change in place afterwards (the first-token layer's row-0 fold)
COPY_OUT = ("linear_dgrad",)
# forward primitives that draw dropout masks
DROPOUT_FWD = ("layernorm_fwd", "attention_fwd", "fused_qkv_attention_fwd")


# ---------------------------------------------------------------------------------------------------------
# recording
# ---------------------------------------------------------------------------------------------------------
def _clone(v):
    if isinstance(v, torch.Tensor):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(t) for t in v)
    return v


class Call:
    """one primitive call: name, args (every parameter by name, defaults applied), out, rng = (seed, epoch) of the
    arena at the call, pre / post = the accumulator arguments before / after it"""

    def __init__(self, name, args, out, rng, pre, post):
        self.name, self.args, self.out, self.rng, self.pre, self.post = name, args, out, rng, pre, post


class Recorder:
    """install(monkeypatch): replace every ops primitive in `names` by a spy that calls the original and records the
    call"""

    names = PRIMITIVES

    def __init__(self):
        self.calls = []

    def install(self, monkeypatch):
        for name in self.names:
            monkeypatch.setattr(ops, name, self._spy(name, getattr(ops, name)))
        return self

    def clear(self):
        self.calls = []

    def _spy(self, name, fn):
        sig = inspect.signature(fn)

        def spy(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            a = dict(bound.arguments)
            pre = {k: _clone(a[k]) for k in ACCUM.get(name, ()) if a.get(k) is not None}
            out = fn(*args, **kwargs)
            arena = getattr(rt._tls, "arena", None)     # none in autograd's backward thread
            state = arena.rng_state if arena is not None else None
            rng = tuple(int(v) for v in state.tolist()) if state is not None else None
            rec = _clone(out) if (name in COPY_OUT or name in ACCUM) else out
            self.calls.append(Call(name, a, rec, rng, pre, {k: _clone(a[k]) for k in pre}))
            return out
        return spy


class Calls:
    """the recorded calls of one layer, consumed in order per primitive"""

    def __init__(self, calls):
        self.q = {}
        for c in calls:
            self.q.setdefault(c.name, []).append(c)

    def next(self, name, what):
        lst = self.q.get(name)
        assert lst, "%s: expected a call of ops.%s" % (what, name)
        return lst.pop(0)

    def done(self):
        left = {k: len(v) for k, v in self.q.items() if v}
        assert not left, "primitive calls the reference layer does not make: %s" % left


# ---------------------------------------------------------------------------------------------------------
# the checker's bookkeeping
# ---------------------------------------------------------------------------------------------------------
class Tally:
    """worst err / bound per stage (printed as "ratio" lines by report()); a failing element raises at once"""

    def __init__(self, label=""):
        self.label = label
        self.worst = {}

    def check(self, what, got, ref, bound):
        got, ref, bound = got.detach(), ref.detach(), bound.detach()
        err = (got.double() - ref).abs()
        ok = err <= bound
        ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
        name = "%s %s" % (self.label, what)
        self.worst[what] = max(self.worst.get(what, 0.0), ratio)
        if not bool(ok.all()):
            bad = (~ok).nonzero()
            i = tuple(int(v) for v in bad[0])
            raise AssertionError("%s: %d of %d elements outside the bound; first %s: got %r ref %r bound %r"
                                 % (name, bad.shape[0], ok.numel(), i, float(got[i]), float(ref[i]), float(bound[i])))

    def report(self):
        for what, r in self.worst.items():
            print("ratio %-70s %.3e" % ("%s %s" % (self.label, what), r))
        return dict(self.worst)


def _chunks(R, chunk=ROW_CHUNK):
    return [slice(r, min(R, r + chunk)) for r in range(0, R, chunk)]


def colsum_bound(x, acc0=None):
    """bound of univl_colsum_bf16 (fixed-order column sums of bf16 rows, added to an fp32 accumulator holding acc0)
    against the fp64 column sums: (rows + 2) U sum|x| + 2 U |acc0|"""
    rows = x.shape[0]
    mag = sum(x[sl].double().abs().sum(0) for sl in _chunks(rows))
    b = (rows + 2) * U * mag
    return b + 2 * U * acc0.double().abs() if acc0 is not None else b


def sum_refs(a, b):
    """reference and bound of a gradient accumulated over two backward calls into one fp32 buffer: the fp32 sum of two
    terms each within its own bound"""
    ref = a[0] + b[0]
    return ref, a[1] + b[1] + U * (a[0].abs() + b[0].abs())


def dense_scale(p):
    """the mode-1 LayerNorm's dropout scale as the kernel computes it: 1.0f / (1.0f - p)"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


# ---------------------------------------------------------------------------------------------------------
# stage references
# ---------------------------------------------------------------------------------------------------------
def check_linear(t, what, got, x, w, bias, want_ref=False):
    """got [T, N] = x [T, K] w [N, K]^T + bias, bf16"""
    K = x.shape[1]
    refs = []
    b64 = bias.double().to(got.device)
    for sl in _chunks(x.shape[0]):
        acc, mag = gc.mm64(x[sl], w)
        ref = acc + b64
        t.check(what, got[sl], ref, gc.elem_bound(mag, K, b64.abs(), ref))
        if want_ref:
            refs.append(ref)
    return torch.cat(refs) if want_ref else None


def check_linear_gelu(t, what, pre_got, h_got, x, w, bias):
    """pre = x w^T + bias (aux_out), h = gelu(pre), both bf16 (tests/gemm_check.py run_epi EPI_GELU)"""
    K = x.shape[1]
    b64 = bias.double().to(h_got.device)
    for sl in _chunks(x.shape[0]):
        acc, mag = gc.mm64(x[sl], w)
        pre = acc + b64
        bpre = gc.elem_bound(mag, K, b64.abs())
        t.check(what + " pre", pre_got[sl], pre, bpre + BF16_ROUND * pre.abs())
        ref = gc.gelu64(pre)
        t.check(what + " h", h_got[sl], ref, gc.GELU_LIP * bpre + gc.GELU_ABS * pre.abs() + BF16_ROUND * ref.abs())


def check_dgrad(t, what, got, dy, w, add=None, gelu_pre=None, want_ref=False):
    """got [T, K] = dy [T, N] w [N, K] (+ add: EPI_ADD) (x gelu'(gelu_pre): EPI_GELU_BWD), bf16"""
    N = dy.shape[1]
    refs = []
    for sl in _chunks(dy.shape[0]):
        acc, mag = gc.mm64(dy[sl], w.t())
        if gelu_pre is not None:
            gd = gc.gelu_grad64(gelu_pre[sl].double())
            ref = acc * gd
            bound = (gc.C_ACC * N * U + gc.EPI_ROUND) * mag * gd.abs() + gc.GELU_ABS * mag + BF16_ROUND * ref.abs()
        elif add is not None:
            a = add[sl].double()
            ref = acc + a
            bound = gc.elem_bound(mag, N, a.abs(), ref)
        else:
            ref = acc
            bound = gc.elem_bound(mag, N, None, ref)
        t.check(what, got[sl], ref, bound)
        if want_ref:
            refs.append(ref)
    return torch.cat(refs) if want_ref else None


def wgrad_ref(dy, x):
    """(dy^T x, bound) of an fp32 weight gradient dW [N, K] over T = dy.shape[0] rows, accumulated into zero"""
    T = dy.shape[0]
    ref = mag = 0
    for sl in _chunks(T):
        a, m = gc.mm64(dy[sl].t(), x[sl].t())
        ref, mag = ref + a, mag + m
    return ref, gc.elem_bound(mag, T)


def keep_elem_cached(cache, seed, stream, epoch, p, rows, cols):
    key = ("elem", stream, epoch, p, rows, cols)
    if key not in cache:
        cache[key] = ac.keep_elem(seed, ac.kernel_stream(stream, epoch), p, rows, cols)
    return cache[key]


class LNSite:
    """one mode-1 LayerNorm: y = LN(dense keep / (1 - p) + res), keep from the element layout of stream `sd`"""

    def __init__(self, dense, res, gamma, beta, p, keep):
        self.dense, self.res, self.p, self.keep = dense, res, p, keep
        self.gamma, self.beta = gamma.detach(), beta.detach()
        self.scale = dense_scale(p)

    def kd(self, sl, dev):
        if self.keep is None:
            return 1.0
        return self.keep[sl].to(dev).double() * self.scale

    def z(self, sl):
        d = self.dense[sl].double()
        return d * self.kd(sl, d.device) + self.res[sl].double()

    def check_fwd(self, t, what, y, mean, rstd, want_ref=False):
        refs = []
        for sl in _chunks(self.dense.shape[0]):
            z = self.z(sl)
            ez = U * (self.dense[sl].double().abs() * self.scale + z.abs()) * 1.01
            r = rc.ln_fwd(z, self.gamma, self.beta, ez=ez)
            t.check(what + " mean", mean[sl], r["mean"], r["b_mean"])
            t.check(what + " rstd", rstd[sl], r["rstd"], r["b_rstd"])
            t.check(what + " y", y[sl], r["y"], r["b_y"])
            if want_ref:
                refs.append(r["y"])
        return torch.cat(refs) if want_ref else None

    def check_bwd(self, t, what, d_parts, g, gd, dense_scaled=True):
        """d_parts: the upstream gradients the reference sums (dy, and dy2 when the block output also feeds a residual);
        g / gd: the kernel's residual and dense outputs.  Returns {"gamma", "beta", "bias"} -> (ref, bound) of the
        column sums."""
        rows = self.dense.shape[0]
        n = rows + 2
        acc = {k: 0 for k in ("gamma", "beta", "bias", "m_gamma", "m_beta", "m_bias", "e_gamma", "e_bias")}
        for sl in _chunks(rows):
            z = self.z(sl)
            d = sum(p[sl].double() for p in d_parts)
            xhat, dz, e_xhat, e_dz = rc.ln_bwd64(z, d, self.gamma)
            t.check(what + " g", g[sl], dz, e_dz + BF16_ROUND * dz.abs())
            kd = self.kd(sl, z.device) if dense_scaled else (self.keep[sl].to(z.device).double()
                                                               if self.keep is not None else 1.0)
            kdt = kd if isinstance(kd, torch.Tensor) else torch.full_like(dz, kd)
            dd = dz * kdt
            t.check(what + " gd", gd[sl], dd, rc.bf16_store(e_dz * kdt + U * dd.abs(), dd))
            acc["gamma"] = acc["gamma"] + (d * xhat).sum(0)
            acc["m_gamma"] = acc["m_gamma"] + (d * xhat).abs().sum(0)
            acc["e_gamma"] = acc["e_gamma"] + (d.abs() * e_xhat).sum(0)
            acc["beta"] = acc["beta"] + d.sum(0)
            acc["m_beta"] = acc["m_beta"] + d.abs().sum(0)
            acc["bias"] = acc["bias"] + dd.sum(0)
            acc["m_bias"] = acc["m_bias"] + dd.abs().sum(0)
            acc["e_bias"] = acc["e_bias"] + (e_dz * kdt).sum(0)
        return {"gamma": (acc["gamma"], n * U * acc["m_gamma"] + acc["e_gamma"]),
                "beta": (acc["beta"], n * U * acc["m_beta"] + 1e-30),
                "bias": (acc["bias"], n * U * acc["m_bias"] + acc["e_bias"] + 1e-30)}


def key_real_of(mask, n_seq):
    return ac.pair_masks(mask.a, mask.b, n_seq, mask.all_pairs)


def attention_keep(layout, seed, stream, epoch, p, n_seq, Sq, Sk, cache):
    if p <= 0:
        return None
    key = (layout, stream, epoch, p, n_seq, Sq, Sk)
    if key not in cache:
        ks = ac.kernel_stream(stream, epoch)
        cache[key] = (ac.keep_rowmajor(seed, ks, p, n_seq * HEADS, Sq) if layout == "rowmajor"
                      else ac.keep_tile(seed, ks, p, n_seq * HEADS, Sq, Sk))
    return cache[key]


def check_attention(t, what, q, k, v, ctx, lse, dctx, dq, dk, dv, n_seq, Sq, Sk, key_real, causal, keep, p, kind):
    """the attention core forward and backward against attn_check.reference, in chunks of sequences; returns the
    (ref, bound) of the three projection-bias gradients (column sums of dq / dk / dv)"""
    per = max(1, SCORE_CHUNK // (HEADS * Sq * Sk))
    bias = {n: [0, 0] for n in ("dq", "dk", "dv")}
    for s0 in range(0, n_seq, per):
        n = min(per, n_seq - s0)
        rq, rk = slice(s0 * Sq, (s0 + n) * Sq), slice(s0 * Sk, (s0 + n) * Sk)
        kp = keep[s0 * HEADS:(s0 + n) * HEADS] if keep is not None else None
        r = ac.reference(q[rq], k[rk], v[rk], n, Sq, Sk, key_real[s0:s0 + n], causal, kp, p, d_o=dctx[rq],
                         o_kernel=ctx[rq], kind=kind)
        t.check(what + " ctx", ctx[rq], r["o"], r["b_o"])
        t.check(what + " lse", lse[s0 * HEADS * Sq:(s0 + n) * HEADS * Sq], r["lse"], r["b_lse"])
        for name, got, rows in (("dq", dq, rq), ("dk", dk, rk), ("dv", dv, rk)):
            t.check(what + " " + name, got[rows], r[name], r["b_" + name])
            bias[name][0] = bias[name][0] + r[name].sum(0)
            bias[name][1] = bias[name][1] + ac.bias_bound(r[name], r["b_" + name])
    return {"b" + n[1]: tuple(v) for n, v in bias.items()}


# ---------------------------------------------------------------------------------------------------------
# the layer walk
# ---------------------------------------------------------------------------------------------------------
class Block:
    """one block of a layer as the reference states it: kind "attn" (xq, xkv, Sq, Sk, mask, causal) or "ffn" (x)"""

    def __init__(self, kind, w, **kw):
        self.kind, self.w = kind, w
        self.__dict__.update(kw)


def layer_blocks(kind, params, x, n_seq, S=None, mask=None, enc=None, L=None, Se=None, slf_mask=None,
                 enc_mask=None, fused=False):
    """the blocks of EncoderLayerFn ("enc"), EncoderLayerClsFn ("cls") or DecoderLayerFn ("dec") with their formula
    inputs; a block input that is another block's output is named by that block ("prev")"""
    att = lambda i: dict(zip(ops.ATT_KEYS, params[i:i + 10]))
    ffn = lambda i: dict(zip(ops.FFN_KEYS, params[i:i + 6]))
    if kind == "enc":
        return [Block("attn", att(0), xq=x, xkv=x, self_attn=True, fused=fused, n_seq=n_seq, Sq=S, Sk=S, mask=mask),
                Block("ffn", ffn(10))]
    if kind == "cls":
        x0 = x.view(n_seq, S, H)[:, 0]
        return [Block("attn", att(0), xq=x0, xkv=x, self_attn=False, fused=False, n_seq=n_seq, Sq=1, Sk=S, mask=mask),
                Block("ffn", ffn(10))]
    return [Block("attn", att(0), xq=x, xkv=x, self_attn=True, fused=fused, n_seq=n_seq, Sq=L, Sk=L, mask=slf_mask),
            Block("attn", att(10), xq="prev", xkv=enc, self_attn=False, fused=False, n_seq=n_seq, Sq=L, Sk=Se,
                  mask=enc_mask),
            Block("ffn", ffn(20))]


def attn_out_fwd(t, C, what, ctx, res, w, arena, p_hid=0.0, keep=None):
    """the attention block's output stages: ao = ctx Wo^T + bo, then y = LN(ao keep / (1 - p) + res) -> (s dict)"""
    ao = C.next("linear_fwd", what + " o").out
    check_linear(t, what + " ao", ao, ctx, arena.bf16(w["o"]), w["bo"].detach())
    y, mean, rstd = C.next("layernorm_fwd", what + " ln").out
    ln = LNSite(ao, res, w["gamma"], w["beta"], p_hid, keep)
    ln.check_fwd(t, what + " ln", y, mean, rstd)
    return dict(ao=ao, y=y, mean=mean, rstd=rstd, ln=ln)


def ffn_fwd(t, C, what, x, w, arena, p_hid=0.0, keep_of=None):
    """the FFN block: pre = x W1^T + b1, h = gelu(pre), fo = h W2^T + b2, y = LN(fo keep / (1 - p) + x); keep_of():
    the LayerNorm's dropout mask, drawn after the GEMMs (None: p = 0) -> (s dict)"""
    w1, w2 = arena.bf16(w["w1"]), arena.bf16(w["w2"])
    c = C.next("linear_fwd", what + " w1")
    h, pre = c.out, c.args["aux_out"]
    check_linear_gelu(t, what + " w1", pre, h, x, w1, w["b1"].detach())
    fo = C.next("linear_fwd", what + " w2").out
    check_linear(t, what + " fo", fo, h, w2, w["b2"].detach())
    y, mean, rstd = C.next("layernorm_fwd", what + " ln").out
    ln = LNSite(fo, x, w["gamma"], w["beta"], p_hid, keep_of() if keep_of is not None else None)
    ln.check_fwd(t, what + " ln", y, mean, rstd)
    return dict(mean=mean, rstd=rstd, x=x, h=h, pre=pre, fo=fo, y=y, ln=ln, w1=w1, w2=w2)


def block_key_real(b):
    """the key mask [n_seq, Sk] of an attention block: given by the walk (key_real), or the block's MaskSpec"""
    kr = getattr(b, "key_real", None)
    return kr if kr is not None else key_real_of(b.mask, b.n_seq)


def check_layer_fwd(t, C, blocks, arena, ph=0.0, pa=0.0, stream=None, rng=None, cache=None, perturb=(),
                    core=False):
    """the forward walk of one layer: every block's stages in the reference's order, teacher-forced, consuming the
    calls from C (a Calls).  stream: [the arena's stream counter before the forward] (advanced per dropout site);
    rng: (seed, epoch) of the dropout masks (None at p = 0).  core: check the attention core's context and lse here
    (a forward-only walk; check_layer checks them with the backward).  Returns the blocks' saved tensors (list of
    dicts); the layer's output is the last one's "y"."""
    cache = {} if cache is None else cache
    stream = [0] if stream is None else stream
    seed, epoch = rng if rng is not None else (0, 0)

    def next_stream():
        stream[0] += 1
        return stream[0]

    p_attn, p_hid = (ph, pa) if "swap_p" in perturb else (pa, ph)
    prev = None
    st = []
    for bi, b in enumerate(blocks):
        what = "block%d %s" % (bi, b.kind)
        s = {}
        if b.kind == "attn":
            xq = prev if isinstance(b.xq, str) else b.xq
            xkv = b.xkv
            w = b.w
            wqkv = arena.bf16_qkv(w["q"], w["k"], w["v"])
            if b.self_attn:
                bqkv = torch.cat([w["bq"], w["bk"], w["bv"]]).detach()
                if b.fused:
                    c = C.next("fused_qkv_attention_fwd", what)
                    ctx, lse, qkv = c.out
                else:
                    qkv = C.next("linear_fwd", what + " qkv").out
                check_linear(t, what + " qkv", qkv, xq, wqkv, bqkv)
                q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
                s.update(qkv=qkv)
            else:
                q = C.next("linear_fwd", what + " q").out
                check_linear(t, what + " q", q, xq, wqkv[:H], w["bq"].detach())
                kv = C.next("linear_fwd", what + " kv").out
                check_linear(t, what + " kv", kv, xkv, wqkv[H:], torch.cat([w["bk"], w["bv"]]).detach())
                k, v = kv[:, :H], kv[:, H:]
                s.update(q=q, kv=kv)
            if not b.fused:
                ctx, lse = C.next("attention_fwd", what + " core").out
            kind = "fused" if b.fused else ("long" if max(b.Sq, b.Sk) > ops.SHORT_ATTN_MAX_S else "short")
            if core:
                r = ac.reference(q, k, v, b.n_seq, b.Sq, b.Sk, block_key_real(b), b.mask.causal if b.mask else False,
                                 kind=kind)
                t.check(what + " core ctx", ctx, r["o"], r["b_o"])
                t.check(what + " core lse", lse, r["lse"], r["b_lse"])
            sa, sd = next_stream(), next_stream()
            if "stream+1" in perturb:
                sa += 1
            layout = "rowmajor" if b.fused else "tile"
            if "tile_layout" in perturb:
                layout = "tile"
            keep = attention_keep(layout, seed, sa, epoch, p_attn, b.n_seq, b.Sq, b.Sk, cache)
            R = xq.shape[0]
            s.update(attn_out_fwd(t, C, what, ctx, xq, w, arena, p_hid,
                                  keep_elem_cached(cache, seed, sd, epoch, p_hid, R, H) if p_hid > 0 else None))
            s.update(xq=xq, xkv=xkv, q=q, k=k, v=v, ctx=ctx, lse=lse, keep=keep, wqkv=wqkv, kind=kind)
        else:
            x = prev
            sd = []

            def keep_of():
                sd.append(next_stream())
                return keep_elem_cached(cache, seed, sd[0], epoch, p_hid, x.shape[0], H) if p_hid > 0 else None
            s.update(ffn_fwd(t, C, what, x, b.w, arena, p_hid, keep_of))
        st.append(s)
        prev = s["y"]
    return st


def check_layer(calls, blocks, arena, ph, pa, stream0, dy, out, dx, denc=None, fold_rows=None, perturb=(),
                label="", fused_bwd=True, want=()):
    """Check one recorded layer call (forward and backward) stage by stage.
    calls: the Recorder's calls of this layer; blocks: layer_blocks(); stream0: the arena's stream counter before the
    forward (the reference layer's dropout sites draw stream0 + 1, + 2, ... in block order: attention core, attention
    LayerNorm, FFN LayerNorm); dy: the upstream gradient; out / dx / denc: what the layer returned (denc: the decoder's
    encoder gradient, None when not asked for); fold_rows: the first-token layer's (n_seq, S).
    perturb: reference perturbations for the negative checks ("stream+1", "tile_layout", "swap_p", "no_dy2",
    "no_dense_scale", "no_fold", "kv_from_x").
    Returns (tally, param_refs {(block index, key): (ref, bound)}, refs {name: fp64 tensor} for the names in want)."""
    t = Tally(label)
    C = Calls(calls)
    cache = {}
    first = next(c for c in calls if c.name in DROPOUT_FWD)
    p_attn = ph if "swap_p" in perturb else pa
    refs = {}
    st = check_layer_fwd(t, C, blocks, arena, ph, pa, [stream0], first.rng, cache, perturb)
    # the layer's output is the last block's LayerNorm output
    y_ref = st[-1]["ln"].check_fwd(t, "out", out, st[-1]["mean"], st[-1]["rstd"], want_ref="out" in want)
    if y_ref is not None:
        refs["out"] = y_ref

    # ---- backward: blocks in reverse; each block's output gradient is the reference's sum of its consumers'
    pr = {}
    up = [dy]                  # gradient parts of the current block's output
    for bi in range(len(blocks) - 1, -1, -1):
        b, s = blocks[bi], st[bi]
        what = "block%d %s" % (bi, b.kind)
        w = b.w
        lnb = C.next("layernorm_bwd", what + " ln bwd")
        g, gd = lnb.out[0], lnb.out[1]
        parts = up[:1] if "no_dy2" in perturb and b.kind == "attn" and len(up) > 1 else up
        col = s["ln"].check_bwd(t, what + " ln bwd", parts, g, gd, dense_scaled="no_dense_scale" not in perturb)
        if b.kind == "ffn":
            pr[(bi, "gamma")], pr[(bi, "beta")], pr[(bi, "b2")] = col["gamma"], col["beta"], col["bias"]
            C.next("linear_wgrad", what + " dw2")
            pr[(bi, "w2")] = wgrad_ref(gd, s["h"])
            dpre = C.next("linear_dgrad", what + " dpre").out
            check_dgrad(t, what + " dpre", dpre, gd, s["w2"], gelu_pre=s["pre"])
            C.next("colsum", what + " db1")
            pr[(bi, "b1")] = (sum(dpre[sl].double().sum(0) for sl in _chunks(dpre.shape[0])), colsum_bound(dpre))
            C.next("linear_wgrad", what + " dw1")
            pr[(bi, "w1")] = wgrad_ref(dpre, s["x"])
            dxd = C.next("linear_dgrad", what + " dx").out
            check_dgrad(t, what + " dx", dxd, dpre, s["w1"])
            up = [dxd, g]      # the FFN input feeds the dense path and the residual
            continue
        pr[(bi, "gamma")], pr[(bi, "beta")], pr[(bi, "bo")] = col["gamma"], col["beta"], col["bias"]
        C.next("linear_wgrad", what + " dwo")
        pr[(bi, "o")] = wgrad_ref(gd, s["ctx"])
        dctx = C.next("linear_dgrad", what + " dctx").out
        check_dgrad(t, what + " dctx", dctx, gd, arena.bf16(w["o"]))
        Sq, Sk, n_seq = b.Sq, b.Sk, b.n_seq
        key_real = key_real_of(b.mask, n_seq)
        if b.self_attn:
            if b.fused and fused_bwd:
                c = C.next("fused_attention_bwd", what + " core bwd")
            else:
                c = C.next("attention_bwd", what + " core bwd")
            dqkv = c.args["dqkv"] if "dqkv" in c.args else torch.cat([c.args["dq"], c.args["dk"], c.args["dv"]], 1)
            dq, dk, dv = dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:]
        else:
            c = C.next("attention_bwd", what + " core bwd")
            dq, dk, dv = c.args["dq"], c.args["dk"], c.args["dv"]
        bias = check_attention(t, what + " core", s["q"], s["k"], s["v"], s["ctx"], s["lse"], dctx, dq, dk, dv, n_seq,
                               Sq, Sk, key_real, b.mask.causal, s["keep"], p_attn, s["kind"])
        for n in ("bq", "bk", "bv"):
            pr[(bi, n)] = bias[n]
        wqkv = s["wqkv"]
        if b.self_attn:
            C.next("linear_wgrad", what + " dwqkv")
            ref, bnd = wgrad_ref(dqkv, s["xq"])
            for j, n in enumerate(("q", "k", "v")):
                pr[(bi, n)] = (ref[j * H:(j + 1) * H], bnd[j * H:(j + 1) * H])
            dxq = C.next("linear_dgrad", what + " dx").out
            check_dgrad(t, what + " dx", dxq, dqkv, wqkv, add=g)
            s["dx_args"] = (dqkv, wqkv, g)
            up = [dxq]
        else:
            C.next("linear_wgrad", what + " dwq")
            pr[(bi, "q")] = wgrad_ref(dq, s["xq"])
            C.next("linear_wgrad", what + " dwkv")
            dkv = torch.cat([dk, dv], 1)
            kv_in = blocks[0].xq if "kv_from_x" in perturb else s["xkv"]
            ref, bnd = wgrad_ref(dkv, kv_in)
            pr[(bi, "k")], pr[(bi, "v")] = (ref[:H], bnd[:H]), (ref[H:], bnd[H:])
            dxq = C.next("linear_dgrad", what + " dxq").out
            check_dgrad(t, what + " dxq", dxq, dq, wqkv[:H], add=g)
            up = [dxq]
            if fold_rows is not None:
                dxkv = C.next("linear_dgrad", what + " dxkv").out
                check_dgrad(t, what + " dxkv", dxkv, dkv, wqkv[H:])
                n_seq_f, S = fold_rows
                ref = dxkv.double().clone()
                if "no_fold" not in perturb:
                    ref.view(n_seq_f, S, H)[:, 0] += dxq.double()
                bound = torch.zeros_like(ref)
                bound.view(n_seq_f, S, H)[:, 0] = (BF16_ROUND + U) * ref.view(n_seq_f, S, H)[:, 0].abs()
                t.check("dx (row-0 fold)", dx, ref, bound)
            elif denc is not None:
                dxkv = C.next("linear_dgrad", what + " denc").out
                r = check_dgrad(t, what + " denc", dxkv, dkv, wqkv[H:], want_ref="denc" in want)
                check_dgrad(t, "denc", denc, dkv, wqkv[H:])
                if r is not None:
                    refs["denc"] = r
    if fold_rows is None:
        dqkv, wqkv, g = st[0]["dx_args"]
        r = check_dgrad(t, "dx", dx, dqkv, wqkv, add=g, want_ref="dx" in want)
        if r is not None:
            refs["dx"] = r
    C.done()
    return t, pr, refs


def check_param_grads(t, blocks, pr, grad_of):
    """every parameter gradient of the layer (16 per encoder layer, 26 per decoder layer) against its reference;
    grad_of(param) -> the gradient the layer left for it.  Returns the number checked."""
    n = 0
    for bi, b in enumerate(blocks):
        for k in (ops.ATT_KEYS if b.kind == "attn" else ops.FFN_KEYS):
            ref, bound = pr[(bi, k)]
            t.check("grad block%d %s" % (bi, k), grad_of(b.w[k]), ref, bound)
            n += 1
    return n
