"""fp64 stage-by-stage references of the cross encoder's evaluation compositions (univl_b200/ops.py pair_layer_eval,
the *_eval_fp8 and *_eval_packed layer functions, CrossModel.first_layer_source_rows), shared by
tests/test_gpu_eval_fp64.py and validated on CPU by tests/test_cpu_eval_check.py.

`EvalRecorder` spies on the eval primitives as well as tests/layer_check.py's, and on PoolerSimFn.  `check_similarity`
then walks one recorded evaluation call (a dense get_similarity_logits, or a score_pairs list) as the reference
states it and checks every stage per element, teacher-forced: each stage's fp64 reference is evaluated on the tensors
the kernels produced for the stages before it.  What feeds a stage comes from the reference formula alone: the pair
sequence of (text i, video j) is text row i then video row j (reference modeling.py:355-370), its key set is
mask_t[i] ++ mask_v[j], its embedding rows sit at position s (text) or W + s with type 1 (video), and on the packed
layout it holds those of its tokens that are valid, in ascending position.  None of this is read from the MaskSpec,
VarlenSeqs or PairPacking the code built, and the tiles are enumerated from modeling._eval_tile /
_packed_eval_tiles / retrieval._pair_chunks.

The references and bounds are the kernels' own: tests/gemm_check.py (bf16 GEMMs), attn_check.py (attention cores),
row_check.py (LayerNorms, the pooler similarity), fp8_check.py (quantizers bit for bit, FP8 GEMMs).  The middle and
last cross layers of the padded bf16 path are EncoderLayerFn / EncoderLayerClsFn forwards and are walked by
layer_check.check_layer_fwd.

Perturbations of the reference (the negative checks) are named in PERTURB."""
import numpy as np
import torch

from tests import attn_check as ac
from tests import fp8_check as f8
from tests import layer_check as lc
from tests import row_check as rc
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200.modules import modeling
from univl_b200.modules.transformer import _layer_params

H = 768
PRIMITIVES = lc.PRIMITIVES + ("attention_pair_fwd", "attention_varlen_fwd", "gather_rows_varlen",
                              "embed_src_rows_eval", "quantize_e4m3_rows", "quantize_e4m3_blocks", "gemm_fp8")
# the reference perturbations the negative checks apply, and the stage each must fail at
PERTURB = {"video_pos": "embed video", "video_type0": "embed video", "res_next_video": "layer0 attn ln",
           "drop_last_key": "core", "quant_prev": "quantize", "kv_as_qk": "weights", "scale_x2": "fp8 gemm",
           "transpose_tiles": "logits"}


class EvalRecorder(lc.Recorder):
    """lc.Recorder over the eval primitives too, and PoolerSimFn.apply (recorded as "pooler_sim").  The fused QKV +
    attention kernel is asked to keep its Q/K/V projections (save_qkv), which the forward-only layers skip, so that
    the walk can check them; its context does not depend on that flag."""

    names = PRIMITIVES

    def install(self, monkeypatch):
        super().install(monkeypatch)
        fused = ops.fused_qkv_attention_fwd
        monkeypatch.setattr(ops, "fused_qkv_attention_fwd",
                            lambda *a, **k: fused(*a, **dict(k, save_qkv=True)))
        apply = ops.PoolerSimFn.apply

        def pooler_sim(u, w, b):
            out = apply(u, w, b)
            self.calls.append(lc.Call("pooler_sim", dict(u=u, w=w, b=b), out, None, {}, {}))
            return out
        monkeypatch.setattr(ops.PoolerSimFn, "apply", pooler_sim)
        return self


def _exact(what, got, ref):
    """bit-for-bit equality (codes as bytes)"""
    view = (lambda x: x.view(torch.uint8)) if got.dtype == f8.E4M3 else (lambda x: x)
    g, r = view(got.detach()).cpu(), view(ref.detach().to(got.device)).cpu()
    if g.shape != r.shape or not torch.equal(g, r):
        n = int((g != r).sum()) if g.shape == r.shape else -1
        raise AssertionError("%s: not bit for bit the reference (%s vs %s, %d elements differ)"
                             % (what, tuple(g.shape), tuple(r.shape), n))


def core_check(t, what, q, k, v, n, Sq, S, key_real, got, rows=None):
    """attention of n padded sequences of S keys (key_real [n, S]) against attn_check.reference; got is compared with
    the reference rows `rows` (flat indices into the [n * Sq] padded query rows), or with all of them"""
    kind = "long" if S > ops.SHORT_ATTN_MAX_S else "short"
    r = ac.reference(q, k, v, n, Sq, S, key_real, kind=kind)
    o, b = r["o"], r["b_o"]
    if rows is not None:
        o, b = o[rows.to(o.device)], b[rows.to(o.device)]
    t.check(what + " core ctx", got, o, b)


def scatter(packed, pidx, n, S):
    """packed rows -> the [n * S] padded rows (zeros at padded tokens, which are masked keys)"""
    out = torch.zeros((n * S, packed.shape[1]), dtype=packed.dtype, device=packed.device)
    out[pidx.to(packed.device)] = packed
    return out


class Walk:
    """the state of one evaluation call's walk"""

    def __init__(self, model, arena, text2d, video2d, mask_t, mask_v, fp8, perturb, label):
        self.cross = model.cross
        self.model, self.arena = model, arena
        self.text2d, self.video2d = text2d, video2d
        self.mt, self.mv = mask_t.cpu().long(), mask_v.cpu().long()
        (self.Nt, self.W), (self.Nv, self.F) = self.mt.shape, self.mv.shape
        self.S = self.W + self.F
        self.fp8, self.perturb = fp8, set(perturb)
        self.t = lc.Tally(label)
        self.layers = [_layer_params(layer) for layer in self.cross.encoder.layer]
        self.L = len(self.layers)
        self.dev = text2d.device

    def att(self, layer):
        return dict(zip(ops.ATT_KEYS, self.layers[layer][:10]))

    def ffn(self, layer):
        return dict(zip(ops.FFN_KEYS, self.layers[layer][10:16]))

    # -----------------------------------------------------------------------------------------------------
    # once per call: FP8 weights, source rows
    # -----------------------------------------------------------------------------------------------------
    def weight_stack(self, layer, name):
        """the fp32 weights of GEMM `name` of a layer, stacked in the order the reference projects them"""
        wa, wf = self.att(layer), self.ffn(layer)
        if name == "kv":
            return (wa["q"], wa["k"]) if "kv_as_qk" in self.perturb else (wa["k"], wa["v"])
        return {"qkv": (wa["q"], wa["k"], wa["v"]), "o": (wa["o"],), "w1": (wf["w1"],), "w2": (wf["w2"],)}[name]

    def check_weights(self, C):
        """every quantize_e4m3_blocks call of fp8_eval_weights: codes and scales bit for bit the rule applied to the
        reference's weights, layer by layer in the reference's GEMM order -> {(layer, name): (codes, scales)}"""
        self.qw = {}
        for layer in range(self.L):
            names = ("kv",) if layer == self.L - 1 else ("o", "w1", "w2") if layer == 0 else ("qkv", "o", "w1", "w2")
            for name in names:
                parts = []
                for w in self.weight_stack(layer, name):
                    c = C.next("quantize_e4m3_blocks", "weights %d %s" % (layer, name))
                    q, s = f8.quant_blocks(w.detach().cpu())
                    _exact("weights layer%d %s codes" % (layer, name), c.out[0], q)
                    _exact("weights layer%d %s scales" % (layer, name), c.out[1], s)
                    parts.append((q, s))
                self.qw[(layer, name)] = (torch.cat([p[0].view(torch.uint8) for p in parts]).view(f8.E4M3),
                                          torch.cat([p[1] for p in parts]))

    def check_sources(self, C):
        """the embedding LayerNorm of every text row (position s, type 0) and video row (position W + s, type 1), and
        the first layer's Q/K/V projection of those rows -> self.X [Nt*W + Nv*F, H], self.QKV [.., 3H]"""
        emb = self.cross.embeddings
        pos, typ = emb.position_embeddings.weight.detach(), emb.token_type_embeddings.weight.detach()
        gamma, beta = emb.LayerNorm.weight.detach(), emb.LayerNorm.bias.detach()
        ys = []
        for name, src, N, n in (("text", self.text2d, self.Nt, self.W), ("video", self.video2d, self.Nv, self.F)):
            c = C.next("embed_src_rows_eval", "embed " + name)
            off = self.W if name == "video" and "video_pos" not in self.perturb else 0
            ty = 1 if name == "video" and "video_type0" not in self.perturb else 0
            a = src.double().view(N, n, H)
            p = pos.double()[off:off + n].to(a.device)
            tr = typ.double()[ty].to(a.device)
            z = (a + p + tr).reshape(-1, H)
            ez = (2 * rc.U * (a.abs() + p.abs() + tr.abs())).reshape(-1, H)
            r = rc.ln_fwd(z, gamma.to(a.device), beta.to(a.device), ez=ez)
            y = c.args["out"]
            self.t.check("embed " + name, y, r["y"], r["b_y"])
            ys.append(y)
        self.X = torch.cat(ys)
        wa = self.att(0)
        c = C.next("linear_fwd", "source qkv")
        lc.check_linear(self.t, "source qkv", c.out, self.X, self.arena.bf16_qkv(wa["q"], wa["k"], wa["v"]),
                        torch.cat([wa["bq"], wa["bk"], wa["bv"]]).detach())
        self.QKV = c.out

    # -----------------------------------------------------------------------------------------------------
    # one tile of pairs
    # -----------------------------------------------------------------------------------------------------
    def pair_rows(self, pairs, j_shift=0):
        """[n, S] rows of self.X / self.QKV of the pair sequences: text i rows i*W + s, then video j rows"""
        ti = torch.tensor([p[0] for p in pairs], dtype=torch.long)
        vj = torch.tensor([(p[1] + j_shift) % self.Nv for p in pairs], dtype=torch.long)
        text = ti[:, None] * self.W + torch.arange(self.W)[None]
        video = self.Nt * self.W + vj[:, None] * self.F + torch.arange(self.F)[None]
        return torch.cat([text, video], 1)

    def key_real(self, pairs):
        ti = torch.tensor([p[0] for p in pairs], dtype=torch.long)
        vj = torch.tensor([p[1] for p in pairs], dtype=torch.long)
        return torch.cat([self.mt[ti], self.mv[vj]], 1)

    def core_ref(self, what, q, k, v, n, Sq, key_real, got, rows=None):
        core_check(self.t, what, q, k, v, n, Sq, self.S, key_real, got, rows)

    def scatter(self, packed, pidx, n):
        return scatter(packed, pidx, n, self.S)

    def quantized(self, C, what, x_ref):
        """a quantize_e4m3_rows call: its input is x_ref (the previous stage's output) bit for bit, and its codes and
        scales are the rule's"""
        c = C.next("quantize_e4m3_rows", what + " quantize")
        _exact(what + " quantize input", c.args["x"], x_ref)
        q, s = f8.quant_rows(c.args["x"].cpu())
        _exact(what + " quantize codes", c.out[0], q)
        _exact(what + " quantize scales", c.out[1], s)
        return c.out

    def gemm(self, C, what, a, layer, name, bias, gelu=False):
        """a gemm_fp8 call: its operands are the quantized activations a = (codes, scales) and the reference's weights
        of (layer, name); its output against the fp64 product of the dequantized operands"""
        c = C.next("gemm_fp8", what + " fp8 gemm")
        _exact(what + " fp8 gemm A", c.args["a"], a[0])
        _exact(what + " fp8 gemm A scales", c.args["a_scale"], a[1])
        qb, sb = self.qw[(layer, name)]
        _exact(what + " weights " + name, c.args["b"], qb)
        _exact(what + " weights " + name + " scales", c.args["b_scale"], sb)
        _exact(what + " fp8 gemm bias", c.args["bias"], bias.detach())
        A = f8.deq_rows(c.args["a"], c.args["a_scale"])
        B = f8.deq_blocks(qb, sb).to(A.device)
        if "scale_x2" in self.perturb:
            B[:128, :128] *= 2
        b64 = bias.detach().double().to(A.device)
        ref = A @ B.t() + b64
        absref = A.abs() @ B.abs().t() + b64.abs()
        if gelu:
            h, hs = c.out
            g = torch.nn.functional.gelu(ref)
            self.t.check(what + " fp8 gemm gelu", f8.deq_rows(h, hs), g, f8.gelu_e4m3_bound(g, absref, hs))
        else:
            self.t.check(what + " fp8 gemm", c.out, ref, f8.bf16_out_bound(ref, absref))
        return c.out

    def tail(self, C, what, layer, ctx, res):
        """attention output + LayerNorm(res) and the FFN of an eval layer (bf16, or the FP8 tail) -> its output"""
        if not self.fp8:
            s = lc.attn_out_fwd(self.t, C, what + " attn", ctx, res, self.att(layer), self.arena)
            return lc.ffn_fwd(self.t, C, what + " ffn", s["y"], self.ffn(layer), self.arena)["y"]
        wa, wf = self.att(layer), self.ffn(layer)
        ao = self.gemm(C, what + " o", self.quantized(C, what + " o", ctx), layer, "o", wa["bo"])
        y, mean, rstd = C.next("layernorm_fwd", what + " attn ln").out
        lc.LNSite(ao, res, wa["gamma"], wa["beta"], 0.0, None).check_fwd(self.t, what + " attn ln", y, mean, rstd)
        h = self.gemm(C, what + " w1", self.quantized(C, what + " w1", ao if "quant_prev" in self.perturb else y),
                      layer, "w1", wf["b1"], gelu=True)
        fo = self.gemm(C, what + " w2", h, layer, "w2", wf["b2"])
        out, mean, rstd = C.next("layernorm_fwd", what + " ffn ln").out
        lc.LNSite(fo, y, wf["gamma"], wf["beta"], 0.0, None).check_fwd(self.t, what + " ffn ln", out, mean, rstd)
        return out

    def tile(self, C, pairs, layout, listed):
        """walk the cross layers of one tile of pairs -> token 0 of every pair's last-layer output [n, H]"""
        n, S, L = len(pairs), self.S, self.L
        first = L == 1
        rows = self.pair_rows(pairs)
        kr = self.key_real(pairs)
        res_rows = self.pair_rows(pairs, 1) if "res_next_video" in self.perturb else rows
        X, QKV = self.X, self.QKV
        dev = X.device
        packed = layout == "packed"
        if packed:
            pflat = kr.reshape(-1).nonzero()[:, 0]                   # valid tokens p * S + s, pair then position
            counts = kr.sum(1)
            starts = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)[:-1]])
            kr_ref = kr.clone()
            if "drop_last_key" in self.perturb:
                last = S - 1 - kr.flip(1).argmax(1)
                kr_ref[torch.arange(n), last] = 0
        else:
            kr_ref = kr
        rows_d, res_d = rows.to(dev), res_rows.to(dev)
        q_all, k_all, v_all = (QKV[rows_d.reshape(-1), c * H:(c + 1) * H] for c in range(3))
        what = "layer0"
        # ---- first layer: Q/K/V from the per-source projections, residual from the per-source embedding rows
        if packed or listed:
            c = C.next("gather_rows_varlen", what + " gather")
            if packed:
                want = X[res_d[:, 0]] if first else X[res_d.reshape(-1)[pflat.to(dev)]]
            else:
                want = X[res_d.reshape(-1)]
            _exact(what + " gather", c.out, want)
        if first:
            res = X[res_d[:, 0]]
        else:
            res = X[res_d.reshape(-1)]
            if packed:
                res = res[pflat.to(dev)]
        ctx = C.next("attention_varlen_fwd" if packed else "attention_pair_fwd", what + " core").out
        Sq = 1 if first else S
        q = QKV[rows_d[:, 0], :H] if first else q_all
        self.core_ref(what, q, k_all, v_all, n, Sq, kr_ref, ctx, None if (first or not packed) else pflat)
        x = self.tail(C, what, 0, ctx, res)
        if first:
            return x
        # ---- middle layers and the last (token 0 only)
        for layer in range(1, L):
            what = "layer%d" % layer
            last = layer == L - 1
            wa = self.att(layer)
            if not packed and not self.fp8:
                n_rows = x.shape[0]
                fused = not last and ops.fused_attention_supported(n, S, H)
                blocks = lc.layer_blocks("cls" if last else "enc", self.layers[layer], x, n, S=S, fused=fused)
                blocks[0].key_real, blocks[0].mask = kr_ref, None
                x = lc.check_layer_fwd(self.t, C, blocks, self.arena, core=True)[-1]["y"]
                assert x.shape[0] == (n if last else n_rows)
                continue
            wqkv = self.arena.bf16_qkv(wa["q"], wa["k"], wa["v"])
            names = ("kv", slice(H, 3 * H), torch.cat([wa["bk"], wa["bv"]])) if last else \
                ("qkv", slice(0, 3 * H), torch.cat([wa["bq"], wa["bk"], wa["bv"]]))
            if self.fp8:
                proj = self.gemm(C, what + " " + names[0], self.quantized(C, what + " " + names[0], x), layer,
                                 names[0], names[2])
            else:
                proj = C.next("linear_fwd", what + " " + names[0]).out
                lc.check_linear(self.t, what + " " + names[0], proj, x, wqkv[names[1]], names[2].detach())
            if last:
                k, v = proj[:, :H], proj[:, H:]
                if packed:
                    x0 = x[starts.to(dev)]
                    c = C.next("gather_rows_varlen", what + " x0")
                    _exact(what + " x0 gather", c.out, x0)
                else:
                    x0 = x.view(n, S, H)[:, 0]
                qc = C.next("linear_fwd", what + " q")
                lc.check_linear(self.t, what + " q", qc.out, x0, wqkv[:H], wa["bq"].detach())
                q = qc.out
            else:
                q, k, v = proj[:, :H], proj[:, H:2 * H], proj[:, 2 * H:]
            ctx = C.next("attention_varlen_fwd" if packed else "attention_fwd", what + " core").out
            if not packed:
                ctx = ctx[0]                                          # (ctx, lse): p = 0, no backward reads lse
            if packed:
                qp = q if last else self.scatter(q, pflat, n)
                self.core_ref(what, qp, self.scatter(k, pflat, n), self.scatter(v, pflat, n), n, 1 if last else S,
                              kr_ref, ctx, None if last else pflat)
            else:
                self.core_ref(what, q, k, v, n, 1 if last else S, kr_ref, ctx)
            if last:
                s = lc.attn_out_fwd(self.t, C, what + " attn", ctx, x0, wa, self.arena)
                x = lc.ffn_fwd(self.t, C, what + " ffn", s["y"], self.ffn(layer), self.arena)["y"]
            else:
                x = self.tail(C, what, layer, ctx, x)
        return x

    def pooled(self, C, first):
        """the pooler's pre-activation of token 0 and PoolerSimFn -> (logits as the kernel wrote them, fp64 ref)"""
        dense = self.cross.pooler.dense
        c = C.next("linear_fwd", "pooler")
        lc.check_linear(self.t, "pooler", c.out, first, self.arena.bf16(dense.weight), dense.bias.detach())
        u = c.out
        c = C.next("pooler_sim", "pooler sim")
        _exact("pooler sim input", c.args["u"], u)
        sd = self.model.similarity_dense
        ref, bound = rc.pooler_sim_ref(u, sd.weight.detach(), sd.bias.detach())
        self.t.check("pooler sim", c.out, ref, bound)
        return c.out, ref


def grid_tiles(mt, mv, layout, budget):
    """(t0, t1, v0, v1) of the dense evaluation, from modeling's tiling of the masks' shapes / valid counts"""
    (Nt, W), (Nv, F) = mt.shape, mv.shape
    if layout == "packed":
        return modeling._packed_eval_tiles(mt.sum(1).tolist(), mv.sum(1).tolist(), budget)
    bt, bv = modeling._eval_tile(Nt, Nv, W + F, budget)
    return [(t0, min(Nt, t0 + bt), v0, min(Nv, v0 + bv)) for t0 in range(0, Nt, bt) for v0 in range(0, Nv, bv)]


def check_similarity(calls, model, arena, text2d, video2d, mask_t, mask_v, result, layout, fp8, budget,
                     pairs=None, perturb=(), label=""):
    """Walk one recorded evaluation call stage by stage.  text2d / video2d: the bf16 encoder outputs [Nt*W, H] /
    [Nv*F, H] it scored; result: its logits, [Nt, Nv] (pairs None: get_similarity_logits) or [P] (pairs = (text_index,
    video_index) host arrays: score_pairs).  layout: "padded" / "packed" as the call ran it (packed falls back to padded
    when a text row's token 0 is padded: decided here from the masks); fp8: UNIVL_EVAL_PRECISION=fp8 with >= 2 cross
    layers; budget: modeling.EVAL_PAIR_TOKENS.  -> (tally, fp64 reference of the result)"""
    w = Walk(model, arena, text2d, video2d, mask_t, mask_v, fp8, perturb, label)
    if layout == "packed" and not bool((w.mt[:, 0] != 0).all()):
        layout = "padded"
    C = lc.Calls(calls)
    if fp8:
        w.check_weights(C)
    w.check_sources(C)
    seen = torch.zeros(w.Nt, w.Nv, dtype=torch.long)
    if pairs is None:
        ref_out = torch.zeros(w.Nt, w.Nv, dtype=torch.float64)
        for t0, t1, v0, v1 in grid_tiles(w.mt, w.mv, layout, budget):
            nt, nv = t1 - t0, v1 - v0
            tile = [(i, j) for i in range(t0, t1) for j in range(v0, v1)]
            first = w.tile(C, tile, layout, False)
            got, ref = w.pooled(C, first)
            for p, (i, j) in enumerate(tile):
                seen[i, j] += 1
            if "transpose_tiles" in w.perturb:
                place = [(t0 + p % nt, v0 + p // nt) for p in range(nt * nv)]
            else:
                place = [(t0 + p // nv, v0 + p % nv) for p in range(nt * nv)]
            at = torch.tensor(place, dtype=torch.long)
            _exact("logits tile (%d:%d, %d:%d)" % (t0, t1, v0, v1), result.cpu()[at[:, 0], at[:, 1]],
                   got.to(result.dtype).cpu())
            ref_out[at[:, 0], at[:, 1]] = ref.cpu()
        assert bool((seen == 1).all()), "logits: pairs scored %s times" % seen.unique().tolist()
    else:
        ti, vi = (np.asarray(p, dtype=np.int64) for p in pairs)
        if layout == "packed":
            cost = w.mt.sum(1).numpy()[ti] + w.mv.sum(1).numpy()[vi]
        else:
            cost = np.full(ti.size, w.S, dtype=np.int64)
        ref_out = torch.zeros(ti.size, dtype=torch.float64)
        count = np.zeros(ti.size, dtype=np.int64)
        for a, b in retrieval._pair_chunks(cost, budget):
            chunk = [(int(ti[p]), int(vi[p])) for p in range(a, b)]
            first = w.tile(C, chunk, layout, True)
            got, ref = w.pooled(C, first)
            count[a:b] += 1
            idx = torch.arange(a, b)
            if "transpose_tiles" in w.perturb:
                idx = idx.flip(0)
            _exact("logits list [%d:%d]" % (a, b), result.cpu()[idx], got.to(result.dtype).cpu())
            ref_out[idx] = ref.cpu()
        assert bool((count == 1).all()), "logits: list entries scored %s times" % np.unique(count).tolist()
    C.done()
    return w.t, ref_out


def check_encoder(calls, model_layers, arena, mask, video_linear=None, label=""):
    """Walk the packed encoder layers of one embed_texts / embed_videos chunk (model_layers: their parameter tuples).
    video_linear: (weight, bias) of the visual embedding's linear, which runs first and is checked on its input.  The layers' input is the first
    QKV GEMM's (the packed embedding rows); every row is a sequence of its valid tokens in ascending position, its
    keys the row's mask -> (tally, the last layer's output rows)"""
    t = lc.Tally(label)
    C = lc.Calls(calls)
    m = mask.cpu().long()
    N, S = m.shape
    pflat = m.reshape(-1).nonzero()[:, 0]
    if video_linear is not None:
        c = C.next("linear_fwd", "video embedding")
        lc.check_linear(t, "video embedding", c.out, c.args["x"], arena.bf16(video_linear[0]),
                        video_linear[1].detach())
    x = next(c for c in C.q["linear_fwd"]).args["x"]
    for li, params in enumerate(model_layers):
        what = "enc layer%d" % li
        wa = dict(zip(ops.ATT_KEYS, params[:10]))
        qkv = C.next("linear_fwd", what + " qkv").out
        lc.check_linear(t, what + " qkv", qkv, x, arena.bf16_qkv(wa["q"], wa["k"], wa["v"]),
                        torch.cat([wa["bq"], wa["bk"], wa["bv"]]).detach())
        ctx = C.next("attention_varlen_fwd", what + " core").out
        q, k, v = (scatter(qkv[:, c * H:(c + 1) * H], pflat, N, S) for c in range(3))
        core_check(t, what, q, k, v, N, S, S, m, ctx, pflat)
        s = lc.attn_out_fwd(t, C, what + " attn", ctx, x, wa, arena)
        x = lc.ffn_fwd(t, C, what + " ffn", s["y"], dict(zip(ops.FFN_KEYS, params[10:16])), arena)["y"]
    C.done()
    return t, x
