"""CPU: validate tests/layer_check.py without a GPU.  The ops primitives are replaced by CPU emulations (fp64, or fp32
arithmetic with bf16 stores at the same stage boundaries as the kernels) and the real EncoderLayerFn /
EncoderLayerClsFn / DecoderLayerFn orchestration runs on them through the checker's spies.
- fp64 at p = 0: the checker's references agree with oracle.univl_oracle's encoder layer, and with the decoder layer
  composed from its multi_head_attention / dense_residual_norm, gradients by autograd;
- fp64 with dropout: they agree with an autograd statement of the layer with the host-Philox masks multiplied in;
- fp32 with bf16 stores: every stage falls inside the bounds, so they are not too tight;
- a perturbed reference is rejected."""
import math
import types

import pytest
import torch

from oracle import univl_oracle as orc
from tests import attn_check as ac
from tests import layer_check as lc
from univl_b200 import ops
from univl_b200 import runtime as rt
from univl_b200.modules import module_decoder, transformer

H = 768
SEED = (1 << 36) + 77
EPOCH = 2
STREAM0 = 5
PH, PA = 0.1, 0.2


class FakeArena:
    """what the layer functions read from the device arena: weight copies in the storage dtype, the RNG state, the
    stream counter"""

    def __init__(self, store):
        self.store = store
        self.root = types.SimpleNamespace()
        self.rng_state = torch.tensor([SEED, EPOCH], dtype=torch.int64)
        self.stream_counter = STREAM0
        self.epoch_host = 1
        self.seed = SEED                     # the emulated kernels take the Philox key itself

    def bf16(self, p):
        return p.detach().to(self.store)

    def bf16_qkv(self, q, k, v):
        return torch.cat([q, k, v]).detach().to(self.store)

    def next_stream(self):
        self.stream_counter += 1
        return self.stream_counter

    def check_epoch(self, epoch, p):
        pass


class Emu:
    """the ops primitives on CPU: arithmetic in `f`, activations stored in `store` (bf16 as the kernels, or fp64)"""

    def __init__(self, exact):
        self.f = torch.float64 if exact else torch.float32
        self.store = torch.float64 if exact else torch.bfloat16

    def install(self, monkeypatch):
        store, f = self.store, self.f
        monkeypatch.setattr(ops, "_empty", lambda shape, dtype, like: torch.empty(
            shape, dtype=store if dtype == torch.bfloat16 else (f if dtype == torch.float32 else dtype)))
        monkeypatch.setattr(ops, "_zeros", lambda shape, dtype, like: torch.zeros(
            shape, dtype=store if dtype == torch.bfloat16 else (f if dtype == torch.float32 else dtype)))
        for name in lc.PRIMITIVES:
            monkeypatch.setattr(ops, name, getattr(self, name))

    def c(self, t):
        return t.to(self.f)

    def st(self, t):
        return t.to(self.store)

    @staticmethod
    def _epoch():
        return int(rt.current().rng_state[1])

    def _gelu(self, x):
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))

    def _gelu_grad(self, x):
        return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)

    # GEMMs
    def linear_fwd(self, x, w16, bias, epi=ops.EPI_BIAS, aux_out=None, out_dtype=None, ld_out=None):
        acc = self.c(x) @ self.c(w16).t() + self.c(bias)
        if epi == ops.EPI_GELU:
            aux_out.copy_(self.st(acc))
            return self.st(self._gelu(acc))
        return self.st(acc)

    def linear_dgrad(self, dy, w16, epi=ops.EPI_BIAS, aux_in=None):
        acc = self.c(dy) @ self.c(w16)
        if epi == ops.EPI_GELU_BWD:
            acc = acc * self._gelu_grad(self.c(aux_in))
        elif epi == ops.EPI_ADD:
            acc = acc + self.c(aux_in)
        return self.st(acc)

    def linear_wgrad(self, dy, x, dw=None):
        dw.add_((self.c(dy).t() @ self.c(x)).to(dw.dtype))
        return dw

    def colsum(self, x, out=None):
        out.add_(self.c(x).sum(0).to(out.dtype))
        return out

    # LayerNorm (mode 1: z = x keep / (1 - p) + res)
    def _z(self, x, res, p, mode, seed, stream):
        z = self.c(x)
        if p > 0 and mode == 1:
            keep = ac.keep_elem(seed, ac.kernel_stream(stream, self._epoch()), p, *x.shape)
            z = z * keep.to(self.f) * lc.dense_scale(p)
        return z + self.c(res) if res is not None else z

    def layernorm_fwd(self, x, res, gamma, beta, p=0.0, mode=0, seed=0, stream=0):
        z = self._z(x, res, p, mode, seed, stream)
        mean = z.mean(1)
        rstd = 1.0 / torch.sqrt(((z - mean[:, None]) ** 2).mean(1) + 1e-12)
        y = self.c(gamma) * (z - mean[:, None]) * rstd[:, None] + self.c(beta)
        return self.st(y), mean, rstd

    def layernorm_bwd(self, dy, dy2, x, res, gamma, mean, rstd, p=0.0, mode=0, seed=0, stream=0, want_dbias=True,
                      want_dx=True, dgamma=None, dbeta=None, dbias=None):
        z = self._z(x, res, p, mode, seed, stream)
        xhat = (z - mean[:, None]) * rstd[:, None]
        d = self.c(dy) + (self.c(dy2) if dy2 is not None else 0)
        g = d * self.c(gamma)
        dz = rstd[:, None] * (g - g.mean(1, keepdim=True) - xhat * (g * xhat).mean(1, keepdim=True))
        kd = 1.0
        if p > 0 and mode == 1:
            kd = ac.keep_elem(seed, ac.kernel_stream(stream, self._epoch()), p, *x.shape).to(self.f) * \
                lc.dense_scale(p)
        dgamma.add_((d * xhat).sum(0).to(dgamma.dtype))
        dbeta.add_(d.sum(0).to(dbeta.dtype))
        dbias.add_((dz * kd).sum(0).to(dbias.dtype))
        dx_res = self.st(dz)
        dx_dense = self.st(dz * kd) if (p > 0 and mode == 1) else dx_res
        return dx_res, dx_dense, dgamma, dbeta, dbias

    # attention (layout "tile" / "rowmajor" of the dropout mask)
    def _probs(self, q, k, n_seq, Sq, Sk, mask):
        qh = self.c(q).reshape(n_seq, Sq, 12, 64).permute(0, 2, 1, 3)
        kh = self.c(k).reshape(n_seq, Sk, 12, 64).permute(0, 2, 1, 3)
        a = ac.additive_mask(lc.key_real_of(mask, n_seq), Sq, mask.causal)[:, None].to(self.f)
        return 0.125 * (qh @ kh.transpose(-1, -2)) + a, qh, kh

    def _keep(self, layout, p, seed, stream, n_seq, Sq, Sk):
        if p <= 0:
            return None
        ks = ac.kernel_stream(stream, self._epoch())
        m = ac.keep_rowmajor(seed, ks, p, n_seq * 12, Sq) if layout else ac.keep_tile(seed, ks, p, n_seq * 12, Sq, Sk)
        return m.view(n_seq, 12, Sq, Sk).to(self.f) / (1.0 - float(torch.tensor(p, dtype=torch.float32)))

    def _fwd(self, q, k, v, n_seq, Sq, Sk, mask, p, seed, stream, layout):
        s, _, _ = self._probs(q, k, n_seq, Sq, Sk, mask)
        lse = torch.logsumexp(s, -1)
        P = torch.exp(s - lse[..., None])
        M = self._keep(layout, p, seed, stream, n_seq, Sq, Sk)
        vh = self.c(v).reshape(n_seq, Sk, 12, 64).permute(0, 2, 1, 3)
        o = ((P * M if M is not None else P) @ vh).permute(0, 2, 1, 3).reshape(n_seq * Sq, H)
        return self.st(o), lse.reshape(-1)

    def _bwd(self, q, k, v, o, lse, d_o, n_seq, Sq, Sk, mask, p, seed, stream, layout):
        s, qh, kh = self._probs(q, k, n_seq, Sq, Sk, mask)
        P = torch.exp(s - lse.view(n_seq, 12, Sq)[..., None])
        M = self._keep(layout, p, seed, stream, n_seq, Sq, Sk)
        heads = lambda t, S: self.c(t).reshape(n_seq, S, 12, 64).permute(0, 2, 1, 3)
        vh, dO, Oh = heads(v, Sk), heads(d_o, Sq), heads(o, Sq)
        Pd = P * M if M is not None else P
        dV = Pd.transpose(-1, -2) @ dO
        dP = dO @ vh.transpose(-1, -2)
        D = (dO * Oh).sum(-1, keepdim=True)
        dS = 0.125 * P * ((dP * M if M is not None else dP) - D)
        un = lambda t: t.permute(0, 2, 1, 3).reshape(-1, H)
        return un(dS @ kh), un(dS.transpose(-1, -2) @ qh), un(dV)

    def attention_fwd(self, q, k, v, n_seq, Sq, Sk, mask, p=0.0, seed=0, stream=0):
        return self._fwd(q, k, v, n_seq, Sq, Sk, mask, p, seed, stream, False)

    def attention_bwd(self, q, k, v, o, lse, d_o, dq, dk, dv, n_seq, Sq, Sk, mask, p=0.0, seed=0, stream=0,
                      dbias=None, rng_layout=0):
        grads = self._bwd(q, k, v, o, lse, d_o, n_seq, Sq, Sk, mask, p, seed, stream, rng_layout == 1)
        for out, gr, db in zip((dq, dk, dv), grads, dbias):
            out.copy_(self.st(gr))
            db.add_(gr.sum(0).to(db.dtype))

    def fused_qkv_attention_fwd(self, x, wqkv, bqkv, n_seq, S, mask, p=0.0, seed=0, stream=0, save_qkv=True):
        qkv = self.st(self.c(x) @ self.c(wqkv).t() + self.c(bqkv))
        o, lse = self._fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], n_seq, S, S, mask, p, seed, stream, True)
        return o, lse, qkv

    def fused_attention_bwd(self, qkv, o, lse, d_o, dqkv, n_seq, S, mask, p=0.0, seed=0, stream=0, dbias=None):
        grads = self._bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], o, lse, d_o, n_seq, S, S, mask, p, seed,
                          stream, True)
        g = torch.cat(grads, 1)
        dqkv.copy_(self.st(g))
        dbias.add_(g.sum(0).to(dbias.dtype))


def _cfg():
    return types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                                 hidden_dropout_prob=PH, attention_probs_dropout_prob=PA)


def _layer(kind, seed):
    torch.manual_seed(seed)
    m = module_decoder.DecoderLayer(_cfg()) if kind == "dec" else transformer.EncoderLayer(_cfg())
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("LayerNorm.weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape))
            elif p.dim() == 1:
                p.copy_(0.1 * torch.randn(p.shape))
    return m


def _params(kind, m):
    if kind == "dec":
        return transformer.attention_param_list(m.slf_attn.att, m.slf_attn.output) + \
            transformer.attention_param_list(m.enc_attn.att, m.enc_attn.output) + \
            transformer.ffn_param_list(m.intermediate, m.output)
    return transformer._layer_params(m)


def _bf(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16)


N_SEQ, S, L, SE = 2, 16, 16, 32


def _run(monkeypatch, kind, exact, ph, pa, fused=True, seed=0, want=(), perturb=(), Se=SE):
    """run one layer on the emulation through the spies, check it -> (tally, param refs, refs, case dict)"""
    emu = Emu(exact)
    emu.install(monkeypatch)
    arena = FakeArena(emu.store)
    monkeypatch.setattr(rt._tls, "arena", arena, raising=False)
    monkeypatch.setattr(ops, "fused_attention_supported", lambda n_seq, S, H: fused)
    rec = lc.Recorder().install(monkeypatch)
    m = _layer(kind, seed)
    params = _params(kind, m)
    key_real = ac.edge_masks(N_SEQ, Se if kind == "dec" else S, seed + 1, kinds=(4, 0))
    T = N_SEQ * (L if kind == "dec" else S)
    x = _bf((T, H), seed + 2).to(emu.store)
    dy = _bf((N_SEQ if kind == "cls" else T, H), seed + 3).to(emu.store)
    xg = x.clone().requires_grad_()
    enc = enc_g = None
    if kind == "dec":
        enc = _bf((N_SEQ * Se, H), seed + 4).to(emu.store)
        enc_g = enc.clone().requires_grad_()
        slf = ops.MaskSpec(ac.edge_masks(N_SEQ, L, seed + 5, kinds=(4,)), causal=True)
        encm = ops.MaskSpec(key_real[:, :Se // 2].contiguous(), key_real[:, Se // 2:].contiguous())
        out = ops.DecoderLayerFn.apply(xg, enc_g, N_SEQ, L, Se, slf, encm, ph, pa, True, *params)
        blocks = lc.layer_blocks(kind, params, x, N_SEQ, enc=enc, L=L, Se=Se, slf_mask=slf, enc_mask=encm,
                                 fused=fused)
    else:
        mask = ops.MaskSpec(key_real)
        fn = ops.EncoderLayerClsFn if kind == "cls" else ops.EncoderLayerFn
        out = fn.apply(xg, N_SEQ, S, mask, ph, pa, True, *params)
        blocks = lc.layer_blocks(kind, params, x, N_SEQ, S=S, mask=mask, fused=fused and kind == "enc")
    out.backward(dy)
    t, pr, refs = lc.check_layer(rec.calls, blocks, arena, ph, pa, STREAM0, dy, out.detach(), xg.grad,
                                 denc=enc_g.grad if enc_g is not None else None,
                                 fold_rows=(N_SEQ, S) if kind == "cls" else None, perturb=perturb,
                                 label="%s exact=%d" % (kind, exact), want=want)
    lc.check_param_grads(t, blocks, pr, lambda p: p.grad)
    t.report()
    return t, pr, refs, dict(m=m, params=params, blocks=blocks, x=x, dy=dy, enc=enc, key_real=key_real)


@pytest.mark.parametrize("kind,fused", [("enc", True), ("enc", False), ("cls", False), ("dec", True)])
def test_float32_emulation_is_within_the_bounds(monkeypatch, kind, fused):
    """fp32 arithmetic with bf16 stores where the kernels store bf16, dropout on with p_hidden != p_attn"""
    t, _, _, _ = _run(monkeypatch, kind, False, PH, PA, fused, seed=3)
    assert len(t.worst) > 30


def _oracle_sd(m):
    return {k: v.detach().double().clone().requires_grad_() for k, v in m.state_dict().items()}


def _compare(refs, pr, blocks, want, grads_of_param, what):
    for name, ref in refs.items():
        torch.testing.assert_close(ref, want[name], rtol=1e-6, atol=1e-8, msg=lambda s: "%s %s: %s" % (what, name, s))
    for (bi, k), (ref, _) in pr.items():
        got = grads_of_param(blocks[bi].w[k])
        torch.testing.assert_close(ref, got, rtol=1e-5, atol=1e-8, msg=lambda s: "%s grad %d %s: %s" % (what, bi, k, s))


def _sd_grad(m, sd):
    by_ptr = {p.data_ptr(): name for name, p in m.named_parameters()}
    return lambda p: sd[by_ptr[p.data_ptr()]].grad


def test_matches_the_oracle_encoder_layer_at_p0(monkeypatch):
    """fp64 emulation at p = 0: the checker's output, dx and all 16 parameter-gradient references equal
    oracle.univl_oracle.encoder_layer and its autograd gradients"""
    _, pr, refs, c = _run(monkeypatch, "enc", True, 0.0, 0.0, True, seed=5, want=("out", "dx"))
    sd = _oracle_sd(c["m"])
    x = c["x"].clone().requires_grad_()
    y = orc.encoder_layer(x.view(N_SEQ, S, H), orc.additive_mask(c["key_real"], torch.float64), sd, "")
    y.backward(c["dy"].view(N_SEQ, S, H))
    _compare(refs, pr, c["blocks"], {"out": y.detach().view(-1, H), "dx": x.grad}, _sd_grad(c["m"], sd), "encoder")


def test_matches_the_oracle_decoder_layer_at_p0(monkeypatch):
    """the decoder layer composed from the oracle's multi_head_attention / dense_residual_norm (caption_decoder's
    per-layer statement): output, dx, denc and all 26 parameter gradients"""
    _, pr, refs, c = _run(monkeypatch, "dec", True, 0.0, 0.0, True, seed=6, want=("out", "dx", "denc"))
    sd = _oracle_sd(c["m"])
    x = c["x"].clone().requires_grad_()
    enc = c["enc"].clone().requires_grad_()
    ans = ac.edge_masks(N_SEQ, L, 6 + 5, kinds=(4,)).double()[:, None, None, :]
    fut = torch.triu(torch.ones(L, L, dtype=torch.float64), diagonal=1)[None, None]
    slf_add = ((1.0 - ans) + fut).gt(0).double() * -10000.0
    enc_add = orc.additive_mask(c["key_real"], torch.float64)
    x3, e3 = x.view(N_SEQ, L, H), enc.view(N_SEQ, SE, H)
    s = orc.dense_residual_norm(orc.multi_head_attention(x3, x3, slf_add, sd, "slf_attn.att."), x3, sd, "slf_attn.output.")
    d = orc.dense_residual_norm(orc.multi_head_attention(s, e3, enc_add, sd, "enc_attn.att."), s, sd, "enc_attn.output.")
    y = orc.dense_residual_norm(orc.gelu(orc.linear(d, sd, "intermediate.dense")), d, sd, "output.")
    y.backward(c["dy"].view(N_SEQ, L, H))
    _compare(refs, pr, c["blocks"], {"out": y.detach().view(-1, H), "dx": x.grad, "denc": enc.grad},
             _sd_grad(c["m"], sd), "decoder")


def test_matches_an_autograd_layer_with_the_masks_multiplied_in(monkeypatch):
    """fp64 emulation with dropout: the references equal an autograd statement of the encoder layer whose attention
    probabilities and dense outputs are multiplied by the host-Philox masks of streams STREAM0 + 1, + 2, + 3"""
    _, pr, refs, c = _run(monkeypatch, "enc", True, PH, PA, True, seed=7, want=("out", "dx"))
    sd = _oracle_sd(c["m"])
    x = c["x"].clone().requires_grad_()
    T = N_SEQ * S
    ka = ac.keep_rowmajor(SEED, ac.kernel_stream(STREAM0 + 1, EPOCH), PA, N_SEQ * 12, S).double()
    ka = ka.view(N_SEQ, 12, S, S) / (1.0 - float(torch.tensor(PA, dtype=torch.float32)))
    k1 = ac.keep_elem(SEED, ac.kernel_stream(STREAM0 + 2, EPOCH), PH, T, H).double() * lc.dense_scale(PH)
    k2 = ac.keep_elem(SEED, ac.kernel_stream(STREAM0 + 3, EPOCH), PH, T, H).double() * lc.dense_scale(PH)
    split = lambda t: t.view(N_SEQ, S, 12, 64).permute(0, 2, 1, 3)
    pf = "attention.self."
    q, k, v = (split(orc.linear(x, sd, pf + n)) for n in ("query", "key", "value"))
    a = orc.additive_mask(c["key_real"], torch.float64)
    P = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + a, -1) * ka
    ctx = (P @ v).permute(0, 2, 1, 3).reshape(T, H)
    ln = lambda z, pfx: orc.layer_norm(z, sd[pfx + "LayerNorm.weight"], sd[pfx + "LayerNorm.bias"])
    y1 = ln(orc.linear(ctx, sd, "attention.output.dense") * k1 + x, "attention.output.")
    y = ln(orc.linear(orc.gelu(orc.linear(y1, sd, "intermediate.dense")), sd, "output.dense") * k2 + y1, "output.")
    y.backward(c["dy"])
    _compare(refs, pr, c["blocks"], {"out": y.detach(), "dx": x.grad}, _sd_grad(c["m"], sd), "masked encoder")


@pytest.mark.parametrize("kind,perturb,stage", [("enc", "stream+1", "core ctx"), ("enc", "tile_layout", "core ctx"),
                                                ("enc", "swap_p", "ctx|ln"), ("enc", "no_dy2", "ln bwd g"),
                                                ("enc", "no_dense_scale", "ln bwd gd"), ("cls", "no_fold", "fold"),
                                                ("dec", "kv_from_x", "grad block1 k")])
def test_perturbed_references_are_rejected(monkeypatch, kind, perturb, stage):
    with pytest.raises(AssertionError, match=stage):     # kv_from_x: Se = L, so x and enc have one shape
        _run(monkeypatch, kind, False, PH, PA, kind != "cls", seed=3, perturb=(perturb,), Se=L if kind == "dec" else SE)
