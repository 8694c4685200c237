"""CPU: validate tests/eval_check.py without a GPU.  The ops primitives, the all-pairs embedding and PoolerSimFn are
replaced by CPU emulations (fp64, or fp32 arithmetic with bf16 stores and e4m3 codes where the kernels store them) and
the real evaluation orchestration runs on them through the checker's spies: UniVL._cross_similarity_eval (grid, padded
and packed, bf16 and FP8) and retrieval.score_pairs (listed pairs), with CrossModel's encode_pairs_first_token_eval*
and the ops.*_eval* layer functions under them.
- fp64: the checker's composed references equal oracle.univl_oracle's cross encoder + pooler + similarity_dense;
- fp32 with bf16 stores: every stage falls inside its bound, so the bounds are not too tight;
- a perturbed reference is rejected at the stage it perturbs."""
import contextlib
import math

import pytest
import torch

from oracle import synth
from oracle import univl_oracle as O
from tests import eval_check as ec
from tests import fp8_check as f8
from tests.model_util import build_model
from tests.test_cpu_layer_check import Emu, FakeArena
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200 import runtime as rt
from univl_b200.modules import modeling, module_cross

H = 768
NT, NV = 5, 4
W, F = 16, 12
S = W + F
BUDGET = 6 * S                     # several tiles, the last one partial, on every layout
TEXT_INDEX = [3, 0, 4, 1, 3, 2, 0]  # unsorted, (3, 2) listed twice
VIDEO_INDEX = [2, 1, 3, 0, 2, 3, 3]


class _TorchAlloc:
    """torch, with empty(dtype=bfloat16) allocating the emulation's storage dtype (CrossModel.first_layer_source_rows
    allocates its source-row buffer directly)"""

    def __init__(self, store):
        self.store = store

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *a, dtype=None, **k):
        return torch.empty(*a, dtype=self.store if dtype == torch.bfloat16 else dtype, **k)


class EvalEmu(Emu):
    """Emu plus the eval primitives"""

    NAMES = ("attention_pair_fwd", "attention_varlen_fwd", "gather_rows_varlen", "embed_src_rows_eval",
             "quantize_e4m3_rows", "quantize_e4m3_blocks", "gemm_fp8")

    def install(self, monkeypatch):
        super().install(monkeypatch)
        for name in self.NAMES:
            monkeypatch.setattr(ops, name, getattr(self, name))
        monkeypatch.setattr(ops.EmbedSrcFn, "apply", self.embed_src_all_pairs)
        monkeypatch.setattr(ops.PoolerSimFn, "apply", self.pooler_sim)
        monkeypatch.setattr(module_cross, "torch", _TorchAlloc(self.store))

    def _ln(self, z, gamma, beta):
        mean = z.mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((z - mean) ** 2).mean(-1, keepdim=True) + 1e-12)
        return self.c(gamma) * (z - mean) * rstd + self.c(beta)

    def _embed(self, a, N, n, pos, typ, off, ty):
        z = self.c(a).view(N, n, H) + self.c(pos[off:off + n]) + self.c(typ[ty])
        return self._ln(z, self.gamma, self.beta)

    def embed_src_rows_eval(self, a, N, W_, pos, type_w, gamma, beta, out):
        self.gamma, self.beta = gamma, beta
        out.copy_(self.st(self._embed(a, N, W_, pos, type_w, 0, 0).reshape(-1, H)))
        return out

    def embed_src_all_pairs(self, a, b, Na, Wa, Nb, Fb, all_pairs, pos, type_w, gamma, beta, p, training):
        assert all_pairs == 1 and not training
        self.gamma, self.beta = gamma, beta
        ta = self._embed(a, Na, Wa, pos, type_w, 0, 0)
        vb = self._embed(b, Nb, Fb, pos, type_w, Wa, 1)
        x = torch.cat([ta[:, None].expand(Na, Nb, Wa, H), vb[None].expand(Na, Nb, Fb, H)], 2)
        return self.st(x.reshape(-1, H))

    def pooler_sim(self, u, w, b):
        return torch.tanh(self.c(u)) @ self.c(w).reshape(-1) + self.c(b)

    def _seq(self, q, k, v):
        """one sequence, every key real: q [Sq, H], k / v [Sk, H] -> [Sq, H] in f"""
        qh, kh, vh = (self.c(t).reshape(t.shape[0], 12, 64).transpose(0, 1) for t in (q, k, v))
        P = torch.softmax(0.125 * qh @ kh.transpose(-1, -2), -1)
        return (P @ vh).transpose(0, 1).reshape(q.shape[0], H)

    def attention_pair_fwd(self, qkv_a, qkv_b, Na, Nb, Sq, mask, pairs=None):
        Wa, Fb = mask.Wa, mask.Fb
        if pairs is not None:
            ti, vi = (t.long() for t in pairs)
            key = torch.cat([mask.a, mask.b], 1)
        else:
            ti, vi = torch.arange(Na).repeat_interleave(Nb), torch.arange(Nb).repeat(Na)
            key = torch.cat([mask.a[ti], mask.b[vi]], 1)
        out = []
        for p in range(ti.numel()):
            rows = [qkv_a[ti[p] * Wa:(ti[p] + 1) * Wa], qkv_b[vi[p] * Fb:(vi[p] + 1) * Fb]]
            qkv = torch.cat(rows)
            real = key[p].bool()
            q = qkv[:Sq, :H]
            qh, kh, vh = (self.c(t).reshape(t.shape[0], 12, 64).transpose(0, 1)
                          for t in (q, qkv[:, H:2 * H], qkv[:, 2 * H:]))
            s = 0.125 * qh @ kh.transpose(-1, -2) + torch.where(real, 0.0, -10000.0).to(self.f)
            out.append((torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(Sq, H))
        return self.st(torch.cat(out))

    def _rows(self, a, b, seqs, p):
        """rows of sequence p under seqs' addressing: [(source, row index tensor)]"""
        cu = seqs.cu.long()
        n = int(cu[p + 1] - cu[p])
        if seqs.idx_a is None:
            return [(a, torch.arange(int(cu[p]), int(cu[p + 1])))]
        la = int(seqs.len_a[p])
        sa, sb = int(seqs.start_a[p]), int(seqs.start_b[p])
        return [(a, seqs.idx_a[sa:sa + la].long()), (b, seqs.idx_b[sb:sb + n - la].long())]

    def gather_rows_varlen(self, a, b, seqs, q_first):
        out = []
        for p in range(seqs.n_seq):
            r = torch.cat([src[i] for src, i in self._rows(a, b, seqs, p)])
            out.append(r[:1] if q_first else r)
        return torch.cat(out)

    def attention_varlen_fwd(self, q, k, v, seqs, q_first, qb=None, kb=None, vb=None):
        out = []
        for p in range(seqs.n_seq):
            K = torch.cat([src[i] for src, i in self._rows(k, kb, seqs, p)])
            V = torch.cat([src[i] for src, i in self._rows(v, vb, seqs, p)])
            if q_first and seqs.idx_a is None:
                Q = q[p:p + 1]
            else:
                Q = torch.cat([src[i] for src, i in self._rows(q, qb, seqs, p)])
                Q = Q[:1] if q_first else Q
            out.append(self._seq(Q, K, V))
        return self.st(torch.cat(out))

    def quantize_e4m3_rows(self, x):
        return f8.quant_rows(x)

    def quantize_e4m3_blocks(self, w, q=None, s=None):
        qq, ss = f8.quant_blocks(w)
        if q is None:
            return qq, ss
        q.view(torch.uint8).copy_(qq.view(torch.uint8))
        s.copy_(ss)
        return q, s

    def gemm_fp8(self, a, a_scale, b, b_scale, bias, gelu=False):
        acc = f8.deq_rows(a, a_scale).to(self.f) @ f8.deq_blocks(b, b_scale).to(self.f).t() + self.c(bias)
        if gelu:
            return f8.quant_rows(0.5 * acc * (1.0 + torch.erf(acc / math.sqrt(2.0))))
        return self.st(acc)


def _masks(seed):
    """as tests/test_gpu_packed_eval.py: ragged prefixes, scattered rows with token 0 kept, a fully padded video"""
    g = torch.Generator().manual_seed(seed)
    lt = torch.randint(1, W + 1, (NT,), generator=g)
    tm = (torch.arange(W)[None] < lt[:, None]).long()
    tm[1::2] = (torch.rand(tm[1::2].shape, generator=g) < 0.5).long()
    tm[:, 0] = 1
    lv = torch.randint(1, F + 1, (NV,), generator=g)
    vm = (torch.arange(F)[None] < lv[:, None]).long()
    vm[1::2] = (torch.rand(vm[1::2].shape, generator=g) < 0.5).long()
    vm[-1] = 0
    tm[0] = 1
    vm[0] = 1
    return tm, vm


def _case(layers, seed=0):
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=layers,
                            max_words=W, max_frames=F)
    sd = synth.make_state_dict(cfg, seed=seed)
    model = build_model(cfg, sd=sd, device="cpu").eval()
    g = torch.Generator().manual_seed(seed + 50)
    seq = torch.randn(NT, W, H, generator=g).to(torch.bfloat16)
    vis = torch.randn(NV, F, H, generator=g).to(torch.bfloat16)
    tm, vm = _masks(seed + 70)
    return cfg, sd, model, seq, vis, tm, vm


def _run(monkeypatch, mode, layout, precision, layers, exact=False, perturb=(), seed=0):
    """run one evaluation call on the emulation through the spies and walk it -> (tally, fp64 reference, case)"""
    cfg, sd, model, seq, vis, tm, vm = _case(layers, seed)
    emu = EvalEmu(exact)
    emu.install(monkeypatch)
    arena = FakeArena(emu.store)
    monkeypatch.setattr(rt._tls, "arena", arena, raising=False)
    monkeypatch.setattr(rt, "use_model", lambda *a, **k: contextlib.nullcontext(arena))
    monkeypatch.setattr(ops, "fused_attention_supported", lambda n, S_, H_: False)
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", BUDGET)
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", layout)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", precision)
    rec = ec.EvalRecorder().install(monkeypatch)
    text2d, video2d = seq.to(emu.store).reshape(-1, H), vis.to(emu.store).reshape(-1, H)
    with torch.no_grad():
        if mode == "grid":
            out = model._cross_similarity_eval(text2d, video2d, tm, vm)
            pairs = None
        else:
            out = retrieval.score_pairs(model, seq, vis, tm, vm, torch.tensor(TEXT_INDEX), torch.tensor(VIDEO_INDEX))
            pairs = (TEXT_INDEX, VIDEO_INDEX)
    fp8 = precision == "fp8" and layers > 1
    t, ref = ec.check_similarity(rec.calls, model, arena, text2d, video2d, tm, vm, out, layout, fp8, BUDGET, pairs,
                                 perturb=perturb, label="%s %s %s L=%d exact=%d" % (mode, layout, precision, layers,
                                                                                    exact))
    t.report()
    return t, ref, (cfg, sd, seq, vis, tm, vm)


@pytest.mark.parametrize("mode,layout", [("grid", "padded"), ("grid", "packed"), ("list", "padded"),
                                         ("list", "packed")])
def test_fp64_references_match_the_oracle(monkeypatch, mode, layout):
    """fp64 emulation: the walk's logit references equal the oracle's cross encoder, pooler and similarity_dense"""
    _, ref, (cfg, sd, seq, vis, tm, vm) = _run(monkeypatch, mode, layout, "bf16", 3, exact=True)
    sd64 = {k: v.double() for k, v in sd.items()}
    want = O.similarity_logits(seq.double(), vis.double(), tm, vm, sd64, cfg)
    if mode == "list":
        want = want[TEXT_INDEX, VIDEO_INDEX]
    torch.testing.assert_close(ref, want, rtol=0, atol=1e-10)


CASES = [("grid", "padded", "bf16", 3), ("grid", "padded", "fp8", 3), ("grid", "packed", "bf16", 3),
         ("grid", "packed", "fp8", 3), ("list", "padded", "bf16", 2), ("list", "padded", "fp8", 2),
         ("list", "packed", "fp8", 3), ("grid", "padded", "bf16", 1), ("list", "packed", "bf16", 1)]


@pytest.mark.parametrize("mode,layout,precision,layers", CASES)
def test_float32_emulation_is_within_the_bounds(monkeypatch, mode, layout, precision, layers):
    t, _, _ = _run(monkeypatch, mode, layout, precision, layers)
    assert max(t.worst.values()) < 1
    if precision == "fp8" and layers > 1:
        assert any("fp8 gemm" in k for k in t.worst)


@pytest.mark.parametrize("perturb,mode,layout,precision", [
    ("video_pos", "grid", "padded", "bf16"), ("video_type0", "list", "packed", "bf16"),
    ("res_next_video", "grid", "padded", "bf16"), ("drop_last_key", "grid", "packed", "bf16"),
    ("quant_prev", "grid", "padded", "fp8"), ("kv_as_qk", "list", "packed", "fp8"),
    ("scale_x2", "grid", "packed", "fp8"), ("transpose_tiles", "grid", "padded", "bf16"),
    ("transpose_tiles", "list", "padded", "bf16")])
def test_perturbed_references_are_rejected(monkeypatch, perturb, mode, layout, precision):
    with pytest.raises(AssertionError, match=ec.PERTURB[perturb]):
        _run(monkeypatch, mode, layout, precision, 2, perturb=(perturb,))
