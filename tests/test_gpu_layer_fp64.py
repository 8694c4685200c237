"""GPU: whole transformer layers (EncoderLayerFn, EncoderLayerClsFn, DecoderLayerFn) checked stage by stage against
fp64 (tests/layer_check.py) with dropout on, p_hidden != p_attn, and again at p = 0: every saved intermediate, both
block outputs, every backward output and every parameter gradient per element, the dropout masks reproduced by the
host Philox from the stream ids the reference layer's sites draw.  Also: the flat gradient sink, a stream census of
one training step, and negative checks that perturb the reference and show the bounds reject the kernels' result.
Each check prints its worst err / bound per stage as "ratio"."""
import copy
import types

import pytest
import torch

from tests import attn_check as ac
from tests import layer_check as lc
from univl_b200 import ops
from univl_b200 import runtime as rt
from univl_b200.modules import module_decoder, transformer

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
H = 768
SEED = (1 << 40) + 0x13579BDF     # rng_state[0]: bits above 32 are part of the Philox key
EPOCH = 5                          # rng_state[1]
STREAM0 = 40                       # the arena's stream counter before the layer
PH, PA = 0.1, 0.2                  # p_hidden != p_attn, so a swap of the two is visible


def _cfg(ph=PH, pa=PA):
    return types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                                 hidden_dropout_prob=ph, attention_probs_dropout_prob=pa)


def _layer(kind, seed):
    """a parameter holder (the arena makes its bf16 copies) with LayerNorm and bias parameters away from 1 / 0"""
    torch.manual_seed(seed)
    m = module_decoder.DecoderLayer(_cfg()) if kind == "dec" else transformer.EncoderLayer(_cfg())
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("LayerNorm.weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return m.to(DEV)


def _params(kind, m):
    if kind == "dec":
        return transformer.attention_param_list(m.slf_attn.att, m.slf_attn.output) + \
            transformer.attention_param_list(m.enc_attn.att, m.enc_attn.output) + \
            transformer.ffn_param_list(m.intermediate, m.output)
    return transformer._layer_params(m)


def _bf_randn(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, device=DEV, generator=g).to(BF16)


class Case:
    """one layer call with its inputs; run() does forward + backward under the model context at a fixed RNG state"""

    def __init__(self, kind, n_seq, S=None, mask=None, L=None, Se=None, slf_mask=None, enc_mask=None, ph=PH, pa=PA,
                 enc_grad=True, seed=0, m=None):
        self.kind, self.n_seq, self.S, self.mask = kind, n_seq, S, mask
        self.L, self.Se, self.slf_mask, self.enc_mask = L, Se, slf_mask, enc_mask
        self.ph, self.pa, self.enc_grad = ph, pa, enc_grad
        self.m = m if m is not None else _layer(kind, seed)
        self.params = _params(kind, self.m)
        T = n_seq * (L if kind == "dec" else S)
        self.x = _bf_randn((T, H), seed + 2)
        self.enc = _bf_randn((n_seq * Se, H), seed + 3) if kind == "dec" else None
        self.dy = _bf_randn((n_seq if kind == "cls" else T, H), seed + 4)

    def run(self, reset_grads=True):
        """reset_grads: drop the parameters' gradients first (not under a flat sink, whose views they are)"""
        for p in self.params:
            if reset_grads:
                p.grad = None
        dev = torch.device("cuda", torch.cuda.current_device())
        with rt.use_model(self.m, dev) as arena:
            arena.seed
            arena.rng_state.copy_(torch.tensor([SEED, EPOCH], device=DEV))
            arena.stream_counter = STREAM0
            x = self.x.clone().requires_grad_()
            if self.kind == "dec":
                enc = self.enc.clone().requires_grad_(self.enc_grad)
                out = ops.DecoderLayerFn.apply(x, enc, self.n_seq, self.L, self.Se, self.slf_mask, self.enc_mask,
                                               self.ph, self.pa, True, *self.params)
            else:
                enc = None
                fn = ops.EncoderLayerClsFn if self.kind == "cls" else ops.EncoderLayerFn
                out = fn.apply(x, self.n_seq, self.S, self.mask, self.ph, self.pa, True, *self.params)
            out.backward(self.dy)
        torch.cuda.synchronize()
        self.arena = arena
        self.out, self.dx = out.detach(), x.grad
        self.denc = enc.grad if enc is not None and self.enc_grad else None
        return [self.out, self.dx] + ([self.denc] if self.denc is not None else []) + \
            [p.grad.clone() if p.grad is not None else None for p in self.params]

    def blocks(self, fused):
        return lc.layer_blocks(self.kind, self.params, self.x, self.n_seq, S=self.S, mask=self.mask, enc=self.enc,
                               L=self.L, Se=self.Se, slf_mask=self.slf_mask, enc_mask=self.enc_mask, fused=fused)

    def check(self, calls, fused, fused_bwd=True, perturb=(), label="", grads=True):
        blocks = self.blocks(fused)
        t, pr, _ = lc.check_layer(calls, blocks, self.arena, self.ph, self.pa, STREAM0, self.dy, self.out, self.dx,
                                  denc=self.denc, fold_rows=(self.n_seq, self.S) if self.kind == "cls" else None,
                                  perturb=perturb, label=label, fused_bwd=fused_bwd)
        if grads:
            n = lc.check_param_grads(t, blocks, pr, lambda p: p.grad)
            assert n == (26 if self.kind == "dec" else 16)
        return t


def _record(monkeypatch, case):
    rec = lc.Recorder().install(monkeypatch)
    case.run()
    return rec


def _uses(rec, name):
    return any(c.name == name for c in rec.calls)


def _masks(n_seq, S, seed, kinds=(0, 1, 2, 3, 4)):
    return ac.edge_masks(n_seq, S, seed, kinds).to(DEV)


# ---------------------------------------------------------------------------------------------------------
# EncoderLayerFn
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("what,p", [("text", (PH, PA)), ("text", (0.0, 0.0)), ("video", (PH, PA))])
def test_encoder_layer_fused_fp64(monkeypatch, what, p):
    """the bench shape 32 x 48: fused QKV + attention forward (row-major masks), wgmma backward, LayerNorm mode 1 at
    both sites; text with edge-case key masks, video with prefix masks.  The spies change no bit."""
    n_seq, S = 32, 48
    mask = _masks(n_seq, S, 7, (0, 1, 2, 3, 4) if what == "text" else (4,))
    case = Case("enc", n_seq, S, ops.MaskSpec(mask), ph=p[0], pa=p[1], seed=11 if what == "text" else 12)
    plain = case.run()
    rec = _record(monkeypatch, case)
    spied = [case.out, case.dx] + [q.grad for q in case.params]
    for a, b in zip(plain, spied):
        assert torch.equal(a, b), "a spied run differs from an unspied one"
    assert _uses(rec, "fused_qkv_attention_fwd") and _uses(rec, "fused_attention_bwd")
    case.check(rec.calls, fused=True, label="enc fused %s p=%s" % (what, p)).report()


def test_encoder_layer_fused_fwd_mma_bwd_fp64(monkeypatch):
    """UNIVL_FUSED_ATTN_BWD=0: the fused forward's row-major masks regenerated by the mma.sync backward (rng_layout 1)"""
    monkeypatch.setenv("UNIVL_FUSED_ATTN_BWD", "0")
    n_seq, S = 32, 48
    case = Case("enc", n_seq, S, ops.MaskSpec(_masks(n_seq, S, 8)), seed=13)
    rec = _record(monkeypatch, case)
    bwd = [c for c in rec.calls if c.name == "attention_bwd"]
    assert len(bwd) == 1 and bwd[0].args["rng_layout"] == 1
    case.check(rec.calls, fused=True, fused_bwd=False, label="enc fused fwd mma bwd").report()


@pytest.mark.parametrize("n_seq,S,env,p", [(8, 33, None, (PH, PA)), (8, 33, None, (0.0, 0.0)),
                                           (16, 48, "0", (PH, PA)), (2, 300, None, (PH, PA))])
def test_encoder_layer_unfused_fp64(monkeypatch, n_seq, S, env, p):
    """QKV GEMM + attention core: S = 33 (a partial 16-key tile), the fused path switched off at S = 48, and the
    key-tiled core at S = 300; tile-layout masks"""
    if env is not None:
        monkeypatch.setenv("UNIVL_FUSED_ATTN", env)
    case = Case("enc", n_seq, S, ops.MaskSpec(_masks(n_seq, S, S)), ph=p[0], pa=p[1], seed=S)
    rec = _record(monkeypatch, case)
    assert not _uses(rec, "fused_qkv_attention_fwd")
    case.check(rec.calls, fused=False, label="enc unfused n%d S%d p=%s" % (n_seq, S, p)).report()


# ---------------------------------------------------------------------------------------------------------
# cross layers: all-pairs masks, and the first-token layer
# ---------------------------------------------------------------------------------------------------------
def _pair_case(kind, Na, Nb, G, seed, p=(PH, PA)):
    W = F = 48
    ma = ac.edge_masks(Na, W, seed, kinds=(4, 0, 2, 1)).to(DEV)
    mb = ac.edge_masks(Nb, F, seed + 1, kinds=(4, 0, 1)).to(DEV)
    return Case(kind, Na * Nb // G, W + F, ops.MaskSpec(ma, mb, all_pairs=G), ph=p[0], pa=p[1], seed=seed)


@pytest.mark.parametrize("kind", ["enc", "cls"])
@pytest.mark.parametrize("Na,G,p", [(8, 1, (PH, PA)), (8, 2, (PH, PA)), (8, 1, (0.0, 0.0)), (32, 1, (PH, PA))])
def test_cross_layer_pairs_fp64(monkeypatch, kind, Na, G, p):
    """MaskSpec(..., all_pairs=G) at 8 x 8 pairs x 96 tokens and at the FT-Align bench shape 32 x 32 x 96 (98 304
    rows).  EncoderLayerClsFn: the query side on the token-0 rows (Sq = 1 masks) and the row-0 gradient fold."""
    case = _pair_case(kind, Na, Na, G, 20 + Na + G)
    case.ph, case.pa = p
    rec = _record(monkeypatch, case)
    fused = kind == "enc"
    assert _uses(rec, "fused_qkv_attention_fwd") == fused
    case.check(rec.calls, fused=fused, label="%s pairs %dx%d G%d p=%s" % (kind, Na, Na, G, p)).report()


# ---------------------------------------------------------------------------------------------------------
# DecoderLayerFn
# ---------------------------------------------------------------------------------------------------------
def _dec_case(n_seq, L, Se, enc_grad, seed, p=(PH, PA)):
    answer = ac.edge_masks(n_seq, L, seed, kinds=(4,)).to(DEV)          # answer padding: random prefixes
    W = Se // 2
    ea = ac.edge_masks(n_seq, W, seed + 1, kinds=(4, 0)).to(DEV)
    eb = ac.edge_masks(n_seq, Se - W, seed + 2, kinds=(4, 1)).to(DEV)
    return Case("dec", n_seq, L=L, Se=Se, slf_mask=ops.MaskSpec(answer, causal=True), enc_mask=ops.MaskSpec(ea, eb),
                ph=p[0], pa=p[1], enc_grad=enc_grad, seed=seed)


@pytest.mark.parametrize("enc_grad,p", [(True, (PH, PA)), (False, (PH, PA)), (True, (0.0, 0.0))])
def test_decoder_layer_fp64(monkeypatch, enc_grad, p):
    """the caption shape: L = 48 (causal + answer padding), Se = 96; three blocks sharing one _Drop, cross-attention
    K/V from enc, denc (or none when enc needs no gradient)"""
    case = _dec_case(32, 48, 96, enc_grad, 31, p)
    rec = _record(monkeypatch, case)
    assert (case.denc is not None) == enc_grad
    case.check(rec.calls, fused=True, label="dec enc_grad=%d p=%s" % (enc_grad, p)).report()


# ---------------------------------------------------------------------------------------------------------
# the flat gradient sink
# ---------------------------------------------------------------------------------------------------------
def test_flat_gradient_sink_fp64(monkeypatch):
    """one encoder layer registered through optim.flatten: the backward adds into the flat views (autograd receives
    None, so nothing is added twice), two forward / backward pairs accumulate to g1 + g2 within the bound, and the q/k/v
    bias as a zero-copy view of the flat buffer gives the same bits as the concatenated copy of separate parameters"""
    from univl_b200 import optim
    n_seq, S = 16, 48
    mask = ops.MaskSpec(_masks(n_seq, S, 41))
    base = _layer("enc", 41)
    plain = Case("enc", n_seq, S, mask, m=copy.deepcopy(base), seed=41)
    want = plain.run()
    flat_case = Case("enc", n_seq, S, mask, m=base, seed=41)
    flat = optim.flatten(base)
    wa = dict(zip(ops.ATT_KEYS, flat_case.params[:10]))
    assert rt.packed_bias(wa["bq"], wa["bk"], wa["bv"]).data_ptr() == wa["bq"].data_ptr()
    pp = dict(zip(ops.ATT_KEYS, plain.params[:10]))
    assert rt.packed_bias(pp["bq"], pp["bk"], pp["bv"]).data_ptr() != pp["bq"].data_ptr()
    flat.zero_grad()
    views = [flat.grad_view(p) for p in flat_case.params]

    def run_flat(case):
        case.run(reset_grads=False)

    run_flat(flat_case)
    got1 = [flat_case.out, flat_case.dx] + [v.clone() for v in views]
    for a, b in zip(want, got1):
        assert torch.equal(a, b), "the zero-copy bias view and the concatenated copy differ"
    for p, v in zip(flat_case.params, views):
        assert p.grad is not None and p.grad.data_ptr() == v.data_ptr(), "autograd replaced a flat gradient view"
    # two recorded forward / backward pairs with different inputs, accumulated into the zeroed sink
    flat.zero_grad()
    rec = lc.Recorder().install(monkeypatch)
    prs = []
    for i in range(2):
        rec.clear()
        flat_case.x = _bf_randn((n_seq * S, H), 50 + i)
        flat_case.dy = _bf_randn((n_seq * S, H), 60 + i)
        run_flat(flat_case)
        blocks = flat_case.blocks(True)
        t, pr, _ = lc.check_layer(rec.calls, blocks, flat_case.arena, PH, PA, STREAM0, flat_case.dy, flat_case.out,
                                  flat_case.dx, label="flat sink pass %d" % i)
        t.report()
        prs.append((blocks, pr))
    blocks = prs[0][0]
    total = {k: lc.sum_refs(prs[0][1][k], prs[1][1][k]) for k in prs[0][1]}
    t = lc.Tally("flat sink g1 + g2")
    assert lc.check_param_grads(t, blocks, total, lambda p: flat.grad_view(p)) == 16
    t.report()
    rt.set_grad_sink(None, base)


# ---------------------------------------------------------------------------------------------------------
# stream census of one training step
# ---------------------------------------------------------------------------------------------------------
def test_dropout_stream_census(monkeypatch):
    """one FT-Align training step at dropout 0.1 through the spies: every dropout site with p > 0 draws its own stream
    id, all below 2^20 (the epoch's shift), and each backward regenerates its mask from its own forward's id"""
    from oracle import synth
    from tests.model_util import build_model, to_device
    cfg = synth.task_config(mode="ft_align", batch_size=6, text_layers=2, visual_layers=1, cross_layers=2,
                            max_words=16, max_frames=12)
    torch.manual_seed(3)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=2), dropout=0.1)
    batch = to_device(synth.make_batch(cfg, seed=3))
    rec = lc.Recorder().install(monkeypatch)
    model(**batch).backward()
    torch.cuda.synchronize()
    fwd = {}
    ids = []
    for c in rec.calls:
        if c.name in lc.DROPOUT_FWD and c.args["p"] > 0:
            ids.append(c.args["stream"])
            key = c.out[1].data_ptr()                 # layernorm_fwd: mean; attention forwards: lse
            assert key not in fwd, "two live forwards share one saved statistic"
            fwd[key] = c.args["stream"]
    assert len(ids) >= 3 * (2 + 1 + 2), ids
    assert len(set(ids)) == len(ids), "two dropout sites draw the same stream: %s" % ids
    assert all(0 < s < 2 ** 20 for s in ids), ids
    n_bwd = 0
    for c in rec.calls:
        if c.name in ("layernorm_bwd", "attention_bwd", "fused_attention_bwd") and c.args["p"] > 0:
            key = (c.args["mean"] if c.name == "layernorm_bwd" else c.args["lse"]).data_ptr()
            assert key in fwd and c.args["stream"] == fwd[key], "%s regenerates another site's mask" % c.name
            n_bwd += 1
    assert n_bwd == len(ids)


# ---------------------------------------------------------------------------------------------------------
# negative checks: perturb the reference, the bound must reject the kernels' result
# ---------------------------------------------------------------------------------------------------------
def _rejects(case, calls, perturb, stage, **kw):
    with pytest.raises(AssertionError, match=stage):
        case.check(calls, perturb=(perturb,), label="perturbed: " + perturb, **kw)


def test_checker_rejects_wiring_errors(monkeypatch):
    n_seq, S = 32, 48
    case = Case("enc", n_seq, S, ops.MaskSpec(_masks(n_seq, S, 9)), seed=14)
    rec = _record(monkeypatch, case)
    case.check(rec.calls, fused=True, label="unperturbed")
    _rejects(case, rec.calls, "stream+1", "core ctx", fused=True)          # the neighbouring stream's mask
    _rejects(case, rec.calls, "tile_layout", "core ctx", fused=True)       # tile layout for the fused forward
    _rejects(case, rec.calls, "swap_p", "ctx|ln", fused=True)              # p_hidden and p_attn swapped
    _rejects(case, rec.calls, "no_dy2", "block0 attn ln bwd g", fused=True)
    _rejects(case, rec.calls, "no_dense_scale", "ln bwd gd", fused=True)
    rec.clear()
    cls = _pair_case("cls", 4, 4, 1, 15)
    cls.run()
    cls.check(rec.calls, fused=False, label="cls unperturbed")
    _rejects(cls, rec.calls, "no_fold", "row-0 fold", fused=False)
    rec.clear()
    dec = _dec_case(8, 48, 48, True, 16)                                    # Se = L: x and enc have one shape
    dec.run()
    dec.check(rec.calls, fused=True, label="dec unperturbed")
    _rejects(dec, rec.calls, "kv_from_x", "grad block1 k", fused=True)
