"""GPU: the cross encoder's evaluation paths checked stage by stage against fp64 (tests/eval_check.py): the all-pairs
grid (get_similarity_logits), listed pairs (score_pairs) and the packed layout, in bf16 and FP8, with 1-3 cross
layers, at 16 + 12, 48 + 48 and 128 + 160 tokens (288 keys: the key-tiled attention kernel).  Every embedding row,
projection, attention core, LayerNorm, FP8 quantization and GEMM, the pooler, PoolerSimFn and each logit's place are
checked per element, from the source rows to the [Nt, Nv] result, and each pair is scored exactly once.  Also the
packed encoder layers of embed_texts / embed_videos on rows whose valid tokens are scattered, and negative checks
that perturb the reference on real recorded calls.  Each check prints its worst err / bound per stage as "ratio"."""
import pytest
import torch

from oracle import synth
from tests import eval_check as ec
from tests.model_util import build_model
from univl_b200 import ops
from univl_b200 import retrieval
from univl_b200 import runtime as rt
from univl_b200.modules import modeling
from univl_b200.modules.transformer import _layer_params

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768
NT, NV = 5, 4
TEXT_INDEX = [3, 0, 4, 1, 3, 2, 0]  # unsorted, (3, 2) listed twice
VIDEO_INDEX = [2, 1, 3, 0, 2, 3, 3]


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _masks(W, F, seed):
    """as tests/test_gpu_packed_eval.py: ragged prefixes (even rows), scattered rows with token 0 kept (odd rows), the
    last video fully padded; text row 0 and video row 0 full, so the longest pair has all W + F tokens"""
    g = _g(seed)
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
    return tm.to(DEV), vm.to(DEV)


def _case(layers, W, F, seed=0):
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=layers,
                            max_words=W, max_frames=F)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=seed)).eval()
    g = _g(seed + 50)
    seq = torch.randn(NT, W, H, generator=g).to(torch.bfloat16).to(DEV)
    vis = torch.randn(NV, F, H, generator=g).to(torch.bfloat16).to(DEV)
    tm, vm = _masks(W, F, seed + 70)
    return model, seq, vis, tm, vm


class Entries:
    """the C entry points a call ran (ops.call spied)"""

    def __init__(self, monkeypatch):
        self.names = set()
        call = ops.call

        def spy(name, *a):
            self.names.add(name)
            return call(name, *a)
        monkeypatch.setattr(ops, "call", spy)


def _record(monkeypatch, model, args, mode, layout, precision, budget):
    """one evaluation call under the spies -> (calls, result, entries, arena)"""
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", layout)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", precision)
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", budget)
    ent = Entries(monkeypatch)
    rec = ec.EvalRecorder().install(monkeypatch)
    seq, vis, tm, vm = args
    with torch.no_grad(), rt.use_model(model, torch.device(DEV, torch.cuda.current_device())) as arena:
        if mode == "grid":
            out = model.get_similarity_logits(seq, vis, tm, vm)
        else:
            out = retrieval.score_pairs(model, seq, vis, tm, vm, torch.tensor(TEXT_INDEX, device=DEV),
                                        torch.tensor(VIDEO_INDEX, device=DEV))
    torch.cuda.synchronize()
    monkeypatch.undo()
    return rec.calls, out, ent.names, arena


def _walk(model, arena, args, calls, out, mode, layout, fp8, budget, perturb=(), label=""):
    seq, vis, tm, vm = args
    pairs = None if mode == "grid" else (TEXT_INDEX, VIDEO_INDEX)
    with torch.no_grad(), rt.use_model(model, torch.device(DEV, torch.cuda.current_device())):
        return ec.check_similarity(calls, model, arena, seq.reshape(-1, H), vis.reshape(-1, H), tm, vm, out, layout,
                                   fp8, budget, pairs, perturb=perturb, label=label)


@pytest.mark.parametrize("W,F", [(16, 12), (48, 48), (128, 160)])
@pytest.mark.parametrize("layers", [1, 2, 3])
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
@pytest.mark.parametrize("layout", ["grid", "list", "packed"])
def test_eval_stages_within_fp64_bounds(monkeypatch, layout, precision, layers, W, F):
    model, *args = _case(layers, W, F)
    S = W + F
    budget = (2 if layout == "packed" else 6) * S   # several tiles (chunks) on every layout, the last one partial
    runs = [("grid", "padded"), ("list", "padded")] if layout != "packed" else [("grid", "packed"), ("list", "packed")]
    if layout != "packed":
        runs = [r for r in runs if r[0] == layout]
    fp8 = precision == "fp8" and layers > 1
    for mode, lay in runs:
        calls, out, entries, arena = _record(monkeypatch, model, args, mode, lay, precision, budget)
        names = {c.name for c in calls}
        assert ("attention_varlen_fwd" in names) == (lay == "packed")
        assert ("gemm_fp8" in names) == fp8
        assert ("attention_pair_fwd" in names) == (lay == "padded")
        if S > ops.SHORT_ATTN_MAX_S and lay == "padded" and layers > 1:
            assert "univl_attention_long_fwd" in entries
        label = "%s %s %s L=%d W=%d F=%d" % (mode, lay, precision, layers, W, F)
        t, _ = _walk(model, arena, args, calls, out, mode, lay, fp8, budget, label=label)
        t.report()
        n_tiles = sum(c.name == "pooler_sim" for c in calls)
        assert n_tiles >= 2, n_tiles


def test_checker_rejects_wiring_errors(monkeypatch):
    """each perturbation of the reference, applied to real recorded calls, fails at the stage it perturbs"""
    W, F = 16, 12
    budget = 6 * (W + F)
    model, *args = _case(2, W, F, seed=3)
    for layout, precision, perturbs in (("padded", "fp8", ("video_pos", "video_type0", "res_next_video", "quant_prev",
                                                           "kv_as_qk", "scale_x2", "transpose_tiles")),
                                        ("packed", "bf16", ("drop_last_key", "res_next_video"))):
        calls, out, _, arena = _record(monkeypatch, model, args, "grid", layout, precision, budget)
        t, _ = _walk(model, arena, args, calls, out, "grid", layout, precision == "fp8", budget)   # unperturbed: ok
        for p in perturbs:
            # on the packed layout the residual rows are gathered: a wrong one fails at the gather
            stage = "layer0 gather" if (p, layout) == ("res_next_video", "packed") else ec.PERTURB[p]
            with pytest.raises(AssertionError, match=stage):
                _walk(model, arena, args, calls, out, "grid", layout, precision == "fp8", budget, perturb=(p,))
    calls, out, _, arena = _record(monkeypatch, model, args, "list", "padded", "bf16", budget)
    with pytest.raises(AssertionError, match="logits"):
        _walk(model, arena, args, calls, out, "list", "padded", False, budget, perturb=("transpose_tiles",))


def _scattered(N, S, seed):
    """rows whose valid tokens are not a prefix: Bernoulli(0.6), token 0 padded on odd rows, at least one valid"""
    g = _g(seed)
    m = (torch.rand(N, S, generator=g) < 0.6).long()
    m[1::2, 0] = 0
    m[:, -1] = 1
    m[0] = 1
    return m.to(DEV)


@pytest.mark.parametrize("which", ["texts", "videos"])
def test_gallery_encoder_layers_within_fp64_bounds(monkeypatch, which):
    cfg = synth.task_config(mode="ft_joint", batch_size=2, text_layers=2, visual_layers=2, cross_layers=1,
                            max_words=48, max_frames=40)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, seed=4)).eval()
    rec = ec.EvalRecorder().install(monkeypatch)
    N = 6
    with torch.no_grad(), rt.use_model(model, torch.device(DEV, torch.cuda.current_device())) as arena:
        if which == "texts":
            mask = _scattered(N, 48, 11)
            ids = torch.randint(1000, 3000, (N, 48), generator=_g(12)).to(DEV)
            out = retrieval.embed_texts(model, ids, mask)
            layers, lin = model.bert.encoder.layer, None
        else:
            mask = _scattered(N, 40, 13)
            video = torch.randn(N, 40, cfg.video_dim, generator=_g(14)).to(DEV)
            out = retrieval.embed_videos(model, video, mask)
            layers = model.visual.encoder.layer
            emb = model.visual.embeddings.word_embeddings
            lin = (emb.weight, emb.bias)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out).all())
        t, _ = ec.check_encoder(rec.calls, [_layer_params(layer) for layer in layers], arena, mask, lin,
                                label="embed_" + which)
    t.report()
    assert len(layers) == 2 and any("enc layer1 core" in k for k in t.worst)
