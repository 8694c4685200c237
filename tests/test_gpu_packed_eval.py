"""GPU: packed cross-encoder evaluation (UNIVL_EVAL_LAYOUT=packed, UniVL._cross_similarity_eval_packed) against the
padded layout and the fp32 CPU oracle, its independence of the tiling, the attention_mask[:, 0] fallback, the paths
that never read the switch, and its memory next to the padded path's."""
import pytest
import torch

from oracle import synth
from oracle import univl_oracle as O
from tests.model_util import build_model
from univl_b200 import ops
from univl_b200 import runtime as rt
from univl_b200.modules import modeling

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768

# Packed vs padded.  Both layouts run every row through the same GEMM, LayerNorm and FFN kernels; a padded key adds
# exactly 0 to its row's softmax sums, so the two differ only in the order of the fp32 sums inside attention, and each
# attention context element may round to a neighbouring bf16 value (2^-8 relative).  That is the same kind of
# difference as between the fused and the unfused attention kernels, which tests/test_gpu_pair_scoring.py holds to 2e-2
# on the logits: bf16 packed vs padded is held to 2e-2.  Under FP8 a neighbouring context value can move an e4m3 code,
# whose unit is 2^-4 instead of 2^-8 (E4M3_OVER_BF16_UNIT in tests/test_gpu_fp8_eval.py): 16 x 2e-2.
PACKED_VS_PADDED = {"bf16": 2e-2, "fp8": 16 * 2e-2}
# the oracle bounds of tests/test_gpu_pair_scoring.py (bf16) and tests/test_gpu_fp8_eval.py (fp8: 16 x the bf16 error)
BF16_ORACLE_BOUND = 2e-2
E4M3_OVER_BF16_UNIT = 16


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _masks(Nt, W, Nv, F, seed):
    """text rows ragged prefixes (even rows) or scattered with token 0 kept (odd rows); video rows ragged prefixes,
    scattered, and the last one fully padded.  Text row 0 and video row 0 are full, so the longest packed pair has all
    W + F tokens (at (128, 160): 288 keys, the key-tiled kernel)"""
    g = _g(seed)
    lt = torch.randint(1, W + 1, (Nt,), generator=g)
    tm = (torch.arange(W)[None] < lt[:, None]).long()
    tm[1::2] = (torch.rand(tm[1::2].shape, generator=g) < 0.5).long()
    tm[:, 0] = 1
    lv = torch.randint(1, F + 1, (Nv,), generator=g)
    vm = (torch.arange(F)[None] < lv[:, None]).long()
    vm[1::2] = (torch.rand(vm[1::2].shape, generator=g) < 0.5).long()
    vm[-1] = 0
    tm[0] = 1
    vm[0] = 1
    return tm.to(DEV), vm.to(DEV)


def _case(cross_layers, W, F, Nt, Nv, seed=0):
    cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1, cross_layers=cross_layers,
                            max_words=W, max_frames=F)
    sd = synth.make_state_dict(cfg, seed=seed)
    model = build_model(cfg, sd=sd).eval()
    seq = (torch.randn((Nt, W, H), generator=_g(50 + seed))).to(torch.bfloat16).to(DEV)
    vis = (torch.randn((Nv, F, H), generator=_g(60 + seed))).to(torch.bfloat16).to(DEV)
    am, vm = _masks(Nt, W, Nv, F, 70 + seed)
    return cfg, sd, model, (seq, vis, am, vm)


class _Spy:
    """records the longest sequence of every ops.attention_varlen_fwd call: proof that the packed path ran"""

    def __init__(self, monkeypatch):
        self.max_sk = []
        real = ops.attention_varlen_fwd

        def spy(q, k, v, seqs, *a, **kw):
            self.max_sk.append(seqs.max_sk)
            return real(q, k, v, seqs, *a, **kw)
        monkeypatch.setattr(ops, "attention_varlen_fwd", spy)


def _logits(model, args, layout, monkeypatch, precision="bf16"):
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", layout)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", precision)
    with torch.no_grad():
        return model.get_similarity_logits(*args)


@pytest.mark.parametrize("W,F", [(16, 16), (48, 48), (128, 160)])
@pytest.mark.parametrize("cross_layers", [1, 2, 3])
def test_packed_equals_padded_and_the_oracle(W, F, cross_layers, monkeypatch):
    Nt, Nv = 5, 4
    cfg, sd, model, args = _case(cross_layers, W, F, Nt, Nv, seed=cross_layers)
    # 7 pairs of W + F tokens per tile: both layouts run several tiles, the last one partial
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 7 * (W + F))
    seq, vis, am, vm = args
    ref = O.similarity_logits(seq.float().cpu(), vis.float().cpu(), am.cpu(), vm.cpu(), sd, cfg)
    err = {}
    spy = _Spy(monkeypatch)
    for precision in ("bf16", "fp8"):
        padded = _logits(model, args, "padded", monkeypatch, precision)
        assert spy.max_sk == []
        packed = _logits(model, args, "packed", monkeypatch, precision)
        # the packed path ran, with the call's longest pair (the full text row 0 with the full video row 0)
        assert spy.max_sk and set(spy.max_sk) == {W + F}
        spy.max_sk.clear()
        assert packed.shape == (Nt, Nv) and bool(torch.isfinite(packed).all())
        diff = float((packed - padded).abs().max())
        err[precision] = (float((packed.cpu() - ref).abs().max()), float((padded.cpu() - ref).abs().max()))
        print("W=%d F=%d L=%d %s: max |packed - padded| %.3g, |packed - oracle| %.3g, |padded - oracle| %.3g"
              % (W, F, cross_layers, precision, diff, err[precision][0], err[precision][1]))
        assert diff <= PACKED_VS_PADDED[precision]
    assert max(err["bf16"]) <= BF16_ORACLE_BOUND
    if cross_layers > 1:
        assert err["fp8"][0] <= E4M3_OVER_BF16_UNIT * err["bf16"][0]
    else:  # one cross layer has no FP8 GEMM over pair tokens: the fp8 switch changes nothing
        assert err["fp8"] == err["bf16"]


@pytest.mark.parametrize("W,F,cross_layers", [(24, 20, 2), (128, 160, 3)])
@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_packed_result_does_not_depend_on_the_tiling_and_repeats(W, F, cross_layers, precision, monkeypatch):
    _, _, model, args = _case(cross_layers, W, F, 7, 5, seed=4)
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 1 << 30)
    one = _logits(model, args, "packed", monkeypatch, precision)
    for budget in (6 * (W + F), 2 * (W + F), 1):
        monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", budget)
        assert torch.equal(_logits(model, args, "packed", monkeypatch, precision), one), budget
    assert torch.equal(_logits(model, args, "packed", monkeypatch, precision), one)
    rt.reserve_sms(40)
    try:
        assert torch.equal(_logits(model, args, "packed", monkeypatch, precision), one)
    finally:
        rt.reserve_sms(0)


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_a_text_row_without_token_0_takes_the_padded_path(precision, monkeypatch):
    _, _, model, args = _case(2, 20, 13, 4, 3, seed=5)
    seq, vis, am, vm = args
    am = am.clone()
    am[2, 0] = 0
    args = (seq, vis, am, vm)
    padded = _logits(model, args, "padded", monkeypatch, precision)
    spy = _Spy(monkeypatch)
    assert torch.equal(_logits(model, args, "packed", monkeypatch, precision), padded)
    assert spy.max_sk == []  # the packed path did not run


def test_training_gradients_and_micro_batches_never_read_the_switch(monkeypatch):
    _, _, model, args = _case(2, 20, 13, 4, 4, seed=6)
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", "padded")
    with torch.enable_grad():
        grad_ref = model.get_similarity_logits(*args).detach()
    seq, vis, am, vm = (a.reshape(-1, a.shape[-1]) if a.dim() == 3 else a for a in args)
    with torch.no_grad(), rt.use_model(model, model._device()):
        micro_ref = model._cross_similarity(seq, vis, am, vm, groups=2)
    model.train()
    for m in model.modules():  # dropout off, so the training-mode result repeats
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    with torch.no_grad():
        train_ref = model.get_similarity_logits(*args)
    # an invalid value: any path that read the switch would raise
    monkeypatch.setenv("UNIVL_EVAL_LAYOUT", "bogus")
    with torch.no_grad():
        assert torch.equal(model.get_similarity_logits(*args), train_ref)
    model.eval()
    with torch.enable_grad():
        assert torch.equal(model.get_similarity_logits(*args).detach(), grad_ref)
    with torch.no_grad(), rt.use_model(model, model._device()):
        assert torch.equal(model._cross_similarity(seq, vis, am, vm, groups=2), micro_ref)
    with torch.no_grad(), pytest.raises(ValueError, match="UNIVL_EVAL_LAYOUT"):
        model.get_similarity_logits(*args)


def test_1024_by_1024_pairs_peak_no_higher_than_padded(monkeypatch):
    Nt = Nv = 1024
    W = F = 48
    _, _, model, args = _case(2, W, F, Nt, Nv, seed=7)
    peaks, out = {}, {}
    for layout in ("padded", "packed"):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out[layout] = _logits(model, args, layout, monkeypatch)
        torch.cuda.synchronize()
        peaks[layout] = torch.cuda.max_memory_allocated() - base
    print("1024 x 1024 pairs, W = F = 48, 2 cross layers: peak padded %.2f GiB, packed %.2f GiB"
          % (peaks["padded"] / 2 ** 30, peaks["packed"] / 2 ** 30))
    assert peaks["packed"] <= peaks["padded"]
    assert bool(torch.isfinite(out["packed"]).all())
    assert float((out["packed"] - out["padded"]).abs().max()) <= PACKED_VS_PADDED["bf16"]
