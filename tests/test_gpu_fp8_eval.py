"""GPU: FP8 cross-encoder evaluation (UNIVL_EVAL_PRECISION=fp8): the e4m3 quantizers, the block-scaled FP8 GEMM and
the model's FP8 eval path (CrossModel.encode_pairs_first_token_eval_fp8).

Bottom up: the quantizers are bit-exact against a torch statement of the scaling rule (csrc/fp8.cuh); the GEMM is
checked element by element against fp64 on its dequantized operands, under a written bound, by a checker that is shown
to reject a dropped K block and a wrong block scale; the eval logits do not depend on the tiling or the row order; the
switch leaves every other path bit for bit as it is."""
import pytest
import torch

from oracle import synth
from oracle import univl_oracle as O
from tests.fp8_check import ACC, bf16_out_ok, deq_blocks, deq_rows, gelu_e4m3_bound, ref_codes, ref_scale  # noqa: F401
from tests.model_util import build_model, to_device
from univl_b200 import ops
from univl_b200.modules import modeling

pytestmark = pytest.mark.gpu

DEV = "cuda"
H = 768
E4M3 = torch.float8_e4m3fn


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=_g(seed)) * scale


def _activations(M, K, seed):
    """bf16 rows whose 128-column blocks span many magnitudes, with the edge cases of the scaling rule"""
    x = _randn((M, K), seed)
    mag = torch.pow(10.0, torch.empty(M, K // 128).uniform_(-6, 4, generator=_g(seed + 1)))
    x = x * mag.repeat_interleave(128, dim=1)
    x[0, :128] = 0.0                                           # an all-zero block
    if K >= 256:
        x[0, 128:256] = torch.linspace(-460.0, 460.0, 128)     # values around 448: scale 2, codes near the top
    if M > 1 and K >= 256:
        x[1, 128:256] = _randn((128,), seed + 2, 2.0 ** -8)    # small values next to a large one: e4m3 subnormals
        x[1, 128] = 300.0
        x[1, :128] = torch.full((128,), 448.0)                 # amax exactly 448: scale 1
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("M,K", [(1, 128), (37, 768), (300, 3072), (1000, 768)])
def test_quantize_rows_is_bit_exact(M, K):
    x = _activations(M, K, M + K)
    q, s = ops.quantize_e4m3_rows(x.to(DEV))
    assert q.shape == (M, K) and q.dtype == E4M3 and s.shape == (K // 128, M)
    xf = x.float().view(M, K // 128, 128)
    es = ref_scale(xf.abs().amax(-1))
    eq = ref_codes(xf, es[..., None]).view(M, K)
    assert torch.equal(s.cpu(), es.t().contiguous())
    assert torch.equal(q.cpu().view(torch.uint8), eq.view(torch.uint8))
    # the edge cases are there: the zero block codes to 0 with scale 1, the blocks around 448 get scales 2 and 1, and
    # subnormal codes occur
    assert s[0, 0].item() == 1.0 and int(q[0, :128].view(torch.uint8).max()) == 0
    if M > 1 and K >= 256:
        assert s[1, 0].item() == 2.0 and s[0, 1].item() == 1.0 and s[1, 1].item() == 1.0
        codes = q[1, 129:256].view(torch.uint8)
        assert bool((((codes & 0x78) == 0) & ((codes & 0x07) != 0)).any())  # exponent field 0: subnormal e4m3


def test_quantize_rows_reads_a_strided_view():
    x = _activations(64, 1024, 5).to(DEV)
    q, s = ops.quantize_e4m3_rows(x[:, 128:896])
    q2, s2 = ops.quantize_e4m3_rows(x[:, 128:896].contiguous())
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s, s2)


@pytest.mark.parametrize("N,K", [(128, 128), (768, 768), (3072, 768), (768, 3072)])
def test_quantize_blocks_is_bit_exact(N, K):
    w = _randn((N, K), N + K, 0.03)
    mag = torch.pow(10.0, torch.empty(N // 128, K // 128).uniform_(-4, 2, generator=_g(7)))
    w = w * mag.repeat_interleave(128, 0).repeat_interleave(128, 1)
    w[:128, :128] = 0.0
    q, s = ops.quantize_e4m3_blocks(w.to(DEV))
    blocks = w.view(N // 128, 128, K // 128, 128)
    es = ref_scale(blocks.abs().amax(dim=(1, 3)))
    eq = ref_codes(blocks, es[:, None, :, None]).view(N, K)
    assert torch.equal(s.cpu(), es)
    assert torch.equal(q.cpu().view(torch.uint8), eq.view(torch.uint8))
    assert s[0, 0].item() == 1.0


# ---------------------------------------------------------------------------------------------------------
# FP8 GEMM against fp64 on the dequantized operands, under tests/fp8_check.py's bound (ACC)
def _gemm_case(M, N, K, seed):
    x = _randn((M, K), seed) * torch.pow(10.0, torch.empty(M, 1).uniform_(-2, 2, generator=_g(seed + 1)))
    a, sa = ops.quantize_e4m3_rows(x.to(torch.bfloat16).to(DEV))
    b, sb = ops.quantize_e4m3_blocks(_randn((N, K), seed + 2, 0.03).to(DEV))
    bias = _randn((N,), seed + 3, 0.1).to(DEV)
    A, B = deq_rows(a, sa), deq_blocks(b, sb)
    ref = A @ B.t() + bias.double()
    absref = A.abs() @ B.abs().t() + bias.double().abs()
    return a, sa, b, sb, bias, A, B, ref, absref


@pytest.mark.parametrize("N", [768, 1536, 3072])
@pytest.mark.parametrize("K", [768, 3072])
@pytest.mark.parametrize("M", [1, 300])
def test_gemm_fp8_bias_bf16_within_the_bound(M, N, K):
    a, sa, b, sb, bias, A, B, ref, absref = _gemm_case(M, N, K, M + N + K)
    out = ops.gemm_fp8(a, sa, b, sb, bias)
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    ok, worst = bf16_out_ok(out, ref, absref)
    print("M=%d N=%d K=%d: max |err| / sum|a b| = %.3g (bf16 output rounding included)" % (M, N, K, worst))
    assert ok, worst
    assert torch.equal(ops.gemm_fp8(a, sa, b, sb, bias), out)  # deterministic
    # a row does not depend on the other rows of the launch
    if M > 130:
        sub = ops.gemm_fp8(a[130:M].contiguous(), sa[:, 130:M].contiguous(), b, sb, bias)
        assert torch.equal(sub, out[130:M])


@pytest.mark.parametrize("K", [128, 384, 640, 256])
def test_gemm_fp8_odd_and_short_k(K):
    """an odd number of K blocks takes the one-temporary mainloop, an even one the alternating pair"""
    M, N = 300, 768
    a, sa, b, sb, bias, A, B, ref, absref = _gemm_case(M, N, K, K)
    ok, worst = bf16_out_ok(ops.gemm_fp8(a, sa, b, sb, bias), ref, absref)
    assert ok, worst
    h, hs = ops.gemm_fp8(a, sa, b, sb, bias, gelu=True)
    g = torch.nn.functional.gelu(ref)
    assert bool(((deq_rows(h, hs) - g).abs() <= gelu_e4m3_bound(g, absref, hs)).all())


def test_gemm_fp8_many_waves_and_the_checker_rejects_wrong_results():
    M, N, K = 4000, 3072, 768
    a, sa, b, sb, bias, A, B, ref, absref = _gemm_case(M, N, K, 11)
    out = ops.gemm_fp8(a, sa, b, sb, bias)
    ok, worst = bf16_out_ok(out, ref, absref)
    print("M=%d N=%d K=%d: max |err| / sum|a b| = %.3g" % (M, N, K, worst))
    assert ok, worst
    # one K block dropped
    dropped = (ref - A[:, 256:384] @ B[:, 256:384].t()).to(torch.bfloat16)
    assert not bf16_out_ok(dropped, ref, absref)[0]
    # one wrong block scale (a weight block's scale doubled)
    B2 = B.clone()
    B2[128:256, 384:512] *= 2
    wrong = (A @ B2.t() + bias.double()).to(torch.bfloat16)
    assert not bf16_out_ok(wrong, ref, absref)[0]


@pytest.mark.parametrize("M,K", [(300, 768), (1, 768), (700, 3072)])
def test_gemm_fp8_gelu_e4m3_epilogue(M, K):
    N = 3072 if K == 768 else 768
    a, sa, b, sb, bias, A, B, ref, absref = _gemm_case(M, N, K, M + K + 1)
    h, hs = ops.gemm_fp8(a, sa, b, sb, bias, gelu=True)
    assert h.shape == (M, N) and h.dtype == E4M3 and hs.shape == (N // 128, M)
    g = torch.nn.functional.gelu(ref)
    deq = deq_rows(h, hs)
    bound = gelu_e4m3_bound(g, absref, hs)
    err = (deq - g).abs()
    print("gelu e4m3 M=%d K=%d: max |err| / bound = %.3g" % (M, K, float((err / bound).max())))
    assert bool((err <= bound).all())
    # every scale is a power of two and puts its block's largest code in e4m3's top binade
    bits = hs.view(torch.int32)
    assert bool(((bits & 0x7FFFFF) == 0).all())
    top = h.float().abs().view(M, N // 128, 128).amax(-1)
    assert bool(((top >= 224) & (top <= 448)).all())


# ---------------------------------------------------------------------------------------------------------
# model
def _model_case(kind, cross_layers, W, F, Nt, Nv, seed=0):
    if kind == "stage_two":
        cfg = synth.task_config(mode="caption", task_type="retrieval", batch_size=2, text_layers=1, visual_layers=1,
                                cross_layers=cross_layers, decoder_layers=1, max_words=W, max_frames=F)
    else:
        cfg = synth.task_config(mode="ft_align", batch_size=2, text_layers=1, visual_layers=1,
                                cross_layers=cross_layers, max_words=W, max_frames=F)
    sd = synth.make_state_dict(cfg, seed=seed)
    model = build_model(cfg, sd=sd).eval()
    seq = _randn((Nt, W, H), 50 + seed).to(torch.bfloat16).to(DEV)
    vis = _randn((Nv, F, H), 60 + seed).to(torch.bfloat16).to(DEV)
    am = _lengths_mask(Nt, W, 70 + seed)
    vm = _lengths_mask(Nv, F, 80 + seed, empty_rows=(Nv - 1,))
    return cfg, sd, model, (seq, vis, am, vm)


def _lengths_mask(N, L, seed, empty_rows=()):
    lens = torch.randint(1, L + 1, (N,), generator=_g(seed))
    m = (torch.arange(L).view(1, L) < lens.view(N, 1)).long()
    for r in empty_rows:
        m[r] = 0
    return m.to(DEV)


def _eval_logits(model, args):
    with torch.no_grad():
        return model.get_similarity_logits(*args)


@pytest.fixture
def fp8(monkeypatch):
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "fp8")


# Model-level bound.  The bf16 eval path's logits are within 2e-2 of the fp32 oracle (tests/test_gpu_pair_scoring.py;
# measured 0.008-0.009 on these cases).  The FP8 path computes the same thing and differs only in the operands of the
# GEMMs it runs in FP8, rounded with e4m3's unit 2^-4 instead of bf16's 2^-8.  Rounding errors of that kind propagate
# linearly to the logit, so the FP8 path's error against the oracle is bounded by 16 times the bf16 path's error on the
# same inputs: 0.13-0.15 here, where a fixed bound of 16 x 2e-2 would allow 0.32.  Measured: 0.06-0.11, 6-14 times.
BF16_ORACLE_BOUND = 2e-2
E4M3_OVER_BF16_UNIT = 16


@pytest.mark.parametrize("kind,cross_layers,W,F", [("ft_align", 2, 48, 48), ("stage_two", 2, 20, 13),
                                                   ("ft_align", 3, 16, 12)])
def test_fp8_eval_logits_match_the_oracle(kind, cross_layers, W, F, monkeypatch):
    cfg, sd, model, args = _model_case(kind, cross_layers, W, F, 3, 4, seed=1)
    seq, vis, am, vm = args
    ref = O.similarity_logits(seq.float().cpu(), vis.float().cpu(), am.cpu(), vm.cpu(), sd, cfg)
    bf16 = _eval_logits(model, args)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "fp8")
    got = _eval_logits(model, args)
    e8 = float((got.cpu() - ref).abs().max())
    e16 = float((bf16.cpu() - ref).abs().max())
    print("%s L=%d W=%d F=%d: max |logit - oracle| fp8 %.4g, bf16 %.4g (logit std %.4g)"
          % (kind, cross_layers, W, F, e8, e16, float(ref.std())))
    assert not torch.equal(got, bf16)  # the FP8 path ran
    assert e16 <= BF16_ORACLE_BOUND
    assert e8 <= E4M3_OVER_BF16_UNIT * e16


def test_one_cross_layer_fp8_changes_nothing(monkeypatch):
    _, _, model, args = _model_case("ft_align", 1, 16, 12, 5, 4)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "fp8")
    got = _eval_logits(model, args)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "bf16")
    assert torch.equal(got, _eval_logits(model, args))


def test_fp8_logits_do_not_depend_on_tiling_or_row_order(fp8, monkeypatch):
    _, _, model, args = _model_case("ft_align", 2, 20, 13, 7, 5)
    seq, vis, am, vm = args
    S = 20 + 13
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 1 << 30)
    one = _eval_logits(model, args)
    assert bool(torch.isfinite(one).all())  # video 4 is fully padded
    for budget in (6 * S, 2 * S, S):
        monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", budget)
        assert torch.equal(_eval_logits(model, args), one), budget
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 4 * S)
    pt = torch.randperm(7, generator=_g(3)).to(DEV)
    pv = torch.randperm(5, generator=_g(4)).to(DEV)
    perm = _eval_logits(model, (seq[pt], vis[pv], am[pt], vm[pv]))
    assert torch.equal(perm, one[pt][:, pv])


def test_bf16_switch_is_the_existing_path(monkeypatch):
    monkeypatch.setenv("UNIVL_FUSED_ATTN", "0")
    _, _, model, args = _model_case("ft_align", 2, 24, 20, 5, 4)
    monkeypatch.delenv("UNIVL_EVAL_PRECISION", raising=False)
    unset = _eval_logits(model, args)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "bf16")
    assert torch.equal(_eval_logits(model, args), unset)
    with torch.enable_grad():  # the all-pairs path, which tests/test_gpu_pair_scoring.py pins the eval path to
        assert torch.equal(model.get_similarity_logits(*args).detach(), unset)
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "FP8")
    with pytest.raises(ValueError, match="UNIVL_EVAL_PRECISION"):
        _eval_logits(model, args)


def _train_step(model, batch):
    model.train()
    model.zero_grad(set_to_none=True)
    loss = model(**batch)
    loss.backward()
    return loss.detach().clone(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


def test_training_and_grad_enabled_calls_ignore_the_switch(monkeypatch):
    cfg = synth.task_config(mode="ft_align", batch_size=4, text_layers=1, visual_layers=1, cross_layers=2,
                            max_words=16, max_frames=12)
    model = build_model(cfg)
    batch = to_device(synth.make_batch(cfg, seed=5))
    monkeypatch.delenv("UNIVL_EVAL_PRECISION", raising=False)
    loss0, grads0 = _train_step(model, batch)
    model.eval()
    _, _, _, args = _model_case("ft_align", 2, 16, 12, 3, 4)
    with torch.enable_grad():
        sim0 = model.get_similarity_logits(*args).detach()
    monkeypatch.setenv("UNIVL_EVAL_PRECISION", "fp8")
    loss1, grads1 = _train_step(model, batch)
    assert torch.equal(loss0, loss1)
    assert grads0.keys() == grads1.keys() and all(torch.equal(grads0[n], grads1[n]) for n in grads0)
    model.eval()
    with torch.enable_grad():
        assert torch.equal(model.get_similarity_logits(*args).detach(), sim0)


def test_fp8_weights_are_requantized_after_an_in_place_edit(fp8):
    cfg, sd, model, args = _model_case("ft_align", 2, 16, 12, 3, 4)
    before = _eval_logits(model, args)

    def edit(m):
        with torch.no_grad():
            for name, p in m.named_parameters():
                if name.startswith("cross.encoder") and p.dim() == 2:
                    p.mul_(1.5)

    edit(model)
    after = _eval_logits(model, args)
    fresh = build_model(cfg, sd=sd).eval()
    edit(fresh)
    assert not torch.equal(after, before)
    assert torch.equal(after, _eval_logits(fresh, args))
