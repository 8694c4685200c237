"""GPU: cross-encoder similarity in evaluation, scored in tiles with the first cross layer's Q/K/V projections computed
once per text row and once per video row (UniVL._cross_similarity_eval, csrc/attention_pair.cu).

Everything that makes the eval path exact is pinned here, bottom up: the GEMM gives a row the same bits whatever other
rows and tile width it runs with; the per-source embedding rows are the all-pairs embedding's rows; the pair attention
entry equals the existing attention entries on the materialised per-pair q/k/v.  On top of that the model's eval logits
equal the training-path logits bit for bit on the same (non-fused) kernels, whatever the tiling."""
import math
import os
import sys

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
H, HEADS = 768, 12


def _g(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=_g(seed)) * scale).to(DEV)


def _lengths_mask(N, L, seed, min_len=1, empty_rows=()):
    lens = torch.randint(min_len, L + 1, (N,), generator=_g(seed))
    m = (torch.arange(L).view(1, L) < lens.view(N, 1)).long()
    for r in empty_rows:
        m[r] = 0
    return m.to(DEV)


# ---------------------------------------------------------------------------------------------------------
# the GEMM assumption everything below relies on
def test_bias_gemm_rows_do_not_depend_on_the_other_rows_or_the_tile_width():
    """A row of a bias-epilogue GEMM has the same bits whether computed among M rows or among a subset of them, at any
    tile width and for any subset of the output columns (the separate Q and K/V projections of the last layer)."""
    M, K, N = 3000, H, 3 * H
    x = _randn((M, K), 1).to(torch.bfloat16)
    w = _randn((N, K), 2, 0.03).to(torch.bfloat16)
    b = _randn((N,), 3, 0.1).float()
    full = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(x, w, M, N, K, full, bias=b, block_n=256)
    for r0, r1 in [(37, 337), (0, 128), (2999, 3000), (1000, 2900)]:
        for bn in (0, 64, 128):
            part = torch.empty(r1 - r0, N, dtype=torch.bfloat16, device=DEV)
            ops.gemm(x[r0:r1], w, r1 - r0, N, K, part, bias=b, block_n=bn)
            assert torch.equal(part, full[r0:r1]), (r0, r1, bn)
        for c0, c1 in [(0, H), (H, 3 * H)]:
            part = torch.empty(r1 - r0, c1 - c0, dtype=torch.bfloat16, device=DEV)
            ops.gemm(x[r0:r1], w[c0:c1], r1 - r0, c1 - c0, K, part, bias=b[c0:c1].contiguous())
            assert torch.equal(part, full[r0:r1, c0:c1]), (r0, r1, c0, c1)


# ---------------------------------------------------------------------------------------------------------
# kernel
def _pair_call(qkv_a, qkv_b, Na, Nb, Sq, mask):
    """univl_attention_pair_fwd with its lse"""
    n_seq = Na * Nb
    o = torch.empty(n_seq * Sq, H, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(n_seq * HEADS * Sq, dtype=torch.float32, device=DEV)
    a, b = qkv_a, qkv_b
    rt.call("univl_attention_pair_fwd", a.data_ptr(), a.stride(0), a[:, H:].data_ptr(), a.stride(0),
            a[:, 2 * H:].data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), b[:, H:].data_ptr(), b.stride(0),
            b[:, 2 * H:].data_ptr(), b.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr(), rt.ptr(mask.a),
            rt.ptr(mask.b), Na, mask.Wa, Nb, mask.Fb, HEADS, Sq, 0.125)
    return o, lse


def _materialised(qkv_a, qkv_b, Na, Wa, Nb, Fb):
    """[Na*Nb*(Wa+Fb), 3H]: the per-pair sequences concat(a_i, b_j), p = i*Nb + j, gathered with torch"""
    i = torch.arange(Na, device=DEV).repeat_interleave(Nb)
    j = torch.arange(Nb, device=DEV).repeat(Na)
    seq = torch.cat([qkv_a.view(Na, Wa, -1)[i], qkv_b.view(Nb, Fb, -1)[j]], dim=1)
    return seq.reshape(Na * Nb * (Wa + Fb), -1).contiguous()


@pytest.mark.parametrize("Na,Wa,Nb,Fb", [(3, 48, 4, 48), (2, 128, 3, 96), (2, 128, 3, 160), (2, 512, 2, 512),
                                         (3, 20, 5, 13)])
@pytest.mark.parametrize("first_token", [False, True])
def test_pair_attention_equals_attention_on_materialised_pairs(Na, Wa, Nb, Fb, first_token):
    S = Wa + Fb
    Sq = 1 if first_token else S
    qkv_a = _randn((Na * Wa, 3 * H), 10 + Wa, 0.5).to(torch.bfloat16)
    qkv_b = _randn((Nb * Fb, 3 * H), 20 + Fb, 0.5).to(torch.bfloat16)
    mask = ops.MaskSpec(_lengths_mask(Na, Wa, 30), _lengths_mask(Nb, Fb, 31, empty_rows=(1,)), all_pairs=1)
    o, lse = _pair_call(qkv_a, qkv_b, Na, Nb, Sq, mask)
    o2, lse2 = _pair_call(qkv_a, qkv_b, Na, Nb, Sq, mask)
    assert torch.equal(o, o2) and torch.equal(lse, lse2)
    seq = _materialised(qkv_a, qkv_b, Na, Wa, Nb, Fb)
    q = seq.view(Na * Nb, S, -1)[:, 0].contiguous() if first_token else seq
    ref_o, ref_lse = ops.attention_fwd(q[:, :H], seq[:, H:2 * H], seq[:, 2 * H:], Na * Nb, Sq, S, mask)
    assert torch.equal(o, ref_o)
    assert torch.equal(lse, ref_lse)
    # video 1 is fully padded: its pairs keep the softmax of their raw scores, finite as in the reference
    assert bool(torch.isfinite(o.float()).all())
    # the eval wrapper gives the same context
    assert torch.equal(ops.attention_pair_fwd(qkv_a, qkv_b, Na, Nb, Sq, mask), o)


def test_source_embedding_rows_equal_the_all_pairs_embedding_rows():
    Nt, W, Nv, F = 3, 20, 4, 13
    t = _randn((Nt * W, H), 40).to(torch.bfloat16)
    v = _randn((Nv * F, H), 41).to(torch.bfloat16)
    pos = _randn((1024, H), 42, 0.1).float()
    typ = _randn((2, H), 43, 0.1).float()
    gamma = _randn((H,), 44, 0.2).float() + 1.0
    beta = _randn((H,), 45, 0.1).float()
    n_seq, S = Nt * Nv, W + F
    y = torch.empty(n_seq * S, H, dtype=torch.bfloat16, device=DEV)
    mean = torch.empty(n_seq * S, dtype=torch.float32, device=DEV)
    rstd = torch.empty_like(mean)
    rt.call("univl_embed_src_fwd", t.data_ptr(), v.data_ptr(), pos.data_ptr(), typ.data_ptr(), gamma.data_ptr(),
            beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), Nt, W, Nv, F, 1, H, ops.LN_EPS, 0.0, None,
            0)
    ts = ops.embed_src_rows_eval(t, Nt, W, pos, typ, gamma, beta, torch.empty_like(t))
    vs = ops.embed_src_rows_eval(v, Nv, F, pos[W:], typ[1:], gamma, beta, torch.empty_like(v))
    pairs = y.view(Nt, Nv, S, H)
    for i in range(Nt):
        for j in range(Nv):
            assert torch.equal(pairs[i, j, :W], ts.view(Nt, W, H)[i])
            assert torch.equal(pairs[i, j, W:], vs.view(Nv, F, H)[j])


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
    seq = _randn((Nt, W, H), 50 + seed).to(torch.bfloat16)
    vis = _randn((Nv, F, H), 60 + seed).to(torch.bfloat16)
    am = _lengths_mask(Nt, W, 70 + seed)
    vm = _lengths_mask(Nv, F, 80 + seed, empty_rows=(Nv - 1,))
    return cfg, sd, model, (seq, vis, am, vm)


def _eval_logits(model, args):
    with torch.no_grad():
        return model.get_similarity_logits(*args)


def _old_path_logits(model, args):
    """the existing all-pairs path: _cross_similarity in eval mode with gradients enabled"""
    with torch.enable_grad():
        return model.get_similarity_logits(*args).detach()


CASES = [("ft_align", 1, 16, 12), ("ft_align", 2, 48, 48), ("stage_two", 2, 20, 13), ("ft_align", 2, 160, 128),
         ("stage_two", 1, 128, 160)]


@pytest.mark.parametrize("kind,cross_layers,W,F", CASES)
def test_eval_logits_equal_the_old_path_bit_for_bit_without_the_fused_layer(kind, cross_layers, W, F, monkeypatch):
    monkeypatch.setenv("UNIVL_FUSED_ATTN", "0")
    _, _, model, args = _model_case(kind, cross_layers, W, F, 5, 4)
    got = _eval_logits(model, args)
    assert got.shape == (5, 4) and got.dtype == torch.float32
    assert torch.equal(got, _old_path_logits(model, args))


@pytest.mark.parametrize("kind,cross_layers,W,F", CASES)
def test_eval_logits_match_the_old_fused_path_and_the_oracle(kind, cross_layers, W, F):
    cfg, sd, model, args = _model_case(kind, cross_layers, W, F, 3, 4, seed=1)
    got = _eval_logits(model, args)
    old = _old_path_logits(model, args)
    seq, vis, am, vm = args
    ref = O.similarity_logits(seq.float().cpu(), vis.float().cpu(), am.cpu(), vm.cpu(), sd, cfg)
    # the bound of tests/test_gpu_api.py::test_eval_similarity_rectangular_and_mean_pool for cross similarity
    assert (got - old).abs().max() <= 2e-2
    assert (got.cpu() - ref).abs().max() <= 2e-2


# ---------------------------------------------------------------------------------------------------------
# tiling
def test_tiled_result_equals_the_one_tile_result_and_repeats(monkeypatch):
    _, _, model, args = _model_case("ft_align", 2, 24, 20, 7, 5)
    S = 24 + 20
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 1 << 30)
    one = _eval_logits(model, args)
    monkeypatch.setattr(modeling, "EVAL_PAIR_TOKENS", 6 * S)
    assert modeling._eval_tile(7, 5, S, 6 * S) == (3, 2)  # ragged tiles in both directions: 3 + 3 + 1 by 2 + 2 + 1
    tiled = _eval_logits(model, args)
    assert torch.equal(tiled, one)
    assert torch.equal(_eval_logits(model, args), one)
    rt.reserve_sms(40)
    try:
        assert torch.equal(_eval_logits(model, args), one)
    finally:
        rt.reserve_sms(0)


def test_scale_1024_by_1024_pairs_in_bounded_memory():
    """1024 x 1024 pairs at W = F = 48 with two cross layers (about 1.35 PFLOP): 1.9 TB of pair activations for the
    old path, a few GiB here"""
    Nt = Nv = 1024
    W = F = 48
    _, _, model, args = _model_case("ft_align", 2, W, F, Nt, Nv, seed=2)
    seq, vis, am, vm = args
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    got = _eval_logits(model, args)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert got.shape == (Nt, Nv) and bool(torch.isfinite(got).all())
    # a tile's peak (modeling.EVAL_PAIR_TOKENS) plus what grows with the inputs: the per-source embedding rows and their
    # Q/K/V projections, and the result
    per_source = (Nt * W + Nv * F) * (H + 3 * H) * 2
    assert peak <= (8 << 30) + per_source + Nt * Nv * 4, peak
    g = _g(90)
    for _ in range(8):
        rows_t = torch.randperm(Nt, generator=g)[:16].sort().values.to(DEV)
        rows_v = torch.randperm(Nv, generator=g)[:16].sort().values.to(DEV)
        sub = _eval_logits(model, (seq[rows_t], vis[rows_v], am[rows_t], vm[rows_v]))
        assert torch.equal(sub, got[rows_t][:, rows_v])


# ---------------------------------------------------------------------------------------------------------
# the reference's own evaluation driver at its default eval batch
class _Clips(torch.utils.data.Dataset):
    """items shaped like Youcook_DataLoader.__getitem__ (dataloaders/dataloader_youcook_retrieval.py:188-189)"""

    def __init__(self, cfg, n):
        b = synth.make_batch(cfg, seed=78, b=n)
        self.t = [b["input_ids"], b["attention_mask"], b["token_type_ids"], b["video"].double(), b["video_mask"],
                  b["input_ids"], torch.full_like(b["input_ids"], -1), b["video"].double(),
                  torch.full_like(b["video_mask"], -1)]

    def __len__(self):
        return self.t[0].shape[0]

    def __getitem__(self, i):
        return tuple(t[i] for t in self.t)


def test_reference_eval_epoch_at_batch_size_val_3500(tmp_path):
    import argparse

    from oracle import build_ref
    from tests.model_util import bert_dir
    root = build_ref.ref_root()
    if root is None:
        pytest.skip("reference checkout not staged (oracle/build_ref.py)")
    from univl_b200 import launcher
    os.environ["MASTER_PORT"] = str(29800 + (os.getpid() % 100))
    launcher.prepare(os.path.join(root, "main_task_retrieval.py"))
    import importlib
    drv = importlib.import_module("main_task_retrieval")
    import util
    drv.logger = util.get_logger(str(tmp_path / "log.txt"))
    args = argparse.Namespace(
        do_pretrain=False, do_train=False, do_eval=True, task_type="retrieval", datatype="youcook", stage_two=False,
        train_sim_after_cross=True, batch_size=4, batch_size_val=3500, n_gpu=1, n_pair=1, margin=0.1,
        negative_weighting=1, hard_negative_rate=0.5, use_mil=False, sampled_use_mil=False, video_dim=1024,
        max_words=16, max_frames=12, local_rank=0, world_size=1, text_num_hidden_layers=2,
        visual_num_hidden_layers=1, cross_num_hidden_layers=2, decoder_num_hidden_layers=1, init_model=None,
        bert_model=bert_dir(), visual_model="visual-base", cross_model="cross-base", decoder_model="decoder-base",
        cache_dir=str(tmp_path), lr=1e-3, coef_lr=0.1, warmup_proportion=0.1, gradient_accumulation_steps=1,
        n_display=1, epochs=1, output_dir=str(tmp_path), seed=42, fp16=False)
    device = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = drv.init_model(args, device, 1, 0)
    cfg = synth.task_config(mode="ft_align", batch_size=4, text_layers=2, visual_layers=1, cross_layers=2,
                            max_words=16, max_frames=12)
    # compute_metrics gets a LIST of row blocks with n_gpu == 1 (main_task_retrieval.py:443-445), the reference's own
    # single-GPU bug (see tests/test_gpu_dropin.py): give it the concatenated matrix
    import numpy as np
    import metrics
    seen = []

    def _metrics(sm):
        sm = np.concatenate(tuple(sm), axis=0) if isinstance(sm, list) else sm
        seen.append(sm.shape)
        return metrics.compute_metrics(sm)

    drv.compute_metrics = _metrics
    loader = torch.utils.data.DataLoader(_Clips(cfg, 512), batch_size=args.batch_size_val)
    r1 = drv.eval_epoch(args, model, loader, device, 1)
    assert seen == [(512, 512)]
    assert 0.0 <= float(r1) <= 1.0 and not math.isnan(float(r1))
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
    sys.modules.pop("main_task_retrieval", None)
