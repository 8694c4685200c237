"""GPU: the rest of the reference-facing surface — inference entry points (get_sequence_visual_output /
get_similarity_logits with Bt != Bv / decoder_caption), sub-model forwards, the flat-gradient fast path against the
autograd-returned gradients, the fused optimizer inside a real training step, CUDA-graph replay with fresh dropout."""
import pytest
import torch

from oracle import synth
from oracle import univl_oracle as O
from tests.model_util import build_model, grads_by_name, to_device

pytestmark = pytest.mark.gpu


def _small(mode, **kw):
    base = dict(mode=mode, batch_size=3, text_layers=2, visual_layers=1, cross_layers=1, decoder_layers=1,
                max_words=16, max_frames=12)
    base.update(kw)
    return synth.task_config(**base)


def test_eval_similarity_rectangular_and_mean_pool():
    """eval-time retrieval: all (text batch x video batch) pairs with Bt != Bv (main_task_retrieval.py:367-381)."""
    for mode in ("ft_joint", "ft_align"):
        cfg = _small(mode, batch_size=4)
        sd = synth.make_state_dict(cfg)
        model = build_model(cfg, sd=sd).eval()
        batch = synth.make_batch(cfg, seed=3)
        b = to_device(batch)
        with torch.no_grad():
            assert model(**b) is None  # eval-mode forward returns None like the reference (modeling.py:270-271)
            seq, vis = model.get_sequence_visual_output(b["input_ids"], b["token_type_ids"], b["attention_mask"],
                                                        b["video"], b["video_mask"])
            sim = model.get_similarity_logits(seq[:3], vis[1:], b["attention_mask"][:3], b["video_mask"][1:])
        assert sim.shape == (3, 3) and sim.dtype == torch.float32
        flat = lambda t: t.view(-1, t.shape[-1])  # noqa: E731
        vid = O.normalize_video(batch["video"], sd)
        s, v = O.sequence_visual_output(flat(batch["input_ids"]), flat(batch["token_type_ids"]),
                                        flat(batch["attention_mask"]), vid, flat(batch["video_mask"]), sd, cfg)
        ref = O.similarity_logits(s[:3], v[1:], flat(batch["attention_mask"])[:3], flat(batch["video_mask"])[1:], sd,
                                  cfg)
        assert (sim.cpu() - ref).abs().max() <= (2e-2 if mode == "ft_align" else 2e-3)


def test_decoder_caption_logits_and_argmax():
    cfg = _small("caption", batch_size=2)
    sd = synth.make_state_dict(cfg)
    model = build_model(cfg, sd=sd).eval()
    batch = synth.make_batch(cfg, seed=4)
    b = to_device(batch)
    with torch.no_grad():
        seq, vis = model.get_sequence_visual_output(b["input_ids"], b["token_type_ids"], b["attention_mask"],
                                                    b["video"], b["video_mask"])
        logits = model.decoder_caption(seq, vis, b["input_ids"], b["attention_mask"], b["video_mask"],
                                       b["input_caption_ids"], b["decoder_mask"], get_logits=True)
        ids = model.decoder_caption(seq, vis, b["input_ids"], b["attention_mask"], b["video_mask"],
                                    b["input_caption_ids"], b["decoder_mask"])
    _, parts = O.univl_forward(sd, cfg, batch, return_parts=True)
    ref = parts["decoder_logits"]
    assert logits.shape == ref.shape
    assert (logits.cpu() - ref).abs().max() <= 6e-2 * max(1.0, float(ref.abs().max()))
    assert torch.equal(ids.cpu(), logits.cpu().argmax(-1))
    # the argmax agrees with the reference wherever the reference's top-2 margin exceeds the bf16 noise
    top2 = ref.topk(2, -1).values
    confident = (top2[..., 0] - top2[..., 1]) > 0.25
    assert bool((ids.cpu()[confident] == ref.argmax(-1)[confident]).all())


def test_submodel_forward_surfaces():
    cfg = _small("ft_joint", batch_size=2)
    model = build_model(cfg).eval()
    batch = to_device(synth.make_batch(cfg, seed=5))
    ids = batch["input_ids"].view(-1, 16)
    with torch.no_grad():
        layers, pooled = model.bert(ids, torch.zeros_like(ids), batch["attention_mask"].view(-1, 16))
        last, _ = model.bert(ids, output_all_encoded_layers=False)
        video = model.normalize_video(batch["video"])
        vlayers, vpooled = model.visual(video, batch["video_mask"].view(-1, 12))
    assert len(layers) == 2 and layers[-1].shape == (2, 16, 768) and pooled.shape == (2, 768)
    assert last.shape == (2, 16, 768)
    assert len(vlayers) == 1 and vlayers[0].shape == (2, 12, 768) and vpooled.shape == (2, 768)
    assert float(pooled.float().abs().max()) <= 1.0  # tanh


def _flat_sink_case(mode):
    from univl_b200.optim import flatten
    cfg = _small(mode, batch_size=3)
    sd = synth.make_state_dict(cfg)
    batch = synth.make_batch(cfg, seed=6)
    ref_model = build_model(cfg, sd=sd)
    ref_model(**to_device(batch)).backward()
    ref = grads_by_name(ref_model)
    # a parameter used by several layers (tied weights) gets one gradient per use: autograd adds them in its own
    # order, the flat sink in kernel launch order, so with three or more uses the last bits may differ
    uses = {}
    for name, p in ref_model.named_parameters(remove_duplicate=False):
        uses.setdefault(id(p), []).append(name)
    tied = {names[0] for names in uses.values() if len(names) > 1}
    model = build_model(cfg, sd=sd)
    flat = flatten(model, sink_grads=True)
    for _ in range(2):  # second pass checks zero_grad + re-accumulation
        flat.zero_grad()
        model(**to_device(batch)).backward()
    torch.cuda.synchronize()
    got = grads_by_name(model)
    assert set(got) >= set(ref)
    for k, r in ref.items():
        g = got[k]
        if k in tied:
            assert (g - r).abs().max() <= 1e-5 * float(r.abs().max()) + 1e-12, k
        else:
            assert torch.equal(g, r), k
    # state_dict is unchanged by flattening (parameters are views now)
    for k, v in sd.items():
        assert torch.equal(model.state_dict()[k].cpu(), v), k


def test_flat_gradient_sinks_match_autograd_gradients():
    """backward kernels accumulating straight into the flat gradient buffer (fast path) give the same gradients as
    the autograd-returned ones (the path the reference's DistributedDataParallel wrap uses): the same bits, since every
    kernel adds its sums in a fixed order into a zeroed buffer either way (pretraining stage two: every head)."""
    _flat_sink_case("pretrain2")


def test_flat_gradient_sinks_match_autograd_gradients_ft_align():
    """the same on the retrieval fine-tuning path, which has no tied weights: every gradient bit for bit"""
    _flat_sink_case("ft_align")


def test_training_steps_with_fused_optimizer_reduce_the_loss():
    from univl_b200.modules.optimization import BertAdam
    cfg = _small("ft_align", batch_size=4)
    model = build_model(cfg, sd=synth.make_state_dict(cfg, init_law=True), dropout=0.0)  # deterministic descent
    batch = to_device(synth.make_batch(cfg, seed=7))
    named = list(model.named_parameters())
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    opt = BertAdam(groups, lr=1e-4, warmup=0.1, t_total=60, max_grad_norm=1.0, model=model)
    losses = []
    for _ in range(16):
        opt.zero_grad()
        loss = model(**batch)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(l == l for l in losses)
    assert losses[-1] < losses[0] - 1e-3 and min(losses) == min(losses[-4:]), losses
    assert opt.get_lr()[0] > 0


def test_cuda_graph_replay_draws_fresh_dropout_masks():
    cfg = _small("ft_joint", batch_size=4)
    model = build_model(cfg, dropout=0.3)
    batch = to_device(synth.make_batch(cfg, seed=8))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            model(**batch).backward()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for p in model.parameters():
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = model(**batch)
    vals = []
    for _ in range(4):
        graph.replay()
        vals.append(float(loss))
    assert len(set(vals)) == 4, vals  # same launch arguments, different device-side RNG epoch each replay


def test_device_side_masking_feeds_pretrain_stage_two():
    """univl_b200.masking samples the MLM / MFM masks on the device (dataloader_howto100m.py:103-125, :314-329 restated):
    the model accepts the result in place of the dataloader's four tensors, and with the SAME masks moved to the CPU the
    oracle agrees on the loss."""
    from univl_b200 import masking
    from tests.oracle_util import run_oracle
    cfg = synth.task_config(mode="pretrain2", batch_size=4, max_words=16, max_frames=12, text_layers=2, visual_layers=1,
                            cross_layers=1, decoder_layers=1)
    sd = synth.make_state_dict(cfg, seed=5)
    batch = synth.make_batch(cfg, seed=6)
    for k in ("pairs_masked_text", "pairs_token_labels", "masked_video", "video_labels_index"):
        batch.pop(k)
    dev_batch = to_device(batch)
    gen = torch.Generator(device="cuda").manual_seed(3)
    full = masking.mask_pretrain_batch(dev_batch, p=0.3, generator=gen)   # p raised so the tiny batch surely has picks
    assert all(v.is_cuda for v in full.values())
    assert int((full["pairs_token_labels"] != -1).sum()) > 0 and int((full["video_labels_index"] != -1).sum()) > 0
    model = build_model(cfg, sd=sd)
    loss = model(**full)
    loss.backward()
    got = float(loss.detach())
    o_loss, parts, _ = run_oracle(cfg, {k: v.cpu() for k, v in full.items()}, sd=sd, backward=False)
    # pretrain stage-two tolerance of test_gpu_model_parity.py, with 65 bounding the joint-similarity logits of these weights
    tol = 2e-3 * abs(float(o_loss)) + 2.0 ** -7 * (65.0 + float(parts["mfm_loss"]))
    assert abs(got - float(o_loss)) <= tol, (got, float(o_loss), tol)
