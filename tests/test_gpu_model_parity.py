"""GPU: the CUDA path (through the reference-facing UniVL class, down the C ABI) against
 (a) the golden outputs of the unmodified reference (tests/golden/, made by oracle/make_golden.py) and
 (b) the CPU oracle on the same seeded inputs — loss, hidden states and every gradient tensor.

Stated tolerances (bf16 activations, fp32 accumulation / statistics / losses; the reference is fp32):
  loss   retrieval loss with the reference's own random-init law (BASELINE.json configs[0]; *_init cases):
                                                                  |d| <= 1e-3                  (north_star)
         retrieval loss on the stress weights (2x init std, random LayerNorm gains/biases): |d| <= 4e-3
         cross-entropy losses over the vocabulary / frames (caption, pretrain-II):            |d| <= 2e-3 * |loss|
         MIL-NCE on UN-normalised dot products (use_mil): |d| <= 2^-8 * max|sim| — the logits are only resolved to
         bf16 precision relative to their magnitude (~25 here)
         pretrain stage-two (five objectives summed): 2e-3 * |loss| for the three vocabulary / similarity cross-entropies
         + 2^-7 * (max|joint sim| + MFM-NCE loss value) for the two NCE terms whose logits are UN-normalised dot products of
         two bf16-rounded vectors (each operand carries 2^-9 relative error, 2^-8 on the product; the NCE loss inherits the
         absolute error of its largest logits, and a loss of L nats means logits of magnitude >= L).  With the stress
         weights these logits reach 40-65; with the reference's init law the same case agrees to 1e-2.
  similarity matrix   mean-pool (cosine) similarity: |d| <= 2^-7.  Cross-encoder similarity (FT-Align: similarity_dense of
         the pooled cross output): |d| <= 2^-5 * max(1, max|sim|) — a 768-term dot product of hidden values that carry
         the stack's ~1e-2 relative error with a weight vector of norm 0.55 (init law) / 1.1 (stress weights).
  hidden states   relative Frobenius error <= 2 * sqrt(7 * (layers + 1)) * 2^-9 / sqrt(3).  Derivation: every layer
                  stores 7 bf16 tensors on the path to its output (qkv, context, attention-out, LN1-out, FFN
                  pre-activation / activation, FFN-out, LN2-out; +1 "layer" for the embedding / input projection); a
                  round-to-nearest bf16 store has relative error uniform in [-2^-9, 2^-9], RMS 2^-9 / sqrt(3); the
                  roundings are independent, so the expected relative Frobenius error of an L-layer stack is
                  sqrt(7 (L + 1)) * 2^-9 / sqrt(3)  (2 layers 5.2e-3, 6 layers 7.9e-3, 12 layers 1.08e-2); the bound is
                  twice that.  Measured / expected is 1.1-1.2 (LayerNorm gains of the stress weights); the achieved
                  margins are written to the file UNIVL_PARITY_MARGINS names.  Worst single element:
                  0.1 absolute on values of magnitude 2-4 (~6 bf16 ulps).
  gradients       per tensor ||g - g_oracle|| <= 0.10 * max(||g_oracle||, 0.05 * largest gradient norm) and, for tensors
                  above that floor, norm within 6 %.  The floor exists because some gradients are mathematically (key
                  biases: softmax shift invariance) or numerically (q/k weights of deep layers once attention has
                  become uniform: 1e-4 of the value-weight gradients) zero; there only the absolute error is
                  meaningful in bf16.  A tensor that misses these bounds is still accepted if its error is within 2.5x of
                  the error the CPU oracle itself makes when its activations / activation-gradients are rounded to
                  bf16 (oracle.univl_oracle.emulate_bf16) — the conditioning of the gradient, not the kernels.
"""
import pytest
import torch

from oracle import synth
from tests.model_util import build_model, grads_by_name, to_device
from tests.oracle_util import load_golden, run_oracle

pytestmark = pytest.mark.gpu

import json
import os

CASES = ["ft_joint_npair2", "pretrain1_mil", "caption_small", "pretrain2_small", "cfg1_ft_joint", "cfg1_ft_align",
         "cfg1_ft_joint_init", "cfg1_ft_align_init",
         # BASELINE.json configs[3], [4], [1] at their real sequence lengths and full 12/6/2/3 depth
         "cfg4_caption", "cfg5_pretrain2", "cfg5_pretrain2_npair3_init", "cfg2_ft_align_b32_init"]
GOLDEN_ONLY = {"cfg2_ft_align_b32_init"}   # 1024 pair sequences: checked against the reference's stored outputs only

_MARGINS = {}


def _record(name, **kw):
    """achieved margins, written to the JSON file UNIVL_PARITY_MARGINS names (if set)"""
    _MARGINS.setdefault(name, {}).update(kw)
    out = os.environ.get("UNIVL_PARITY_MARGINS")
    if not out:
        return
    try:
        with open(out, "w") as fh:
            json.dump(_MARGINS, fh, indent=1, sort_keys=True)
    except OSError:
        pass


def loss_tolerance(cfg, gold, parts=None):
    init_law = bool(gold.get("weight_kwargs", {}).get("init_law"))
    if cfg.mode in ("ft_joint", "ft_align"):
        return 1e-3 if (init_law or cfg.mode == "ft_joint") else 4e-3
    if cfg.use_mil and not getattr(cfg, "stage_two", False):
        return 2.0 ** -8 * max(float(s.abs().max()) for s in gold["sim_matrices"])
    tol = 2e-3 * abs(gold["loss"])
    if cfg.mode == "pretrain2" and parts is not None:
        tol += 2.0 ** -7 * (float(gold["sim_matrices"][0].abs().max()) + float(parts["mfm_loss"]))
    return tol


@pytest.mark.parametrize("name", CASES)
def test_loss_hidden_and_grads_match_reference(name):
    gold = load_golden(name)
    cfg = synth.task_config(**gold["cfg_kwargs"])
    wkw = gold.get("weight_kwargs", {})
    sd = synth.make_state_dict(cfg, seed=gold["weight_seed"], **wkw)
    batch = synth.make_batch(cfg, **gold["batch_kwargs"])
    model = build_model(cfg, sd=sd)
    loss = model(**to_device(batch))
    loss.backward()
    torch.cuda.synchronize()
    got = float(loss.detach())
    o_loss = parts = o_grads = None
    if name not in GOLDEN_ONLY:
        o_loss, parts, o_grads = run_oracle(cfg, batch, sd=sd, backward=True)
    tol = loss_tolerance(cfg, gold, parts)
    _record(name, loss=got, ref_loss=gold["loss"], loss_err=abs(got - gold["loss"]), loss_tol=tol)
    assert abs(got - gold["loss"]) <= tol, "loss %r vs reference %r (tol %g)" % (got, gold["loss"], tol)
    grads = grads_by_name(model)
    assert set(grads) == set(gold["grad_norms"]), sorted(set(grads) ^ set(gold["grad_norms"]))[:8]
    biggest = max(gold["grad_norms"].values())
    floor = 0.05 * biggest

    model.eval()
    with torch.no_grad():
        b = to_device(batch)
        seq, vis = model.get_sequence_visual_output(b["input_ids"], b["token_type_ids"], b["attention_mask"],
                                                    b["video"], b["video_mask"])
        if gold["sim_matrices"] and cfg.mode in ("ft_joint", "ft_align"):
            sim = model.get_similarity_logits(seq, vis, b["attention_mask"], b["video_mask"]).float().cpu()
            ref_sim = gold["sim_matrices"][-1]
            sim_err = float((sim - ref_sim).abs().max())
            _record(name, sim_max_err=sim_err, sim_scale=float(ref_sim.abs().max()))
            sim_tol = 2.0 ** -7 if cfg.mode == "ft_joint" else 2.0 ** -5 * max(1.0, float(ref_sim.abs().max()))
            assert sim_err <= sim_tol, (sim_err, sim_tol)
    seq, vis = seq.float().cpu(), vis.float().cpu()
    assert (seq[:, :6, :16] - gold["seq_slice"]).abs().max() <= 1e-1
    assert (vis[:, :6, :16] - gold["vis_slice"]).abs().max() <= 1e-1
    # Frobenius norm of the reference's hidden states from the stored sum of squares
    for tag, ours, summ in (("seq", seq, gold["seq_summary"]), ("vis", vis, gold["vis_summary"])):
        rel = abs(float(ours.double().norm()) - summ["sq_sum"] ** 0.5) / summ["sq_sum"] ** 0.5
        _record(name, **{tag + "_norm_rel_err": rel})
        assert rel <= 2.0 ** -9 * 4, (tag, rel)

    if name in GOLDEN_ONLY:
        worst = 0.0
        for k, ref_norm in gold["grad_norms"].items():
            if ref_norm < floor:
                continue
            ratio = float(grads[k].double().norm()) / ref_norm
            worst = max(worst, abs(ratio - 1.0))
        _record(name, grad_norm_worst_rel=worst)
        assert worst <= 0.06, worst
        return

    assert abs(got - float(o_loss)) <= tol
    # hidden states after an L-layer bf16 stack against the fp32 reference algorithm: derived bound on the relative
    # Frobenius error (see the module docstring); worst single element ~6 bf16 ulps of |x| = 2..4.
    for tag, ours, ref, layers in (("seq", seq, parts["sequence_output"].detach(), cfg.text_num_hidden_layers),
                                   ("vis", vis, parts["visual_output"].detach(), cfg.visual_num_hidden_layers)):
        rel = float((ours - ref).norm() / ref.norm())
        bound = 2.0 * (7.0 * (layers + 1)) ** 0.5 * 2.0 ** -9 / 3.0 ** 0.5
        _record(name, **{tag + "_rel_fro": rel, tag + "_bound": bound, tag + "_max_abs": float((ours - ref).abs().max())})
        assert rel <= bound, (tag, rel, bound)
        assert float((ours - ref).abs().max()) <= 1e-1

    bad = []
    emu = None
    worst_err, worst_ratio, n_emu = 0.0, 0.0, 0
    for k, ref_norm in gold["grad_norms"].items():
        g, r = grads[k].double(), o_grads[k].double()
        abs_err = float((g - r).norm())
        err = abs_err / max(float(r.norm()), floor)
        ratio = float(g.norm()) / max(ref_norm, 1e-30)
        if err <= 0.10 and (ref_norm < floor or 0.94 <= ratio <= 1.06):
            worst_err = max(worst_err, err)
            if ref_norm >= floor:
                worst_ratio = max(worst_ratio, abs(ratio - 1.0))
            continue
        # ill-conditioned gradient (e.g. the all-pairs hinge loss at random init: d loss / d sim sums to zero while
        # every pair back-propagates nearly the same vector).  Budget: what rounding the reference algorithm's own
        # activations and activation-gradients to bf16 does (oracle bf16 emulation), with a 2.5x allowance.
        if emu is None:
            _, _, emu = run_oracle(cfg, batch, sd=sd, backward=True, bf16_emulation=True)
        emu_err = float((emu[k].double() - r).norm())
        n_emu += 1
        if abs_err > 2.5 * emu_err:
            bad.append((k, round(err, 4), round(ratio, 4), "bf16-emulated oracle error %.3e vs ours %.3e" % (
                emu_err, abs_err)))
    _record(name, grad_worst_rel_err=worst_err, grad_worst_norm_dev=worst_ratio, grads_judged_by_bf16_emulation=n_emu,
            grads_total=len(gold["grad_norms"]))
    assert not bad, "gradient mismatches (name, relative error, norm ratio): %s" % bad[:12]
