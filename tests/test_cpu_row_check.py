"""CPU: the fp64 references of tests/row_check.py against independent statements (F.layer_norm, F.normalize,
scipy.special.erfc, F.cross_entropy and the loss functions of oracle/univl_oracle.py), the GELU bound against a float32
emulation of common.cuh gelu_erf / gelu_erf_grad over every bf16 input, and each negative check's perturbation
outside its bound."""
import argparse
import math

import numpy as np
import torch
import torch.nn.functional as F
from scipy.special import erfc

from oracle import univl_oracle as O
from tests import row_check as rc

f32 = np.float32


def _outside(perturbed, ref, bound):
    return bool(((perturbed.double() - ref).abs() > bound).any())


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _gelu_terms(x):
    """common.cuh erf_exp_terms in float32: w = 1 - Phi(|x|) by Abramowitz & Stegun 7.1.26, and exp(-x^2 / 2)"""
    with np.errstate(over="ignore", invalid="ignore"):
        t = (f32(1) / _fma(np.abs(x), f32(0.3275911 * 0.70710678118654752440), f32(1))).astype(f32)
        gauss = np.exp2((x * x).astype(f32) * f32(-0.5 * 1.44269504088896340736)).astype(f32)
        poly = _fma(f32(0.5 * 1.061405429), t, f32(0.5 * -1.453152027))
        poly = _fma(poly, t, f32(0.5 * 1.421413741))
        poly = _fma(poly, t, f32(0.5 * -0.284496736))
        poly = _fma(poly, t, f32(0.5 * 0.254829592))
        return ((poly * t).astype(f32) * gauss).astype(f32), gauss


def _all_finite_bf16():
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    return x[torch.isfinite(x)]


def test_gelu_emulation_inside_bound_over_every_bf16_input():
    x = _all_finite_bf16()
    xn = x.numpy()
    w, gauss = _gelu_terms(xn)
    # the A&S 7.1.26 formula itself, in fp64: the 7.0e-8 of row_check's GELU comment
    xa = np.abs(xn.astype(np.float64))
    t = 1.0 / (1.0 + 0.3275911 * xa / math.sqrt(2.0))
    poly = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t
    w_formula = 0.5 * poly * np.exp(-0.5 * xa * xa)
    assert float(np.abs(w_formula - 0.5 * erfc(xa / math.sqrt(2.0))).max()) <= 7.0e-8
    with np.errstate(over="ignore", invalid="ignore"):
        gelu = _fma(-np.minimum(np.abs(xn), f32(1e30)), w, np.maximum(xn, f32(0)))
        grad = _fma((np.clip(xn, f32(-1e30), f32(1e30)) * f32(0.39894228040143267794)).astype(f32), gauss,
                    np.where(xn >= 0, (f32(1) - w).astype(f32), w))
    xd = x.double()
    ref = rc.gelu64(xd)
    assert torch.allclose(ref, xd * 0.5 * torch.from_numpy(erfc(-xd.numpy() / math.sqrt(2.0))), rtol=1e-12,
                          atol=1e-300)
    err = (torch.from_numpy(gelu).double() - ref).abs()
    assert bool((err <= rc.gelu_bound(xd)).all()), float((err / rc.gelu_bound(xd)).max())
    gerr = (torch.from_numpy(grad).double() - rc.gelu_grad64(xd)).abs()
    assert bool((gerr <= rc.gelu_grad_bound(xd)).all()), float((gerr / rc.gelu_grad_bound(xd)).max())
    # the tail the comment describes: relative error of the formula beyond 10% where gelu is about 1e-6
    tail = (xd <= -5.25) & (ref != 0)
    assert float((err[tail] / ref[tail].abs()).max()) > 0.1


def test_ln_reference_and_unbiased_variance_rejected():
    g = torch.Generator().manual_seed(0)
    for C in (256, 768, 1024):
        z = torch.randn(9, C, generator=g, dtype=torch.float64) * 2 + 0.5
        z[3] = 64 + 1e-2 * torch.randn(C, generator=g, dtype=torch.float64)
        z = z.float().double()                  # fp32 rows, as NormalizeVideo reads them: no input rounding
        gamma = 1 + 0.1 * torch.randn(C, generator=g)
        beta = 0.1 * torch.randn(C, generator=g)
        ref = rc.ln_fwd(z, gamma, beta)
        want = F.layer_norm(z, (C,), gamma.double(), beta.double(), eps=rc.EPS32)
        assert torch.allclose(ref["y"], want, rtol=1e-10, atol=1e-10)
        # the fp32 statement of the same row lands inside the bound
        z32 = z.float()
        m32 = z32.mean(1, keepdim=True)
        r32 = torch.rsqrt(((z32 - m32) ** 2).mean(1, keepdim=True) + rc.EPS32)
        assert bool(((r32[:, 0].double() - ref["rstd"]).abs() <= ref["b_rstd"]).all())
        bad = rc.ln_fwd(z, gamma, beta, unbiased=True)
        assert _outside(bad["rstd"], ref["rstd"], ref["b_rstd"])


def test_meanpool_reference_and_counted_first_position_rejected():
    g = torch.Generator().manual_seed(1)
    N, S, H = 6, 10, 768
    x = torch.randn(N * S, H, generator=g).to(torch.bfloat16)
    mask = (torch.arange(S)[None, :] < torch.tensor([10, 2, 5, 7, 3, 9])[:, None]).long()
    dy = torch.randn(N, H, generator=g)
    for skip_first, guard, l2 in ((True, False, True), (False, True, True), (True, False, False)):
        ref = rc.meanpool_ref(x, mask, N, S, skip_first, guard, l2, dy=dy)
        on = rc.meanpool_on(mask, skip_first).double()[:, :, None]
        u = (x.double().view(N, S, H) * on).sum(1) / on.sum(1)
        want = F.normalize(u, dim=-1) if l2 else u
        assert torch.allclose(ref["out"], want, rtol=1e-12, atol=1e-14)
        if skip_first and not l2:               # the L2 normalisation cancels the denominator
            bad = rc.meanpool_ref(x, mask, N, S, skip_first, guard, l2, count_first=True)
            assert _outside(bad["out"], ref["out"], ref["b_out"])


def _loss_cfg(B, P):
    return argparse.Namespace(margin=0.1, batch_size=B // P, n_gpu=1, n_pair=P, negative_weighting=1,
                              hard_negative_rate=0.5)


def test_loss_references_match_oracle_and_reject_perturbations():
    g = torch.Generator().manual_seed(2)
    for B, P in ((32, 1), (48, 3)):
        sim = torch.round(torch.randn(B, B, generator=g, dtype=torch.float64) * 256) / 64
        sim[:4] *= 7
        cfg = _loss_cfg(B, P)
        for fn, ref_fn in ((lambda s: rc.crossen_ref(s), O.cross_en_loss),
                           (lambda s: rc.milnce_ref(s, B // P, P), lambda s: O.mil_nce_loss(s, cfg))):
            loss, b_loss, dsim, b_dsim = fn(sim)
            s = sim.clone().requires_grad_()
            want = ref_fn(s)
            want.backward()
            assert abs(float(loss) - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
            assert torch.allclose(dsim, s.grad, rtol=1e-10, atol=1e-14)
        ws, wd = rc.maxmargin_weights(B // P, P, 0.5) if P > 1 else (1.0, 1.0)
        loss, b_loss, dsim, b_dsim, _ = rc.maxmargin_ref(sim, float(np.float32(0.1)), P if P > 1 else 0, ws, wd)
        cfg.margin = float(np.float32(0.1))
        s = sim.clone().requires_grad_()
        want = O.max_margin_loss(s, cfg)
        want.backward()
        assert abs(float(loss) - float(want)) <= 1e-6 * abs(float(want))
        assert torch.allclose(dsim, s.grad, rtol=1e-6, atol=1e-12)
        _, _, bad, _, _ = rc.maxmargin_ref(sim, 0.1, P if P > 1 else 0, ws, wd, drop_diag=B // 2)
        assert _outside(bad, dsim, b_dsim)
        if P == 3:
            loss, b_loss, _, _ = rc.milnce_ref(sim, B // P, P)
            bad, _, _, _ = rc.milnce_ref(sim, B // P, P, pick_offset=0)
            assert _outside(bad.view(1), loss.view(1), b_loss.view(1))


def test_xent_reference_matches_cross_entropy_and_rejects_a_dropped_row():
    g = torch.Generator().manual_seed(3)
    T, V, G = 60, 1000, 3
    logits = 3 * torch.randn(T, V, generator=g)
    labels = torch.randint(0, V, (T,), generator=g)
    labels[torch.rand(T, generator=g) < 0.3] = -1
    labels[0], labels[20], labels[40] = 0, V - 1, 5
    ref = rc.xent_ref(logits, labels, V, 0, G, gscale=0.5)
    R = T // G
    want = sum(F.cross_entropy(logits[k * R:(k + 1) * R].double(), labels[k * R:(k + 1) * R], ignore_index=-1)
               for k in range(G)) / G
    assert abs(float(ref["loss"]) - float(want)) <= 1e-12
    x = logits.double().requires_grad_()
    (0.5 * sum(F.cross_entropy(x[k * R:(k + 1) * R], labels[k * R:(k + 1) * R], ignore_index=-1)
               for k in range(G)) / G).backward()
    assert torch.allclose(ref["dl"], x.grad, rtol=1e-10, atol=1e-15)
    bad = rc.xent_ref(logits, labels, V, 0, G, gscale=0.5, drop_row=0)
    assert _outside(bad["loss"].view(1), ref["loss"].view(1), ref["b_loss"].view(1))


def test_cast_truncation_differs_from_round_to_nearest():
    # ties of both parities and values just above a tie: truncation keeps the low half, round-to-nearest-even does not
    x = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -20, -(1.0 + 2.0 ** -7 + 2.0 ** -9)])
    rn = x.to(torch.bfloat16).view(torch.int16)
    trunc = (x.view(torch.int32) >> 16).to(torch.int16)
    assert rn.tolist() != trunc.tolist()
    assert x.to(torch.bfloat16).float().tolist() == [1.0, 1.0 + 2.0 ** -6, 1.0 + 2.0 ** -7, -(1.0 + 2.0 ** -7)]
