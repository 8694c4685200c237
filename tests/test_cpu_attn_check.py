"""CPU: the attention checker itself (tests/attn_check.py).  The host Philox reproduces Random123's published
known-answer vectors; a CPU emulation of the kernels' arithmetic (fp32 scores and softmax, bf16 P, fp32 P V, bf16
outputs, and the matching backward) passes every bound; and the perturbations the GPU tests reject fail here too."""
import numpy as np
import pytest
import torch

from tests import attn_check as ac

H = ac.HEADS * ac.HD


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in ac.philox4x32(ctr, key)) == want


def test_dropout_layouts_words_and_threshold():
    """counter / word layout of each generator against a direct Philox call, the threshold, the 64-bit stream"""
    seed, stream = (5 << 33) + 17, (3 << 32) + 9
    r = ac.philox4x32((7, 0, stream & ac.M32, stream >> 32), (seed & ac.M32, seed >> 32))
    table = ac.philox_u16(seed, stream, 8)
    assert [int(table[7, w]) for w in range(8)] == [int(r[w >> 1]) >> (16 * (w & 1)) & 0xFFFF for w in range(8)]
    assert ac.threshold16(0.1) == 58982 and ac.threshold16(0.25) == 49152 and ac.threshold16(0.0) == 65536
    assert ac.kernel_stream(2 ** 32 - 5, 3) == 2 ** 32 - 5 + (3 << 20)
    # tile layout: element (bh=1, i=9, j=18) of Sq = 20, Sk = 40 (nQb = 2, nKb = 3) is call ((1*2 + 0)*3 + 1)*32 +
    # (1 << 2 | 2 >> 1) = 229, word 0 | 1 << 1 | 0 = 2
    keep = ac.keep_tile(seed, stream, 0.5, 2, 20, 40)
    assert bool(keep[1, 9, 18]) == (int(ac.philox_u16(seed, stream, 230)[229, 2]) < ac.threshold16(0.5))
    # row-major layout: (bh=1, i=3, j=13) of S = 16 is call (1*16 + 3)*2 + 1 = 39, word 5
    keep = ac.keep_rowmajor(seed, stream, 0.5, 2, 16)
    assert bool(keep[1, 3, 13]) == (int(ac.philox_u16(seed, stream, 40)[39, 5]) < ac.threshold16(0.5))
    keep = ac.keep_elem(seed, stream, 0.5, 3, 20)
    assert bool(keep[2, 7]) == (int(ac.philox_u16(seed, stream, 6)[47 >> 3, 47 & 7]) < ac.threshold16(0.5))


# ---------------------------------------------------------------------------------------------------------
# a CPU emulation of the kernels' arithmetic
# ---------------------------------------------------------------------------------------------------------
def _bf(t):
    return t.to(torch.bfloat16)


def emulate(q, k, v, n_seq, Sq, Sk, key_real, causal, keep, p, d_o):
    """fp32 scores, fp32 softmax, bf16 P, fp32 P V, bf16 o; backward: P from the lse, dP, D from the bf16 o, bf16 dS /
    P_drop, fp32 products, bf16 gradients -> o, lse, dq, dk, dv"""
    def heads(t, S):
        return t.float().reshape(n_seq, S, ac.HEADS, ac.HD).permute(0, 2, 1, 3)
    qh, kh, vh, dOh = heads(q, Sq), heads(k, Sk), heads(v, Sk), heads(d_o, Sq)
    a = ac.additive_mask(key_real, Sq, causal).float()[:, None]
    c = 1.0 / (1.0 - p) if keep is not None else 1.0
    M = keep.view(n_seq, ac.HEADS, Sq, Sk) if keep is not None else torch.ones(1, dtype=torch.bool)
    s = (qh @ kh.transpose(-1, -2)) * ac.SCALE + a
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    P = e * (1.0 / l)
    Pd = _bf(torch.where(M, P * c, 0.0)).float()
    O = _bf(Pd @ vh)
    lse = m + torch.log(l)
    Pb = torch.exp(s - lse)
    dP = dOh @ vh.transpose(-1, -2)
    g = torch.where(M, dP * c, 0.0)
    D = (dOh * O.float()).sum(-1, keepdim=True)
    dS = _bf(Pb * (g - D) * ac.SCALE).float()
    Pk = _bf(torch.where(M, Pb * c, 0.0)).float()
    dQ = _bf(dS @ kh)
    dK = _bf(dS.transpose(-1, -2) @ qh)
    dV = _bf(Pk.transpose(-1, -2) @ dOh)
    return (ac._unheads(O), lse.reshape(-1), ac._unheads(dQ), ac._unheads(dK), ac._unheads(dV))


def _case(n_seq, Sq, Sk, causal, p, qscale, seed=0):
    g = torch.Generator().manual_seed(seed + Sq + Sk)
    q = _bf(torch.randn(n_seq * Sq, H, generator=g) * qscale)
    k = _bf(torch.randn(n_seq * Sk, H, generator=g))
    v = _bf(torch.randn(n_seq * Sk, H, generator=g))
    d_o = _bf(torch.randn(n_seq * Sq, H, generator=g))
    key_real = ac.edge_masks(n_seq, Sk, seed)
    keep = ac.keep_tile(123 + (1 << 40), 77, p, n_seq * ac.HEADS, Sq, Sk) if p > 0 else None
    return q, k, v, d_o, key_real, keep


CASES = [(5, 33, 33, True, 0.1, 1.0), (3, 1, 17, False, 0.0, 1.0), (2, 20, 52, False, 0.25, 4.0),
         (5, 17, 17, True, 0.0, 4.0)]


@pytest.mark.parametrize("n_seq,Sq,Sk,causal,p,qscale", CASES)
def test_emulated_kernel_arithmetic_is_within_the_bounds(n_seq, Sq, Sk, causal, p, qscale):
    q, k, v, d_o, key_real, keep = _case(n_seq, Sq, Sk, causal, p, qscale)
    o, lse, dq, dk, dv = emulate(q, k, v, n_seq, Sq, Sk, key_real, causal, keep, p, d_o)
    ref = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, causal, keep, p, d_o=d_o, o_kernel=o)
    ratios = ac.check_fwd(o, lse, ref, "emulated") + ac.check_bwd(dq, dk, dv, ref, "emulated")
    assert max(ratios) < 1.0


def test_emulated_perturbations_are_rejected():
    """each perturbation of part 2 of the GPU suite (tests/test_gpu_attention_fp64.py) fails on the emulation too"""
    n_seq, Sq, Sk, p = 3, 33, 33, 0.25
    q, k, v, d_o, key_real, keep = _case(n_seq, Sq, Sk, False, p, 1.0, seed=3)
    key_real[:] = 1
    o, lse, dq, dk, dv = emulate(q, k, v, n_seq, Sq, Sk, key_real, False, keep, p, d_o)

    def rejects(got, ref, bound):
        with pytest.raises(AssertionError):
            ac.within(got, ref, bound, "perturbed")

    ref = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, False, keep, p, d_o=d_o, o_kernel=o, want_p=True)
    ac.check_fwd(o, lse, ref, "unperturbed")
    # one key of the last partial block dropped from the reference
    kr = key_real.clone()
    kr[:, Sk - 1] = 0
    r = ac.reference(q, k, v, n_seq, Sq, Sk, kr, False, keep, p)
    rejects(o, r["o"], r["b_o"])
    # the mask shifted by one key
    r = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, False, keep.roll(1, -1), p)
    rejects(o, r["o"], r["b_o"])
    # one dropout element flipped: the kept element of largest probability
    flip = keep.clone()
    idx = np.unravel_index(int((ref["p"].reshape(flip.shape) * flip).argmax()), tuple(flip.shape))
    flip[idx] = False
    r = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, False, flip, p)
    rejects(o, r["o"], r["b_o"])
    # one row's lse shifted by three times its bound
    bad = lse.clone().double()
    bad[5] += 3 * ref["b_lse"][5]
    rejects(bad, ref["lse"], ref["b_lse"])
    # dK missing the last query row of every sequence
    d0 = d_o.clone().view(n_seq, Sq, H)
    d0[:, -1] = 0
    r = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, False, keep, p, d_o=d0.view(-1, H), o_kernel=o)
    rejects(dk, r["dk"], r["b_dk"])
    # the other dropout layout (row-major instead of tile), at a length both layouts take
    S = 32
    q, k, v, d_o, key_real, keep = _case(2, S, S, False, p, 1.0, seed=4)
    o = emulate(q, k, v, 2, S, S, key_real, False, keep, p, d_o)[0]
    ac.check_fwd(o, emulate(q, k, v, 2, S, S, key_real, False, keep, p, d_o)[1],
                 ac.reference(q, k, v, 2, S, S, key_real, False, keep, p), "unperturbed")
    r = ac.reference(q, k, v, 2, S, S, key_real, False, ac.keep_rowmajor(123 + (1 << 40), 77, p, 2 * ac.HEADS, S), p)
    rejects(o, r["o"], r["b_o"])
