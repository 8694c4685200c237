"""fp64 reference, exact dropout masks and per-element bounds of the attention cores (csrc/attention.cu,
attention_long.cu, fused_attn.cu and the pair entry attention_pair.cu), shared by the attention tests.

The dropout masks are a deterministic function of (seed, stream, element): a host Philox4x32-10 reproduces each
kernel's counter layout, so with the mask known, dropout attention is a fixed function that fp64 checks element by
element like the plain op.  Every output element has its own bound, derived from the kernels' arithmetic (constants
below, in the style of tests/gemm_check.py); `within` prints each check's worst err / bound as "ratio"."""
import numpy as np
import torch

from tests.gemm_check import BF16_ROUND, C_ACC, U, within

HD = 64            # head dim of every kernel
HEADS = 12
SCALE = 0.125      # 1 / sqrt(64), exact
MASK_ADD = -10000.0

# __expf(x) = ex2.approx(x * log2 e): ex2.approx errs by 2 ulp (4U relative), and the rounding of x * log2 e moves the
# result by 1.173 |x| ulp (CUDA C Programming Guide, intrinsic functions): EXP_REL + EXP_ARG * U * |x| relative.
# fused_attn.cu calls ex2.approx on log2-domain arguments directly, inside the same bound.
EXP_REL = 8 * U
EXP_ARG = 3.0
# __logf / __log2f: 2^-21.41 absolute on [0.5, 2], 3 ulp elsewhere; the log of a row sum (<= 1024) is below 7, so
# 2^-19 absolute covers both
LOG_ABS = 2.0 ** -19
# score s = scale * acc + a in fp32: the 64-term wgmma / mma.sync accumulation (C_ACC, tests/gemm_check.py), then up
# to three fp32 roundings of |scale * acc| + |a| (the scale multiply, the mask add, and in fused_attn.cu the log2 e
# factors of the scale and the mask constant).  At the -10000 mask the add alone rounds by ~5e-4 absolute: it is real.
SCORE_ROUNDS = 3


# ---------------------------------------------------------------------------------------------------------
# Philox4x32-10 (Random123) and the kernels' dropout layouts
# ---------------------------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF
PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def philox4x32(ctr, key):
    """Philox4x32-10: ctr = 4 uint32 words (ints or uint64 arrays, broadcast), key = 2 uint32 ints -> the 4 output
    words as uint64 arrays.  A 32 x 32-bit product fits uint64 exactly, so hi / lo are exact."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & np.uint64(M32) for c in ctr)
    k0, k1 = int(key[0]) & M32, int(key[1]) & M32
    lo = np.uint64(M32)
    for _ in range(10):
        p0 = PHILOX_M[0] * c0
        p1 = PHILOX_M[1] * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & lo,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & lo)
        k0, k1 = (k0 + PHILOX_W[0]) & M32, (k1 + PHILOX_W[1]) & M32
    return c0, c1, c2, c3


def philox_u16(seed, stream, n_calls):
    """the 16-bit words of common.cuh philox4x32(seed, stream, c) for the counters c < n_calls -> uint32 [n_calls, 8];
    key (seed lo, seed hi), counter (c lo, c hi, stream lo, stream hi); word w = half (w & 1), low first, of output
    component w >> 1 (common.cuh philox_u16)"""
    c = np.arange(n_calls, dtype=np.uint64)
    r = philox4x32((c & np.uint64(M32), c >> np.uint64(32), stream & M32, stream >> 32), (seed & M32, seed >> 32))
    out = np.empty((n_calls, 8), dtype=np.uint32)
    for comp in range(4):
        out[:, 2 * comp] = (r[comp] & np.uint64(0xFFFF)).astype(np.uint32)
        out[:, 2 * comp + 1] = (r[comp] >> np.uint64(16)).astype(np.uint32)
    return out


def threshold16(p):
    """common.cuh dropout_threshold16: keep iff the 16-bit word < round((1 - p) * 65536), p as the kernels' float"""
    keep = 1.0 - float(np.float32(p))
    return 65536 if keep >= 1.0 else int(keep * 65536.0 + 0.5)


def kernel_stream(stream_id, epoch):
    """the Philox stream a kernel draws from: stream_id + (epoch << 20) mod 2^64 (epoch = rng_state[1])"""
    return (int(stream_id) + (int(epoch) << 20)) & (2 ** 64 - 1)


def _keep(seed, stream, p, n_bh, per_bh, local, word):
    """keep[bh, ...] = word `word` of call bh * per_bh + local < threshold16(p) -> bool torch tensor (CPU)"""
    table = philox_u16(seed, stream, n_bh * per_bh).reshape(n_bh, per_bh, 8)
    return torch.from_numpy(table[:, local, word] < threshold16(p))


def keep_tile(seed, stream, p, n_bh, Sq, Sk):
    """attention.cu / attention_long.cu (tile_rng, rng_layout 0): element (bh, i, j), bh = seq * heads + h, uses counter
    ((bh nQb + i/16) nKb + j/16) 32 + ((i & 7) << 2 | (j & 7) >> 1) and word (j & 1) | ((i >> 3) & 1) << 1 |
    ((j >> 3) & 1) << 2, nQb = ceil(Sq / 16), nKb = ceil(Sk / 16) -> bool [n_bh, Sq, Sk]"""
    nQb, nKb = -(-Sq // 16), -(-Sk // 16)
    i = np.arange(Sq)[:, None]
    j = np.arange(Sk)[None, :]
    local = ((i >> 4) * nKb + (j >> 4)) * 32 + (((i & 7) << 2) | ((j & 7) >> 1))
    word = (j & 1) | (((i >> 3) & 1) << 1) | (((j >> 3) & 1) << 2)
    return _keep(seed, stream, p, n_bh, nQb * nKb * 32, local, word)


def keep_rowmajor(seed, stream, p, n_bh, S):
    """fused_attn.cu (fa_keep_bits) and univl_attention_bwd rng_layout 1: element (bh, i, j) is word j & 7 of counter
    (bh S + i) (S / 8) + j / 8 -> bool [n_bh, S, S]"""
    i = np.arange(S)[:, None]
    j = np.arange(S)[None, :]
    return _keep(seed, stream, p, n_bh, S * (S // 8), i * (S // 8) + (j >> 3), j & 7)


def keep_elem(seed, stream, p, rows, cols):
    """dropout_keep8 (LayerNorm, embeddings): element idx = row * cols + col is word idx & 7 of counter idx >> 3
    -> bool [rows, cols]"""
    idx = np.arange(rows * cols)
    return _keep(seed, stream, p, 1, -(-rows * cols // 8), idx >> 3, idx & 7)[0].view(rows, cols)


# ---------------------------------------------------------------------------------------------------------
# masks
# ---------------------------------------------------------------------------------------------------------
def pair_masks(mask_a, mask_b, n_seq, groups):
    """the per-sequence key mask [n_seq, Wa + Fb] of (mask_a, mask_b) under common.cuh pair_sources: groups 0 =
    aligned, G >= 1 = G groups of Gt x Gv pairs"""
    if mask_b is None:
        return mask_a
    Nb = mask_b.shape[0]
    p = torch.arange(n_seq)
    if groups == 0:
        i = j = p
    else:
        Gv = Nb // groups
        g = p // (n_seq // groups) if groups > 1 else torch.zeros_like(p)
        r = p - g * (n_seq // groups)
        i = g * (n_seq // Nb) + r // Gv
        j = g * Gv + r % Gv
    return torch.cat([mask_a[i.to(mask_a.device)], mask_b[j.to(mask_b.device)]], 1)


def edge_masks(n_seq, Sk, seed, kinds=(0, 1, 2, 3, 4)):
    """int64 [n_seq, Sk] key masks that the model's prefix masks never produce, one kind per sequence in turn (cycling
    through `kinds`): 0 a scattered Bernoulli(0.7) mask with key 0 padded; 1 only the last key real (in the last,
    partial 16-key block when Sk % 16 != 0); 2 every key padded; 3 the first half padded (so a causal row before it
    attends to its future keys at -10000); 4 a random prefix"""
    g = torch.Generator().manual_seed(seed)
    m = torch.zeros(n_seq, Sk, dtype=torch.int64)
    for s in range(n_seq):
        kind = kinds[s % len(kinds)]
        if kind == 0:
            m[s] = (torch.rand(Sk, generator=g) < 0.7).long()
            m[s, 0] = 0
            if Sk > 1 and m[s].sum() == 0:
                m[s, -1] = 1
        elif kind == 1:
            m[s, -1] = 1
        elif kind == 3:
            m[s, Sk // 2:] = 1
        elif kind == 4:
            m[s, :int(torch.randint(1, Sk + 1, (1,), generator=g))] = 1
    return m


def additive_mask(key_real, Sq, causal):
    """[n, 1 or Sq, Sk] fp64: -10000 for a padded key, and under `causal` -10000 once for a padded OR future key"""
    a = torch.where(key_real.bool(), 0.0, MASK_ADD).double()[:, None, :]
    if causal:
        Sk = key_real.shape[1]
        fut = torch.arange(Sk, device=a.device)[None, :] > torch.arange(Sq, device=a.device)[:, None]
        a = torch.where(fut[None] & (a == 0), MASK_ADD, a)
    return a


# ---------------------------------------------------------------------------------------------------------
# fp64 reference with per-element bounds
# ---------------------------------------------------------------------------------------------------------
def _heads(t, n, S):
    return t.double().reshape(n, S, HEADS, HD).permute(0, 2, 1, 3)


def _unheads(t):
    n, h, S, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(n * S, h * d)


def softmax_rel(kind, Sk):
    """relative error of a row's normalisation beyond the per-score terms: the exponentials (EXP_REL), the fp32 row
    sum of Sk terms and the reciprocal / scale multiplies; the key-tiled kernel also rescales its running sum and
    accumulator once per 64-key tile (each rescale errs by EXP_REL + 2U, and the U |m_old - m_new| of its argument is
    weighted by the exp(-|m_old - m_new|) it multiplies: at most U / e in all)"""
    rel = 2 * EXP_REL + (Sk + 4) * U
    if kind == "long":
        rel += -(-Sk // 64) * (EXP_REL + 2 * U) + U
    return rel


def reference(q, k, v, n_seq, Sq, Sk, key_real, causal=False, keep=None, p=0.0, d_o=None, o_kernel=None,
              kind="short", chunk_elems=2 ** 25, want_p=False):
    """fp64 attention of the kernels' bf16 inputs, forward and (with d_o) backward, and the bound of every output.
    q [n_seq Sq, 768], k / v [n_seq Sk, 768] (head h in columns h*64 .. h*64+63); key_real [n_seq, Sk] (nonzero = real
    key); keep: bool [n_seq heads, Sq, Sk] dropout mask or None; o_kernel: the kernel's bf16 context, which its
    backward reads for D_i = dO_i . O_i.  kind: "short" / "long" / "fused" (softmax_rel).
    Returns a dict: o, b_o [n_seq Sq, 768]; lse, b_lse [n_seq heads Sq]; with d_o also dq, b_dq, dk, b_dk, dv, b_dv.
    Computed in chunks of sequences (chunk_elems scores at a time)."""
    dev = q.device
    c = 1.0 / (1.0 - float(np.float32(p))) if keep is not None else 1.0
    per = max(1, chunk_elems // (HEADS * Sq * Sk))
    out = {n: [] for n in ("o", "b_o", "lse", "b_lse", "dq", "b_dq", "dk", "b_dk", "dv", "b_dv", "p")}
    for s0 in range(0, n_seq, per):
        n = min(per, n_seq - s0)
        qh = _heads(q[s0 * Sq:(s0 + n) * Sq], n, Sq)
        kh = _heads(k[s0 * Sk:(s0 + n) * Sk], n, Sk)
        vh = _heads(v[s0 * Sk:(s0 + n) * Sk], n, Sk)
        a = additive_mask(key_real[s0:s0 + n].to(dev), Sq, causal)[:, None]       # [n, 1, Sq|1, Sk]
        M = keep[s0 * HEADS:(s0 + n) * HEADS].to(dev).view(n, HEADS, Sq, Sk).double() if keep is not None else None
        grad = d_o is not None
        qg, kg, vg = (t.clone().requires_grad_(grad) for t in (qh, kh, vh))
        s = SCALE * (qg @ kg.transpose(-1, -2)) + a
        P = torch.softmax(s, -1)
        Pd = c * M * P if M is not None else P
        O = Pd @ vg
        with torch.no_grad():
            sd, Pt = s.detach(), P.detach()
            lse = torch.logsumexp(sd, -1)
            mag = SCALE * (qh.abs() @ kh.abs().transpose(-1, -2))
            delta = (C_ACC * HD * U + SCORE_ROUNDS * U) * mag + SCORE_ROUNDS * U * a.abs()
            Delta = (Pt * delta).sum(-1, keepdim=True)           # P-weighted: the normalisation's share of the errors
            m = sd.amax(-1, keepdim=True)
            rel = softmax_rel(kind, Sk)
            rho = delta + Delta + EXP_ARG * U * (sd - m).abs() + rel
            Pm = c * M * Pt if M is not None else Pt
            b_o = (Pm * (BF16_ROUND + rho + C_ACC * Sk * U)) @ vh.abs() + BF16_ROUND * O.detach().abs()
            b_lse = Delta[..., 0] + rel + LOG_ABS + 8 * U * lse.abs().clamp_min(1.0)
            out["o"].append(_unheads(O.detach()))
            out["b_o"].append(_unheads(b_o))
            out["lse"].append(lse.reshape(-1))
            out["b_lse"].append(b_lse.reshape(-1))
            if want_p:
                out["p"].append(Pt)
        if not grad:
            continue
        dOh = _heads(d_o[s0 * Sq:(s0 + n) * Sq], n, Sq)
        O.backward(dOh)
        with torch.no_grad():
            Ok = _heads(o_kernel[s0 * Sq:(s0 + n) * Sq], n, Sq)
            dP = dOh @ vh.transpose(-1, -2)
            e_dP = C_ACC * HD * U * (dOh.abs() @ vh.abs().transpose(-1, -2))
            D = (dOh * O.detach()).sum(-1, keepdim=True)
            # D_i = dO_i . O_i from the context the backward is given, the kernel's bf16 one (its error against O is
            # checked by the forward bound): that difference exactly, plus a 64-term fp32 dot product
            e_D = (dOh * (Ok - O.detach())).sum(-1, keepdim=True).abs() + \
                C_ACC * HD * U * (dOh.abs() * Ok.abs()).sum(-1, keepdim=True)
            # P recomputed from the saved lse: the score errors, the lse bound, the exponential
            rho_b = delta + b_lse[..., None] + EXP_ARG * U * (sd - lse[..., None]).abs() + EXP_REL + 4 * U
            g = c * M * dP.abs() if M is not None else dP.abs()
            e_g = c * M * e_dP if M is not None else e_dP
            size = g + D.abs() + e_D                                # |c M dP - D| without cancellation
            # dS = scale P (c M dP - D) in fp32 (P, the subtraction and the products: rho_b + 4U), then rounded to bf16
            # for the dQ / dK products: 2^-8 of |dS| itself, which the cancellation in (c M dP - D) can make small
            dS = SCALE * Pt * ((c * M * dP if M is not None else dP) - D)
            e_pre = SCALE * Pt * ((rho_b + 4 * U) * size + e_g + e_D)
            e_dS = e_pre * (1 + BF16_ROUND) + BF16_ROUND * dS.abs()
            m_dS = SCALE * Pt * size
            dQ, dK, dV = _unheads(qg.grad), _unheads(kg.grad), _unheads(vg.grad)
            b_dq = _unheads(e_dS @ kh.abs() + C_ACC * Sk * U * (m_dS @ kh.abs())) + BF16_ROUND * dQ.abs()
            e_dSt, m_dSt = e_dS.transpose(-1, -2), m_dS.transpose(-1, -2)
            b_dk = _unheads(e_dSt @ qh.abs() + C_ACC * Sq * U * (m_dSt @ qh.abs())) + BF16_ROUND * dK.abs()
            Pmt = Pm.transpose(-1, -2)
            b_dv = _unheads((Pmt * (rho_b + BF16_ROUND + 2 * U).transpose(-1, -2)) @ dOh.abs()
                            + C_ACC * Sq * U * (Pmt @ dOh.abs())) + BF16_ROUND * dV.abs()
            for name, val in (("dq", dQ), ("b_dq", b_dq), ("dk", dK), ("b_dk", b_dk), ("dv", dV), ("b_dv", b_dv)):
                out[name].append(val)
    return {name: torch.cat(vals) for name, vals in out.items() if vals}


def bias_bound(grad_ref, b_grad):
    """bound of a projection-bias gradient (column sums of the fp32 accumulators, summed in a fixed order) against the
    column sums of the fp64 gradient: the rows' bounds without their bf16 output rounding, plus the fp32 summation of
    `rows` terms"""
    rows = grad_ref.shape[0]
    acc_bound = (b_grad - BF16_ROUND * grad_ref.abs()).sum(0)
    return acc_bound + (rows + 8) * U * grad_ref.abs().sum(0) + 1e-30


def check_fwd(o, lse, ref, what):
    """o [n_seq Sq, 768] (any row stride) and lse against a reference() dict; returns the two worst ratios"""
    return (within(o, ref["o"], ref["b_o"], what + " o"),
            within(lse, ref["lse"], ref["b_lse"], what + " lse"))


def check_bwd(dq, dk, dv, ref, what):
    return tuple(within(got, ref[n], ref["b_" + n], "%s %s" % (what, n)) for got, n in ((dq, "dq"), (dk, "dk"),
                                                                                        (dv, "dv")))


def old_tolerance_accepts(got, ref, grad=False):
    """the per-tensor fp32 tolerance the attention tests used before this checker: |o - ref| <= 3e-2, and
    |grad - ref| <= 4e-2 max(1, max|ref|)"""
    err = float((got.double() - ref).abs().max())
    return err <= (4e-2 * max(1.0, float(ref.abs().max())) if grad else 3e-2)
