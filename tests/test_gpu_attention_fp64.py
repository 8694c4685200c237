"""GPU: every attention entry point, forward and backward, element by element against fp64 (tests/attn_check.py), with
the dropout masks reproduced bit for bit by a host Philox.

Inputs the model's own shapes never produce: scattered key masks, key 0 padded, a row whose only real key is the last
one, fully padded sequences, causal rows whose past keys are all padded; unit-variance and peaked (q x 4) scores; for
the key-tiled kernel, keys that make every row's running max rise by more than 10 in two later 64-key tiles.  q / k /
v are column slices of NaN-padded buffers; o, lse and the gradients are written into sentinel-filled buffers with
leading dimensions above 768, and the padding must come back untouched.  Dropout runs with a seed that has bits above
32, a non-zero epoch, and a stream id for which stream + (epoch << 20) crosses 2^32."""
import numpy as np
import pytest
import torch

from tests import attn_check as ac
from tests import gemm_check as gc
from univl_b200 import ops
from univl_b200 import runtime as rt

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
H, HEADS = 768, 12
NAN = float("nan")
SEED = (1 << 40) + 0x2468ACE1   # rng_state[0]: bits above 32 are part of the Philox key
EPOCH = 3                        # rng_state[1]
STREAM = 2 ** 32 - (EPOCH << 20) + 11   # the kernels draw from stream + (epoch << 20) = 2^32 + 11


def _rng():
    return torch.tensor([SEED, EPOCH], dtype=torch.int64, device=DEV)


def _stream():
    return ac.kernel_stream(STREAM, EPOCH)


# ---------------------------------------------------------------------------------------------------------
# inputs and outputs
# ---------------------------------------------------------------------------------------------------------
def _inputs(n_seq, Sq, Sk, seed, qscale=1.0, rising=False):
    """q [n_seq Sq, 768] as columns 64..831 of an 832-wide buffer, k / v as columns 0..767 and 832..1599 of a
    1664-wide one; NaN in the gaps, the tails and the 4 rows after the last sequence.  rising: dimension 0 of every
    head is 4 in q, and keys 70 and 200 carry 28 / 56 there (scores +14 / +28 over the other keys'): every row's
    running max rises by > 10 in key tiles 1 and 3"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    qbuf = torch.full((n_seq * Sq + 4, 832), NAN, dtype=BF16, device=DEV)
    kvbuf = torch.full((n_seq * Sk + 4, 1664), NAN, dtype=BF16, device=DEV)
    q, k, v = qbuf[:n_seq * Sq, 64:64 + H], kvbuf[:n_seq * Sk, :H], kvbuf[:n_seq * Sk, 832:832 + H]
    q.copy_(torch.randn(n_seq * Sq, H, device=DEV, generator=g) * qscale)
    k.copy_(torch.randn(n_seq * Sk, H, device=DEV, generator=g))
    v.copy_(torch.randn(n_seq * Sk, H, device=DEV, generator=g))
    if rising:
        q.view(n_seq * Sq, HEADS, 64)[:, :, 0] = 4.0
        kh = k.view(n_seq, Sk, HEADS, 64)
        kh[:, 70, :, 0] = 28.0
        kh[:, 200, :, 0] = 56.0
    d_o = torch.randn(n_seq * Sq, H, device=DEV, generator=g).to(BF16)
    return q, k, v, d_o


def _mask(n_seq, Sk, seed, kinds=(0, 1, 2, 3, 4), rising=False):
    m = ac.edge_masks(n_seq, Sk, seed, kinds)
    if rising:
        for s in range(n_seq):
            if m[s].sum() > 1:
                m[s, 70] = m[s, 200] = 1
    return m.to(DEV)


class Outs:
    """sentinel-filled output buffers: o [rows, 768] (ld 776), lse (+8 sentinels), dq / dk / dv (ld 784 / 792 / 800)"""

    def __init__(self, n_seq, Sq, Sk):
        self.shape = (n_seq, Sq, Sk)
        self.o_buf, self.o, _ = gc.out_buf(n_seq * Sq, H, 776, BF16)
        self.lse_buf = torch.full((n_seq * HEADS * Sq + 8,), gc.SENT_F32, device=DEV)
        self.lse = self.lse_buf[:n_seq * HEADS * Sq]
        self.dq_buf, self.dq, _ = gc.out_buf(n_seq * Sq, H, 784, BF16)
        self.dk_buf, self.dk, _ = gc.out_buf(n_seq * Sk, H, 792, BF16)
        self.dv_buf, self.dv, _ = gc.out_buf(n_seq * Sk, H, 800, BF16)

    def assert_fwd_padding(self, what):
        n_seq, Sq, _ = self.shape
        gc.assert_padding(self.o_buf, n_seq * Sq, H, gc.SENT_BF16, what + " o")
        assert bool((self.lse_buf[n_seq * HEADS * Sq:] == gc.SENT_F32).all()), what + ": lse padding written"

    def assert_bwd_padding(self, what):
        n_seq, Sq, Sk = self.shape
        gc.assert_padding(self.dq_buf, n_seq * Sq, H, gc.SENT_BF16, what + " dq")
        gc.assert_padding(self.dk_buf, n_seq * Sk, H, gc.SENT_BF16, what + " dk")
        gc.assert_padding(self.dv_buf, n_seq * Sk, H, gc.SENT_BF16, what + " dv")


def attn_fwd(kernel, q, k, v, out, n_seq, Sq, Sk, spec, p, rng):
    """univl_attention_fwd (kernel "short") or univl_attention_long_fwd ("long") called directly"""
    entry = "univl_attention_fwd" if kernel == "short" else "univl_attention_long_fwd"
    rt.call(entry, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.o.data_ptr(),
            out.o.stride(0), out.lse.data_ptr(), rt.ptr(spec.a), rt.ptr(spec.b), spec.Wa, spec.Fb, spec.Nb,
            int(spec.all_pairs), n_seq, HEADS, Sq, Sk, int(spec.causal), ac.SCALE, float(p),
            rng.data_ptr() if p > 0 else None, STREAM)


def attn_bwd(kernel, q, k, v, d_o, out, n_seq, Sq, Sk, spec, p, rng, dbias=None, rng_layout=0):
    entry = "univl_attention_bwd" if kernel == "short" else "univl_attention_long_bwd"
    db = dbias if dbias is not None else (None, None, None)
    rt.call(entry, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.o.data_ptr(),
            out.o.stride(0), out.lse.data_ptr(), d_o.data_ptr(), d_o.stride(0), out.dq.data_ptr(), out.dq.stride(0),
            out.dk.data_ptr(), out.dk.stride(0), out.dv.data_ptr(), out.dv.stride(0), rt.ptr(spec.a), rt.ptr(spec.b),
            spec.Wa, spec.Fb, spec.Nb, int(spec.all_pairs), n_seq, HEADS, Sq, Sk, int(spec.causal), ac.SCALE, float(p),
            rng.data_ptr() if p > 0 else None, STREAM, rng_layout, *[rt.ptr(t) for t in db])


def run_and_check(kernel, n_seq, Sq, Sk, causal, p, qscale=1.0, rising=False, kinds=(0, 1, 2, 3, 4), seed=0):
    """forward and backward of one kernel, every output against fp64 under the tile-layout dropout mask"""
    what = "%s n%d Sq%d Sk%d causal%d p%g q x%g%s" % (kernel, n_seq, Sq, Sk, causal, p, qscale,
                                                       " rising" if rising else "")
    q, k, v, d_o = _inputs(n_seq, Sq, Sk, seed + Sq + Sk, qscale, rising)
    key_real = _mask(n_seq, Sk, seed + Sk, kinds, rising)
    spec = ops.MaskSpec(key_real, causal=causal)
    rng = _rng()
    out = Outs(n_seq, Sq, Sk)
    attn_fwd(kernel, q, k, v, out, n_seq, Sq, Sk, spec, p, rng)
    dbias = torch.ones(3, H, device=DEV)
    attn_bwd(kernel, q, k, v, d_o, out, n_seq, Sq, Sk, spec, p, rng, dbias=(dbias[0], dbias[1], dbias[2]))
    torch.cuda.synchronize()
    keep = ac.keep_tile(SEED, _stream(), p, n_seq * HEADS, Sq, Sk) if p > 0 else None
    ref = ac.reference(q, k, v, n_seq, Sq, Sk, key_real, causal, keep, p, d_o=d_o, o_kernel=out.o,
                       kind="long" if kernel == "long" else "short")
    ac.check_fwd(out.o, out.lse, ref, what)
    ac.check_bwd(out.dq, out.dk, out.dv, ref, what)
    for n, name in enumerate(("dq", "dk", "dv")):
        gc.within(dbias[n] - 1.0, ref[name].sum(0), ac.bias_bound(ref[name], ref["b_" + name]), what + " db" + name[1])
    out.assert_fwd_padding(what)
    out.assert_bwd_padding(what)
    return out, ref


# ---------------------------------------------------------------------------------------------------------
# attention.cu (S <= 256) and, at short shapes too, attention_long.cu
# ---------------------------------------------------------------------------------------------------------
OTHER_SQ = {1: 9, 15: 40, 17: 5, 33: 100, 96: 20, 255: 64, 256: 200}
SHORT_CASES = []
for _Sk in (1, 15, 17, 33, 96, 255, 256):
    for _Sq in sorted({_Sk, 1, OTHER_SQ[_Sk]}):
        _i = len(SHORT_CASES)
        SHORT_CASES.append((_Sq, _Sk, _Sq == _Sk and _Sk > 1, (0.0, 0.1, 0.25)[_i % 3], 4.0 if _i % 2 else 1.0))


@pytest.mark.parametrize("Sq,Sk,causal,p,qscale", SHORT_CASES)
def test_short_attention_fp64(Sq, Sk, causal, p, qscale):
    run_and_check("short", 5 if Sk <= 96 else 3, Sq, Sk, causal, p, qscale)


@pytest.mark.parametrize("Sq,Sk,causal,p,qscale", [c for c in SHORT_CASES if c[1] in (1, 17, 96, 256)])
def test_long_kernel_at_short_shapes_fp64(Sq, Sk, causal, p, qscale):
    run_and_check("long", 5 if Sk <= 96 else 3, Sq, Sk, causal, p, qscale)


# ---------------------------------------------------------------------------------------------------------
# attention_long.cu beyond 256 tokens
# ---------------------------------------------------------------------------------------------------------
LONG_CASES = []
for _Sk in (257, 300, 511, 1000, 1023, 1024):
    for _Sq in (1, 5, 63, 64, 65, _Sk):
        _i = len(LONG_CASES)
        LONG_CASES.append((_Sq, _Sk, _Sq == _Sk and _i % 2 == 1, (0.0, 0.1, 0.25)[_i % 3]))


@pytest.mark.parametrize("Sq,Sk,causal,p", LONG_CASES)
def test_long_attention_fp64(Sq, Sk, causal, p):
    # causal: the first-half-padded kind, whose early rows attend to their future keys; otherwise rising maxima
    kinds = (3, 0) if causal else (0, 1, 2) if Sq < Sk else (0, 1)
    run_and_check("long", 2 if Sq == Sk else 3, Sq, Sk, causal, p, qscale=1.0, rising=not causal, kinds=kinds)


def test_short_and_long_kernels_draw_the_same_mask():
    """at a shape both take, both kernels' outputs and gradients pass the checker under the SAME tile-layout mask"""
    for kernel in ("short", "long"):
        run_and_check(kernel, 3, 96, 96, False, 0.25, seed=11)
        run_and_check(kernel, 2, 224, 224, True, 0.1, kinds=(3, 0), seed=12)


# ---------------------------------------------------------------------------------------------------------
# fused_attn.cu: QKV projection + attention forward, wgmma backward
# ---------------------------------------------------------------------------------------------------------
def fused_run_and_check(n_seq, S, causal, p, mask_a, mask_b=None, groups=0, seed=0):
    what = "fused n%d S%d causal%d p%g groups%d" % (n_seq, S, causal, p, groups)
    g = torch.Generator(device=DEV).manual_seed(seed + S)
    T = n_seq * S
    xbuf = torch.full((T + 4, H + 64), NAN, dtype=BF16, device=DEV)
    x = xbuf[:T, :H]
    x.copy_(torch.randn(T, H, device=DEV, generator=g))
    w = (torch.randn(3 * H, H, device=DEV, generator=g) * 0.04).to(BF16)
    b = torch.randn(3 * H, device=DEV, generator=g) * 0.2
    d_o = torch.randn(T, H, device=DEV, generator=g).to(BF16)
    spec = ops.MaskSpec(mask_a, mask_b, all_pairs=groups, causal=causal)
    rng = _rng()
    out = Outs(n_seq, S, S)
    qkv = torch.empty(T, 3 * H, dtype=BF16, device=DEV)

    def fwd(qkv_out, o, lse):
        rt.call("univl_fused_qkv_attention_fwd", x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), b.data_ptr(),
                rt.ptr(qkv_out), 3 * H, o.data_ptr(), o.stride(0), lse.data_ptr(), rt.ptr(spec.a), rt.ptr(spec.b),
                spec.Wa, spec.Fb, spec.Nb, int(spec.all_pairs), n_seq, HEADS, S, int(causal), ac.SCALE, float(p),
                rng.data_ptr() if p > 0 else None, STREAM)
    fwd(qkv, out.o, out.lse)
    dq_buf, dqkv, _ = gc.out_buf(T, 3 * H, 3 * H + 64, BF16)
    dbias = torch.ones(3 * H, device=DEV)
    rt.call("univl_fused_attention_bwd", qkv.data_ptr(), qkv.stride(0), out.o.data_ptr(), out.o.stride(0),
            out.lse.data_ptr(), d_o.data_ptr(), d_o.stride(0), dqkv.data_ptr(), dqkv.stride(0), dbias.data_ptr(),
            rt.ptr(spec.a), rt.ptr(spec.b), spec.Wa, spec.Fb, spec.Nb, int(spec.all_pairs), n_seq, HEADS, S,
            int(causal), ac.SCALE, float(p), rng.data_ptr() if p > 0 else None, STREAM)
    o2 = torch.empty(T, H, dtype=BF16, device=DEV)
    lse2 = torch.empty(n_seq * HEADS * S, device=DEV)
    fwd(None, o2, lse2)
    torch.cuda.synchronize()
    # the saved projections per element (tests/gemm_check.py), then the attention reference on them
    acc, mag = gc.mm64(x, w)
    qkv_ref = acc + b.double()
    gc.within(qkv, qkv_ref, gc.elem_bound(mag, H, b.double().abs(), qkv_ref), what + " qkv")
    assert torch.equal(o2, out.o) and torch.equal(lse2, out.lse), what + ": save_qkv=False changed the context"
    key_real = ac.pair_masks(mask_a, mask_b, n_seq, groups)
    keep = ac.keep_rowmajor(SEED, _stream(), p, n_seq * HEADS, S) if p > 0 else None
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    ref = ac.reference(q, k, v, n_seq, S, S, key_real, causal, keep, p, d_o=d_o, o_kernel=out.o, kind="fused")
    ac.check_fwd(out.o, out.lse, ref, what)
    ac.check_bwd(dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:], ref, what)
    col = torch.cat([ref[n].sum(0) for n in ("dq", "dk", "dv")])
    bnd = torch.cat([ac.bias_bound(ref[n], ref["b_" + n]) for n in ("dq", "dk", "dv")])
    gc.within(dbias - 1.0, col, bnd, what + " dbias")
    out.assert_fwd_padding(what)
    gc.assert_padding(dq_buf, T, 3 * H, gc.SENT_BF16, what + " dqkv")
    # the mma.sync backward on the same saved tensors regenerates the fused forward's row-major mask
    attn_bwd("short", q, k, v, d_o, out, n_seq, S, S, spec, p, rng, rng_layout=1)
    torch.cuda.synchronize()
    ac.check_bwd(out.dq, out.dk, out.dv, ref, what + " mma.sync rng_layout 1")
    out.assert_bwd_padding(what + " mma.sync rng_layout 1")
    return out, qkv, ref


# (n_seq, S): the last row block of G = 128 // S sequences is partial wherever G > 1
@pytest.mark.parametrize("n_seq,S,causal,p", [(11, 16, False, 0.1), (5, 48, False, 0.0), (5, 48, True, 0.25),
                                              (3, 80, False, 0.25), (2, 96, False, 0.1), (3, 112, False, 0.0),
                                              (2, 128, True, 0.1), (9, 16, True, 0.0)])
def test_fused_attention_fp64(n_seq, S, causal, p):
    fused_run_and_check(n_seq, S, causal, p, _mask(n_seq, S, S + n_seq), seed=n_seq)


@pytest.mark.parametrize("groups,p", [(1, 0.0), (2, 0.25)])
def test_fused_attention_pair_masks_fp64(groups, p):
    """all-pairs (text mask i, video mask j for pair (i, j)) and grouped (G = 2 micro-batches) masks"""
    Na, Nb, W, F = (3, 4, 16, 32) if groups == 1 else (4, 4, 16, 32)
    n_seq = Na * Nb // groups
    ma = ac.edge_masks(Na, W, 5, kinds=(0, 4, 2)).to(DEV)
    mb = ac.edge_masks(Nb, F, 6, kinds=(4, 0, 1, 2)).to(DEV)
    fused_run_and_check(n_seq, W + F, False, p, ma, mb, groups)


# ---------------------------------------------------------------------------------------------------------
# attention_pair.cu
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,F,first", [(40, 56, True), (40, 56, False), (128, 160, True), (128, 160, False)])
def test_pair_attention_fp64(W, F, first):
    Na, Nb = 3, 2
    S = W + F
    Sq = 1 if first else S
    g = torch.Generator(device=DEV).manual_seed(W + F + first)
    qkv_a = (torch.randn(Na * W, 3 * H, device=DEV, generator=g)).to(BF16)
    qkv_b = (torch.randn(Nb * F, 3 * H, device=DEV, generator=g)).to(BF16)
    ma = ac.edge_masks(Na, W, 7, kinds=(0, 2, 4)).to(DEV)
    mb = ac.edge_masks(Nb, F, 8, kinds=(4, 1)).to(DEV)
    spec = ops.MaskSpec(ma, mb, all_pairs=True)
    o = ops.attention_pair_fwd(qkv_a, qkv_b, Na, Nb, Sq, spec)
    torch.cuda.synchronize()
    n_seq = Na * Nb
    i = torch.arange(n_seq, device=DEV) // Nb
    j = torch.arange(n_seq, device=DEV) % Nb
    seqs = torch.cat([qkv_a.view(Na, W, 3 * H)[i], qkv_b.view(Nb, F, 3 * H)[j]], 1)      # [n_seq, S, 3H]
    q = seqs[:, :Sq, :H].reshape(-1, H)
    k, v = seqs[:, :, H:2 * H].reshape(-1, H), seqs[:, :, 2 * H:].reshape(-1, H)
    key_real = ac.pair_masks(ma, mb, n_seq, 1)
    ref = ac.reference(q, k, v, n_seq, Sq, S, key_real, kind="short" if S <= 256 else "long")
    gc.within(o, ref["o"], ref["b_o"], "pair W%d F%d Sq%d o" % (W, F, Sq))


# ---------------------------------------------------------------------------------------------------------
# the checker rejects what it is meant to catch
# ---------------------------------------------------------------------------------------------------------
def _rejects(got, ref, bound, what, old_ref=None, grad=False):
    """the checker rejects `got` against the perturbed reference; prints whether the old fp32 tolerance did"""
    with pytest.raises(AssertionError):
        gc.within(got, ref, bound, what)
    if old_ref is not None:
        print("old tolerance accepts %s: %s" % (what, ac.old_tolerance_accepts(got, old_ref, grad)))


def _short_case(p=0.25):
    n_seq, S = 3, 33
    q, k, v, d_o = _inputs(n_seq, S, S, 21)
    key_real = torch.ones(n_seq, S, dtype=torch.int64, device=DEV)
    spec = ops.MaskSpec(key_real)
    out = Outs(n_seq, S, S)
    rng = _rng()
    attn_fwd("short", q, k, v, out, n_seq, S, S, spec, p, rng)
    attn_bwd("short", q, k, v, d_o, out, n_seq, S, S, spec, p, rng)
    torch.cuda.synchronize()
    keep = ac.keep_tile(SEED, _stream(), p, n_seq * HEADS, S, S)
    return n_seq, S, q, k, v, d_o, key_real, out, keep


def test_checker_rejects_a_dropped_last_key():
    """a reference with key 32 (the only key of the last, partial 16-key block) dropped: rejected.  (The old 3e-2
    tolerance rejected it too, measured on an H100; each run prints "old tolerance accepts ...".)"""
    n_seq, S, q, k, v, d_o, key_real, out, keep = _short_case()
    ref = ac.reference(q, k, v, n_seq, S, S, key_real, keep=keep, p=0.25)
    ac.check_fwd(out.o, out.lse, ref, "unperturbed")
    kr = key_real.clone()
    kr[:, -1] = 0
    r = ac.reference(q, k, v, n_seq, S, S, kr, keep=keep, p=0.25)
    _rejects(out.o, r["o"], r["b_o"], "last key dropped", r["o"])


def test_checker_rejects_a_shifted_or_flipped_dropout_mask():
    """the tile mask shifted by one key, and one kept element (the largest probability) flipped to dropped: both
    rejected.  (The old 3e-2 tolerance rejected both as well at these peaked probabilities, measured on an H100; it
    never saw a mask at all, since no old test compared a dropout output with an independent reference.)"""
    n_seq, S, q, k, v, d_o, key_real, out, keep = _short_case()
    ref = ac.reference(q, k, v, n_seq, S, S, key_real, keep=keep, p=0.25, want_p=True)
    ac.check_fwd(out.o, out.lse, ref, "unperturbed")
    r = ac.reference(q, k, v, n_seq, S, S, key_real, keep=keep.roll(1, -1), p=0.25)
    _rejects(out.o, r["o"], r["b_o"], "mask shifted by one key", r["o"])
    flip = keep.clone()
    idx = np.unravel_index(int((ref["p"].reshape(flip.shape).cpu() * flip).argmax()), tuple(flip.shape))
    flip[idx] = False
    r = ac.reference(q, k, v, n_seq, S, S, key_real, keep=flip, p=0.25)
    _rejects(out.o, r["o"], r["b_o"], "one dropout element flipped", r["o"])


def test_checker_rejects_the_other_dropout_layout():
    """the short kernel's output against the row-major mask, and the fused kernel's against the tile mask: rejected.
    (The old 3e-2 tolerance would have rejected both too, measured on an H100, had an old test had a reference mask.)"""
    n_seq, S = 3, 48
    q, k, v, d_o = _inputs(n_seq, S, S, 22)
    key_real = torch.ones(n_seq, S, dtype=torch.int64, device=DEV)
    spec = ops.MaskSpec(key_real)
    out = Outs(n_seq, S, S)
    attn_fwd("short", q, k, v, out, n_seq, S, S, spec, 0.25, _rng())
    torch.cuda.synchronize()
    tile = ac.keep_tile(SEED, _stream(), 0.25, n_seq * HEADS, S, S)
    rowm = ac.keep_rowmajor(SEED, _stream(), 0.25, n_seq * HEADS, S)
    ac.check_fwd(out.o, out.lse, ac.reference(q, k, v, n_seq, S, S, key_real, keep=tile, p=0.25), "unperturbed")
    r = ac.reference(q, k, v, n_seq, S, S, key_real, keep=rowm, p=0.25)
    _rejects(out.o, r["o"], r["b_o"], "short kernel, row-major mask", r["o"])
    fout, qkv, _ = fused_run_and_check(n_seq, S, False, 0.25, key_real.clone(), seed=23)
    r = ac.reference(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], n_seq, S, S, key_real, keep=tile, p=0.25,
                     kind="fused")
    _rejects(fout.o, r["o"], r["b_o"], "fused kernel, tile mask", r["o"])


def test_checker_rejects_a_shifted_lse_and_dk_missing_the_last_query():
    """one row's lse moved by three times its bound, and a reference dK without the last query row's contribution:
    both rejected.  The old tolerances (1e-2 max(1, max|lse|) on lse, 4e-2 max(1, max|dK|) on dK; measured on an
    H100) ACCEPTED the shifted lse and rejected the dK."""
    n_seq, S, q, k, v, d_o, key_real, out, keep = _short_case()
    ref = ac.reference(q, k, v, n_seq, S, S, key_real, keep=keep, p=0.25, d_o=d_o, o_kernel=out.o)
    ac.check_bwd(out.dq, out.dk, out.dv, ref, "unperturbed")
    bad = out.lse.double().clone()
    bad[40] += 3 * ref["b_lse"][40]
    _rejects(bad, ref["lse"], ref["b_lse"], "lse shifted by 3 bounds")
    print("old tolerance accepts lse shifted by 3 bounds: %s" % bool((bad - ref["lse"]).abs().max() <= 1e-2))
    d0 = d_o.clone().view(n_seq, S, H)
    d0[:, -1] = 0
    r = ac.reference(q, k, v, n_seq, S, S, key_real, keep=keep, p=0.25, d_o=d0.view(-1, H), o_kernel=out.o)
    _rejects(out.dk, r["dk"], r["b_dk"], "dK missing the last query row", r["dk"], grad=True)


# ---------------------------------------------------------------------------------------------------------
# LayerNorm and embedding dropout: the element layout (dropout_keep8), element by element
# ---------------------------------------------------------------------------------------------------------
def _assert_dropped_exactly(y, y0, keep, p, what):
    """y = dropout(y0) on `keep`: zero exactly where dropped, y0 / (1 - p) up to two bf16 roundings where kept"""
    c = 1.0 / (1.0 - p)
    keep = keep.to(y.device)
    assert bool((y[~keep] == 0).all()), what + ": an element the mask drops is non-zero"
    want = y0.double() * c * keep
    gc.within(y, want, 2.0 ** -7 * want.abs() + 1e-6, what)


@pytest.mark.parametrize("rows,cols", [(37, 768), (130, 1024)])
def test_layernorm_dropout_masks_are_the_element_layout(rows, cols):
    g = torch.Generator(device=DEV).manual_seed(rows)
    x = torch.randn(rows, cols, device=DEV, generator=g).to(BF16)
    res = torch.randn(rows, cols, device=DEV, generator=g).to(BF16)
    gamma = 1 + 0.1 * torch.randn(cols, device=DEV, generator=g)
    beta = 0.1 * torch.randn(cols, device=DEV, generator=g)
    rng = _rng()
    for p in (0.1, 0.25):
        keep = ac.keep_elem(SEED, _stream(), p, rows, cols).to(DEV)
        c = 1.0 / (1.0 - p)
        # mode 2: y = dropout(LN(x + res))
        y0, _, _ = ops.layernorm_fwd(x, res, gamma, beta)
        y, mean, rstd = ops.layernorm_fwd(x, res, gamma, beta, p=p, mode=2, seed=rng.data_ptr(), stream=STREAM)
        _assert_dropped_exactly(y, y0, keep, p, "layernorm mode 2 p%g" % p)
        dy = torch.randn(rows, cols, device=DEV, generator=g).to(BF16)
        _, _, _, dbeta, _ = ops.layernorm_bwd(dy, None, x, res, gamma, mean, rstd, p=p, mode=2, seed=rng.data_ptr(),
                                              stream=STREAM, want_dbias=False)
        want = (dy.double() * keep * c).sum(0)
        gc.within(dbeta, want, (rows + 8) * ac.U * (dy.double().abs() * c).sum(0) + 1e-6, "layernorm mode 2 dbeta")
        # mode 1: y = LN(dropout(x) + res); dx_dense = dz keep / (1 - p)
        y, mean, rstd = ops.layernorm_fwd(x, res, gamma, beta, p=p, mode=1, seed=rng.data_ptr(), stream=STREAM)
        z = x.double() * keep * c + res.double()
        u = z.mean(-1, keepdim=True)
        ref = gamma.double() * (z - u) / torch.sqrt((z - u).pow(2).mean(-1, keepdim=True) + 1e-12) + beta.double()
        assert float((y.double() - ref).abs().max()) <= 2e-2, "layernorm mode 1 p%g forward mask" % p
        dx_res, dx_dense, _, _, _ = ops.layernorm_bwd(dy, None, x, res, gamma, mean, rstd, p=p, mode=1,
                                                      seed=rng.data_ptr(), stream=STREAM)
        assert dx_dense is not dx_res
        _assert_dropped_exactly(dx_dense, dx_res, keep, p, "layernorm mode 1 p%g dx_dense" % p)


def test_embedding_dropout_masks_are_the_element_layout():
    n, S, V = 3, 20, 1000
    g = torch.Generator(device=DEV).manual_seed(7)
    word = torch.randn(V, H, device=DEV, generator=g) * 0.5
    pos = torch.randn(512, H, device=DEV, generator=g) * 0.5
    type_w = torch.randn(2, H, device=DEV, generator=g) * 0.5
    gamma = 1 + 0.1 * torch.randn(H, device=DEV, generator=g)
    beta = 0.1 * torch.randn(H, device=DEV, generator=g)
    ids = torch.randint(0, V, (n, S), device=DEV, generator=g)
    tids = torch.randint(0, 2, (n, S), device=DEV, generator=g)
    rng = _rng()

    def text(p):
        y = torch.empty(n * S, H, dtype=BF16, device=DEV)
        st = torch.empty(2, n * S, device=DEV)
        rt.call("univl_embed_text_fwd", ids.data_ptr(), tids.data_ptr(), word.data_ptr(), pos.data_ptr(),
                type_w.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), st[0].data_ptr(), st[1].data_ptr(),
                n, S, H, V, ops.LN_EPS, float(p), rng.data_ptr() if p > 0 else None, STREAM)
        return y
    Na, Wa, Nb, Fb, G = 4, 12, 4, 20, 2
    a = torch.randn(Na * Wa, H, device=DEV, generator=g).to(BF16)
    b = torch.randn(Nb * Fb, H, device=DEV, generator=g).to(BF16)

    def src(p):
        rows = Na * Nb // G * (Wa + Fb)
        y = torch.empty(rows, H, dtype=BF16, device=DEV)
        st = torch.empty(2, rows, device=DEV)
        rt.call("univl_embed_src_fwd", a.data_ptr(), b.data_ptr(), pos.data_ptr(), type_w.data_ptr(), gamma.data_ptr(),
                beta.data_ptr(), y.data_ptr(), st[0].data_ptr(), st[1].data_ptr(), Na, Wa, Nb, Fb, G, H, ops.LN_EPS,
                float(p), rng.data_ptr() if p > 0 else None, STREAM)
        return y
    for name, fn in (("embed_text", text), ("embed_src groups 2", src)):
        y0 = fn(0.0)
        for p in (0.1, 0.25):
            y = fn(p)
            torch.cuda.synchronize()
            keep = ac.keep_elem(SEED, _stream(), p, y.shape[0], H)
            _assert_dropped_exactly(y, y0, keep, p, "%s p%g" % (name, p))
