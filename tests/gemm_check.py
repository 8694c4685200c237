"""fp64 reference and per-element checker of the wgmma GEMM (csrc/gemm_wgmma.cu), shared by the GEMM tests.

Each output element is checked against its own bound (see `elem_bound`), so an error confined to a tail row, a tail
column or the last k-block cannot hide under a tolerance sized for the largest element."""
import math

import torch

from univl_b200 import ops

DEV = "cuda"
BF16 = torch.bfloat16
U = 2.0 ** -24          # fp32 unit roundoff
# Per-element accumulation constant.  Recursive fp32 summation of K products with round-to-nearest errs by at most
# K * U * sum|a_k b_k|.  Hopper's wgmma is not documented to round to nearest at every add: if its fp32 accumulation
# truncates, each add may lose a full ulp (2U relative) instead of half a ulp (factor 2), and the multi-term adder
# inside one k16 instruction is not documented to keep every alignment bit of the products it sums (another factor 2).
# C_ACC = 4 covers both.  The observed error is far below it (every check prints its worst err / bound as "ratio"),
# and test_gpu_gemm.py::test_checker_rejects_a_dropped_k_slice_and_a_missing_tail_bias shows the bound still rejects
# one dropped 16-wide k slice, or the bias missing from one tail row.
C_ACC = 4.0
# the epilogue's own fp32 operations (alpha scale, bias / aux / accumulator add, split partial sums): a few roundings
EPI_ROUND = 4 * U
# bf16 outputs: 8 significant bits, so round-to-nearest errs by up to half an ulp = 2^-8 relative (at the bottom of a
# binade); bf16 outputs therefore show err / bound ratios close to 1 by construction
BF16_ROUND = 2.0 ** -8
# erf / exp in the GELU epilogues use Abramowitz & Stegun 7.1.26 (|erf error| <= 1.5e-7) and MUFU approximations:
# 1e-6 absolute on gelu' and 1e-6 relative to |x| on gelu covers both
GELU_ABS = 1e-6
GELU_LIP = 1.13          # max |gelu'(x)|: how far an error of the pre-activation can move gelu
SENT_BF16 = -77.0        # sentinel of output padding (exact in bf16 and fp32)
SENT_F32 = -7777.0


# ---------------------------------------------------------------------------------------------------------
# fp64 reference and the per-element checker
# ---------------------------------------------------------------------------------------------------------
def bf_randn(shape, scale, g):
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(BF16)


def mm64(A, B):
    """(A B^T, |A| |B|^T) in fp64 for bf16 A [M, K], B [N, K] (exact products: bf16 x bf16 fits fp64)"""
    a, b = A.double(), B.double()
    return a @ b.t(), a.abs() @ b.abs().t()


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def elem_bound(mag, K, extra=None, out_ref=None):
    """|got - ref| bound of alpha * sum_k a_k b_k (+ epilogue terms) per element:
    C_ACC * K * U * mag  (accumulation; mag = |alpha| (|A| |B|^T))
    + EPI_ROUND * (mag + |extra|)  (the epilogue's fp32 operations on the accumulator and the added terms)
    + BF16_ROUND * |ref|  (when the output is bf16)"""
    b = C_ACC * K * U * mag + EPI_ROUND * (mag if extra is None else mag + extra)
    if out_ref is not None:
        b = b + BF16_ROUND * out_ref.abs()
    return b


def within(got, ref, bound, what):
    """assert |got - ref| <= bound element by element (NaN fails); returns and prints the worst err / bound"""
    err = (got.double() - ref).abs()
    ok = err <= bound
    ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    print("ratio %-60s %.3e" % (what, ratio))
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(int(v) for v in bad[0])
        raise AssertionError("%s: %d of %d elements outside the bound; first %s: got %r ref %r bound %r"
                             % (what, bad.shape[0], ok.numel(), i, float(got[i]), float(ref[i]), float(bound[i])))
    return ratio


def store(X, mn, pad):
    """the storage passed to the kernel for a logical [rows, K] operand.  K-major: [rows, K] with the leading dimension
    rounded up to `pad`.  MN-major: X^T as [K, rows] with the leading dimension rounded up to `pad` (the padded vocab
    layout).  Padding holds NaN: a kernel that reads past the logical extent poisons its output."""
    rows, K = X.shape
    inner = rows if mn else K
    ld = -(-inner // pad) * pad
    buf = torch.full((K if mn else rows, ld), float("nan"), dtype=BF16, device=DEV)
    if mn:
        buf[:, :rows] = X.t()
        return buf[:, :rows]
    buf[:, :K] = X
    return buf[:, :K]


def out_buf(M, N, ld, dtype, extra_rows=3):
    """output view [M, N] with leading dimension ld inside a sentinel-filled buffer of M + extra_rows rows"""
    sent = SENT_F32 if dtype == torch.float32 else SENT_BF16
    buf = torch.full((M + extra_rows, ld), sent, dtype=dtype, device=DEV)
    return buf, buf[:M, :N], sent


def assert_padding(buf, M, N, sent, what):
    """columns [N, ld) of rows < M and every row >= M of the buffer still hold the sentinel"""
    assert bool((buf[:M, N:] == sent).all()), what + ": padding columns written"
    assert bool((buf[M:] == sent).all()), what + ": rows past M written"


OUT_F32 = (ops.EPI_F32, ops.EPI_ATOMIC)


def run_epi(epi, A, B, As, Bs, a_mn, b_mn, *, alpha=1.0, with_bias=True, ldo=None, ld_aux=None, block_n=0,
             split_k=0, g=None, what=""):
    """run one GEMM + epilogue with strided, sentinel-padded outputs and check every output against fp64"""
    M, K = A.shape
    N = B.shape[0]
    ldo = ldo or N
    ld_aux = ld_aux or N
    f32 = epi in OUT_F32
    acc, mag = mm64(A, B)
    mag = abs(alpha) * mag
    acc = alpha * acc
    bias = torch.randn(N, device=DEV, generator=g) if (with_bias and epi in (ops.EPI_BIAS, ops.EPI_GELU, ops.EPI_F32)) \
        else None
    buf, out, sent = out_buf(M, N, ldo, torch.float32 if f32 else BF16)
    aux_in = aux_out = aux_buf = None
    out0 = None
    if epi in (ops.EPI_GELU_BWD, ops.EPI_ADD):
        aux_full = bf_randn((M + 1, ld_aux), 1.0, g)
        aux_in = aux_full[:M, :N]
    if epi == ops.EPI_GELU:
        aux_buf, aux_out, _ = out_buf(M, N, ld_aux, BF16)
    if epi == ops.EPI_ATOMIC:
        out0 = torch.randn(M, N, device=DEV, generator=g)
        out.copy_(out0)
    ops.gemm(As, Bs, M, N, K, out, epi=epi, bias=bias, aux_in=aux_in, aux_out=aux_out, a_mn=a_mn, b_mn=b_mn,
             alpha=alpha, block_n=block_n, split_k=split_k)
    torch.cuda.synchronize()
    b64 = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=DEV)
    if epi in (ops.EPI_BIAS, ops.EPI_F32):
        ref = acc + b64
        within(out, ref, elem_bound(mag, K, b64.abs(), None if f32 else ref), what)
    elif epi == ops.EPI_GELU:
        pre = acc + b64
        bpre = elem_bound(mag, K, b64.abs())
        within(aux_out, pre, bpre + BF16_ROUND * pre.abs(), what + " aux_out")
        ref = gelu64(pre)
        within(out, ref, GELU_LIP * bpre + GELU_ABS * pre.abs() + BF16_ROUND * ref.abs(), what + " out")
        assert_padding(aux_buf, M, N, SENT_BF16, what + " aux_out")
    elif epi == ops.EPI_GELU_BWD:
        gd = gelu_grad64(aux_in.double())
        ref = acc * gd
        bnd = (C_ACC * K * U + EPI_ROUND) * mag * gd.abs() + GELU_ABS * mag + BF16_ROUND * ref.abs()
        within(out, ref, bnd, what)
    elif epi == ops.EPI_ADD:
        x = aux_in.double()
        ref = acc + x
        within(out, ref, elem_bound(mag, K, x.abs(), ref), what)
    else:
        ref = out0.double() + acc
        within(out, ref, elem_bound(mag, K, out0.double().abs()), what)
    assert_padding(buf, M, N, sent, what)
    return out
