"""Torch statements of the FP8 scaling rule (csrc/fp8.cuh) and the per-element bounds of the block-scaled FP8 GEMM
(csrc/gemm_fp8.cu), shared by tests/test_gpu_fp8_eval.py and the stage-by-stage evaluation walk in
tests/eval_check.py."""
import torch

E4M3 = torch.float8_e4m3fn


def ref_scale(amax):
    """2^ceil(log2(amax / 448)) from the bits of the fp32 quotient, at least 2^-126; 1 for amax == 0"""
    b = (amax.float() / 448.0).view(torch.int32)
    e = ((b >> 23) & 0xFF) - 127 + ((b & 0x7FFFFF) != 0).int()
    s = ((e.clamp(min=-126) + 127) << 23).int().view(torch.float32)
    return torch.where(amax > 0, s, torch.ones_like(s))


def ref_codes(x, s):
    """x / s rounded to nearest even e4m3, saturated (torch's cast turns values above 448 into NaN: clamp first)"""
    inv = ((254 << 23) - s.view(torch.int32)).view(torch.float32)  # 1 / s, exact
    return (x.float() * inv).clamp(-448.0, 448.0).to(E4M3)


def quant_rows(x):
    """quantize_e4m3_rows as the rule states it: bf16 [M, K] -> (e4m3 [M, K], fp32 scales [K/128, M])"""
    M, K = x.shape
    xf = x.float().view(M, K // 128, 128)
    s = ref_scale(xf.abs().amax(-1))
    return ref_codes(xf, s[..., None]).view(M, K), s.t().contiguous()


def quant_blocks(w):
    """quantize_e4m3_blocks as the rule states it: fp32 [N, K] -> (e4m3 [N, K], fp32 scales [N/128, K/128])"""
    N, K = w.shape
    blocks = w.float().view(N // 128, 128, K // 128, 128)
    s = ref_scale(blocks.abs().amax(dim=(1, 3)))
    return ref_codes(blocks, s[:, None, :, None]).view(N, K), s


def deq_rows(q, s):
    """e4m3 [M, K] with scales [K/128, M] -> fp64"""
    return q.double() * s.t().double().repeat_interleave(128, dim=1)


def deq_blocks(q, s):
    """e4m3 [N, K] with scales [N/128, K/128] -> fp64"""
    return q.double() * s.double().repeat_interleave(128, dim=0).repeat_interleave(128, dim=1)


# Bound per element.  The products of e4m3 values are exact in fp32; what is not exact is the tensor cores' sum of a
# K block's 128 products, whose precision Hopper does not document for 8-bit inputs, and the fp32 promotion of each
# block.  We bound both together by ACC * sum_k |a_k b_k| (the absolute product sum, fp64) and measure it.  The bf16
# output adds at most half an ulp, 2^-8 of the value.  ACC = 2^-9 is what the checker needs to be useful: a dropped K
# block or a wrong block scale moves an element by a block's signed sum, about sqrt(128) / K of the absolute sum for
# random operands, several times the bound.  Measured on an H100 (tests/test_gpu_fp8_eval.py prints both): max |err| /
# sum_k |a_k b_k| is 2.4e-3 at K = 768 and 1.1e-3 at K = 3072 for 300 rows, 5e-4 for one row, most of it the bf16
# rounding of the output.  What exceeds that rounding, max(|err| - 2^-8 |ref|, 0) / sum_k |a_k b_k| (the most the
# accumulation can be blamed for), is 5e-6 to 7e-5, 28 or more times below ACC.
ACC = 2.0 ** -9


def bf16_out_bound(ref, absref):
    """the written bound of the bf16 epilogue: 2^-8 (|ref| + ACC absref) + ACC absref"""
    acc = ACC * absref
    return 2.0 ** -8 * (ref.abs() + acc) + acc


def bf16_out_ok(out, ref, absref):
    """the written bound for the bf16 epilogue; -> (ok, max of |err| / absolute product sum)"""
    err = (out.double() - ref).abs()
    ok = bool((err <= bf16_out_bound(ref, absref)).all())
    beyond = float(((err - 2.0 ** -8 * ref.abs()).clamp(min=0) / absref).max())
    print("  max |err| / sum|a b| beyond the bf16 rounding of the output: %.3g (ACC = %.3g)" % (beyond, ACC))
    return ok, float((err / absref).max())


def gelu_e4m3_bound(g, absref, hs):
    """bound of the dequantized e4m3 output of the GELU epilogue against g = gelu(ref): the pre-activation error
    through gelu_erf (slope at most 1.13), then the e4m3 rounding of the result: half an ulp, 2^-4 of the value in
    e4m3's normal range, and half the subnormal spacing, 2^-10 of the scale, below it.  hs: the output scales
    [N/128, M]."""
    ev = 1.13 * ACC * absref + 1e-6 * (g.abs() + 1e-30)
    return 2.0 ** -4 * (g.abs() + ev) + ev + 2.0 ** -10 * hs.t().double().repeat_interleave(128, dim=1)
