// univl_b200 — e4m3 quantizers for the FP8 GEMM's operands (block scaling rules in fp8.cuh).
//   rows:   bf16 activations [M, K] -> e4m3 [M, K] + one scale per (row, 128-column block), scales [K/128, M]
//   blocks: fp32 weights     [N, K] -> e4m3 [N, K] + one scale per 128 x 128 block,      scales [N/128, K/128]
#include "common.cuh"
#include "fp8.cuh"

namespace univl {

// one warp per (row, 128-column block): 4 columns per lane
__global__ void __launch_bounds__(256) quantize_rows_kernel(const bf16* __restrict__ x, long long ldx,
                                                            uint8_t* __restrict__ q, long long ldq,
                                                            float* __restrict__ scale, int M, int KB) {
  pdl_trigger();
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  pdl_wait();
  if (wid >= (long long)M * KB) return;  // whole warps
  const int row = (int)(wid / KB), kb = (int)(wid - (long long)row * KB);
  const int col = kb * 128 + lane * 4;
  const uint2 u = *reinterpret_cast<const uint2*>(x + row * ldx + col);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
  const float amax = warp_max(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
  const float s = e4m3_scale(amax);
  const float inv = e4m3_inv_scale(s);
  const uint32_t lo = e4m3x2(__fmul_rn(a.x, inv), __fmul_rn(a.y, inv));
  const uint32_t hi = e4m3x2(__fmul_rn(b.x, inv), __fmul_rn(b.y, inv));
  *reinterpret_cast<uint32_t*>(q + row * ldq + col) = lo | (hi << 16);
  if (lane == 0) scale[(long long)kb * M + row] = s;
}

// one CTA per 128 x 128 block: the block's amax, then its codes (the second pass reads the block from L1 / L2)
__global__ void __launch_bounds__(256) quantize_blocks_kernel(const float* __restrict__ w, long long ldw,
                                                              uint8_t* __restrict__ q, long long ldq,
                                                              float* __restrict__ scale, int KB) {
  __shared__ float red[8];
  pdl_trigger();
  const int nb = blockIdx.y, kb = blockIdx.x;
  const float* src = w + (long long)nb * 128 * ldw + kb * 128;
  uint8_t* dst = q + (long long)nb * 128 * ldq + kb * 128;
  const int t = threadIdx.x;
  const int c = (t & 31) * 4;  // a warp covers one row of 128 columns per step
  pdl_wait();
  float amax = 0.f;
  for (int r = t >> 5; r < 128; r += 8) {
    const float4 v = *reinterpret_cast<const float4*>(src + r * ldw + c);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  amax = warp_max(amax);
  if ((t & 31) == 0) red[t >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
  const float s = e4m3_scale(amax);
  const float inv = e4m3_inv_scale(s);
  for (int r = t >> 5; r < 128; r += 8) {
    const float4 v = *reinterpret_cast<const float4*>(src + r * ldw + c);
    const uint32_t lo = e4m3x2(__fmul_rn(v.x, inv), __fmul_rn(v.y, inv));
    const uint32_t hi = e4m3x2(__fmul_rn(v.z, inv), __fmul_rn(v.w, inv));
    *reinterpret_cast<uint32_t*>(dst + r * ldq + c) = lo | (hi << 16);
  }
  if (t == 0) scale[(long long)nb * KB + kb] = s;
}

}  // namespace univl

using namespace univl;

extern "C" int univl_quantize_e4m3_rows(const void* x, long long ldx, void* q, long long ldq, float* scale, int M,
                                        int K, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UNIVL_CHECK_ARG(M > 0 && K > 0, "univl_quantize_e4m3_rows: empty problem M=%d K=%d", M, K);
  UNIVL_CHECK_ARG(K % 128 == 0, "univl_quantize_e4m3_rows: K=%d must be a multiple of 128", K);
  UNIVL_CHECK_ARG(x && q && scale, "univl_quantize_e4m3_rows: null input, output or scale");
  UNIVL_CHECK_ARG(ldx >= K && ldq >= K && (ldx % 4) == 0 && (ldq % 4) == 0,
                  "univl_quantize_e4m3_rows: ldx/ldq must be >= K and multiples of 4 (got %lld, %lld, K=%d)", ldx,
                  ldq, K);
  UNIVL_CHECK_ARG(((uintptr_t)x & 7) == 0 && ((uintptr_t)q & 3) == 0,
                  "univl_quantize_e4m3_rows: x must be 8-byte and q 4-byte aligned");
  const long long warps = (long long)M * (K / 128);
  const long long blocks = (warps + 7) / 8;
  UNIVL_CHECK_ARG(blocks <= 0x7fffffffLL, "univl_quantize_e4m3_rows: too many rows");
  cudaError_t e = launch_kernel(quantize_rows_kernel, dim3((unsigned)blocks), dim3(256), 0, stream,
                                reinterpret_cast<const bf16*>(x), ldx, reinterpret_cast<uint8_t*>(q), ldq, scale, M,
                                K / 128);
  if (e != cudaSuccess)
    return set_error(UNIVL_ERR_CUDA, "univl_quantize_e4m3_rows launch: %s", cudaGetErrorString(e));
  UNIVL_CHECK_LAUNCH("quantize_e4m3_rows");
  return UNIVL_OK;
}

extern "C" int univl_quantize_e4m3_blocks(const float* w, long long ldw, void* q, long long ldq, float* scale, int N,
                                          int K, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UNIVL_CHECK_ARG(N > 0 && K > 0, "univl_quantize_e4m3_blocks: empty problem N=%d K=%d", N, K);
  UNIVL_CHECK_ARG(N % 128 == 0 && K % 128 == 0, "univl_quantize_e4m3_blocks: N=%d and K=%d must be multiples of 128",
                  N, K);
  UNIVL_CHECK_ARG(w && q && scale, "univl_quantize_e4m3_blocks: null input, output or scale");
  UNIVL_CHECK_ARG(ldw >= K && ldq >= K && (ldw % 4) == 0 && (ldq % 4) == 0,
                  "univl_quantize_e4m3_blocks: ldw/ldq must be >= K and multiples of 4 (got %lld, %lld, K=%d)", ldw,
                  ldq, K);
  UNIVL_CHECK_ARG(((uintptr_t)w & 15) == 0 && ((uintptr_t)q & 3) == 0,
                  "univl_quantize_e4m3_blocks: w must be 16-byte and q 4-byte aligned");
  UNIVL_CHECK_ARG(N / 128 <= 65535, "univl_quantize_e4m3_blocks: N=%d too large", N);
  cudaError_t e = launch_kernel(quantize_blocks_kernel, dim3(K / 128, N / 128), dim3(256), 0, stream, w, ldw,
                                reinterpret_cast<uint8_t*>(q), ldq, scale, K / 128);
  if (e != cudaSuccess)
    return set_error(UNIVL_ERR_CUDA, "univl_quantize_e4m3_blocks launch: %s", cudaGetErrorString(e));
  UNIVL_CHECK_LAUNCH("quantize_e4m3_blocks");
  return UNIVL_OK;
}
