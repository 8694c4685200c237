// univl_b200 — small HBM-bound utility kernels: bias-gradient column sums, fp32->bf16 weight casts, fills.
#include "common.cuh"

namespace univl {

__device__ __forceinline__ uint4 ld_nc_v4(const bf16* p) {
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
  return u;
}

// partial[row block][c] = sum_r x[r, c] over the block's rows (bf16 in, fp32); univl_colsum_bf16 adds the partials
// to out[c] in row-block order.  Block = 32 column-vectors (256 cols) x 8 row lanes.
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int rows, int cols,
                   int rows_per_block) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[8][257];
  const int cv = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 256 + cv * 8;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = min(rows, r_begin + rows_per_block);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  auto add8 = [&](const uint4& u) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      acc[2 * j] += f.x;
      acc[2 * j + 1] += f.y;
    }
  };
  if (c0 < cols) {
    const bf16* base = x + c0;
    if (c0 + 8 <= cols && (ld & 7) == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0) {
      // four independent 16-byte loads in flight per thread (the one-load loop was 85% long-scoreboard stalls)
      int r = r_begin + rl;
      for (; r + 24 < r_end; r += 32) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = ld_nc_v4(base + (long long)(r + 8 * k) * ld);
#pragma unroll
        for (int k = 0; k < 4; ++k) add8(u[k]);
      }
      for (; r < r_end; r += 8) add8(ld_nc_v4(base + (long long)r * ld));
    } else {
      for (int r = r_begin + rl; r < r_end; r += 8) {
        const bf16* p = base + (long long)r * ld;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (c0 + j < cols) acc[j] += __bfloat162float(p[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][cv * 8 + j] = acc[j];
  __syncthreads();
  const int e = threadIdx.x;
  const int c = blockIdx.x * 256 + e;
  if (c < cols) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][e];
    out[(long long)blockIdx.y * cols + c] = t;  // this row block's partial (partials_reduce sums them in order)
  }
}

__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n && (reinterpret_cast<uintptr_t>(src + i) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst + i) & 15) == 0) {
      const float4 a = *reinterpret_cast<const float4*>(src + i);
      const float4 b = *reinterpret_cast<const float4*>(src + i + 4);
      uint4 u;
      u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
      u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
      *reinterpret_cast<uint4*>(dst + i) = u;
    } else {
      for (long long j = i; j < n && j < i + 8; ++j) dst[j] = __float2bfloat16(src[j]);
    }
  }
}

// table[t] = {src pointer, dst pointer, element count}; grid.y walks the table
__global__ void __launch_bounds__(256)
multi_cast_kernel(const unsigned long long* __restrict__ table) {
  const float* src = reinterpret_cast<const float*>(table[3 * blockIdx.y]);
  bf16* dst = reinterpret_cast<bf16*>(table[3 * blockIdx.y + 1]);
  const long long n = (long long)table[3 * blockIdx.y + 2];
  const long long stride = (long long)gridDim.x * blockDim.x * 8;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n && (reinterpret_cast<uintptr_t>(src + i) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst + i) & 15) == 0) {
      const float4 a = *reinterpret_cast<const float4*>(src + i);
      const float4 b = *reinterpret_cast<const float4*>(src + i + 4);
      uint4 u;
      u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
      u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
      *reinterpret_cast<uint4*>(dst + i) = u;
    } else {
      for (long long j = i; j < n && j < i + 8; ++j) dst[j] = __float2bfloat16(src[j]);
    }
  }
}

// elementwise bf16 helpers: mode 0 out = dy * gelu_erf'(x) ; 1 out = tanh(x) ; 2 out = dy * (1 - y^2) with y = x
__global__ void __launch_bounds__(256)
eltwise_bf16_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x, bf16* __restrict__ out, long long n,
                    int mode) {
  const long long stride = (long long)gridDim.x * blockDim.x * 2;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += stride) {
    const bool pair = i + 1 < n;
    const float x0 = __bfloat162float(x[i]), x1 = pair ? __bfloat162float(x[i + 1]) : 0.f;
    const float d0 = dy ? __bfloat162float(dy[i]) : 0.f, d1 = (dy && pair) ? __bfloat162float(dy[i + 1]) : 0.f;
    float o0, o1;
    if (mode == 0) { o0 = d0 * gelu_erf_grad(x0); o1 = d1 * gelu_erf_grad(x1); }
    else if (mode == 1) { o0 = tanhf(x0); o1 = tanhf(x1); }
    else if (mode == 3) { o0 = gelu_erf(x0); o1 = gelu_erf(x1); }
    else { o0 = d0 * (1.f - x0 * x0); o1 = d1 * (1.f - x1 * x1); }
    out[i] = __float2bfloat16(o0);
    if (pair) out[i + 1] = __float2bfloat16(o1);
  }
}

__global__ void __launch_bounds__(256) fill_f32_kernel(float* __restrict__ p, float v, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

__global__ void rng_advance_kernel(unsigned long long* state) { state[1] += 1; }

}  // namespace univl

using namespace univl;

extern "C" int univl_rng_advance(unsigned long long* rng_state, void* stream) {
  UNIVL_CHECK_ARG(rng_state != nullptr, "rng_advance: null state");
  rng_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(rng_state);
  UNIVL_CHECK_LAUNCH("rng_advance");
  return UNIVL_OK;
}

extern "C" int univl_colsum_bf16(const void* x, long long ld, float* out, int rows, int cols, void* stream) {
  UNIVL_CHECK_ARG(x && out && rows >= 0 && cols > 0, "colsum: bad arguments");
  if (rows == 0) return UNIVL_OK;
  const int col_blocks = (cols + 255) / 256;
  int row_blocks = (device_sms() * 4 + col_blocks - 1) / col_blocks;
  if (row_blocks > (rows + 63) / 64) row_blocks = (rows + 63) / 64;
  if (row_blocks < 1) row_blocks = 1;
  const int rpb = (rows + row_blocks - 1) / row_blocks;
  row_blocks = (rows + rpb - 1) / rpb;
  float* part;
  if (int rc = scratch_alloc((void**)&part, (size_t)row_blocks * cols * sizeof(float), (cudaStream_t)stream)) return rc;
  launch_kernel(colsum_bf16_kernel, dim3(col_blocks, row_blocks), dim3(256), 0, (cudaStream_t)stream, (const bf16*)x, ld,
                part, rows, cols, rpb);
  UNIVL_CHECK_LAUNCH("colsum_bf16");
  return partials_reduce(part, row_blocks, 1, cols, out, cols, (cudaStream_t)stream);
}

extern "C" int univl_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream) {
  UNIVL_CHECK_ARG(src && dst && n >= 0, "cast: bad arguments");
  if (n == 0) return UNIVL_OK;
  long long blocks = (n + 2047) / 2048;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  cast_f32_bf16_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(src, (bf16*)dst, n);
  UNIVL_CHECK_LAUNCH("cast_f32_to_bf16");
  return UNIVL_OK;
}

namespace univl {
// dst(fp32) = src(bf16): the gradient payload coming back from a bf16 all-reduce (univl_b200/ddp.py)
__global__ void __launch_bounds__(256) cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long n8 = n >> 3;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(src + i * 8);
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    *reinterpret_cast<float4*>(dst + i * 8) = make_float4(a.x, a.y, b.x, b.y);
    *reinterpret_cast<float4*>(dst + i * 8 + 4) = make_float4(c.x, c.y, d.x, d.y);
  }
  if (blockIdx.x == 0)
    for (long long i = n8 * 8 + threadIdx.x; i < n; i += blockDim.x) dst[i] = __bfloat162float(src[i]);
}
}  // namespace univl

extern "C" int univl_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream) {
  UNIVL_CHECK_ARG(src && dst && n >= 0, "cast: bad arguments");
  UNIVL_CHECK_ARG(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0, "cast_bf16_to_f32: 16-byte alignment");
  if (n == 0) return UNIVL_OK;
  long long blocks = (n + 2047) / 2048;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  cast_bf16_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const bf16*)src, dst, n);
  UNIVL_CHECK_LAUNCH("cast_bf16_to_f32");
  return UNIVL_OK;
}

// device table of n_tensors x {src, dst, count} (uint64 each); one launch refreshes every bf16 weight copy
extern "C" int univl_multi_cast_f32_to_bf16(const unsigned long long* device_table, int n_tensors, int blocks_per_tensor,
                                            void* stream) {
  UNIVL_CHECK_ARG(device_table && n_tensors >= 0 && blocks_per_tensor > 0, "multi_cast: bad arguments");
  if (n_tensors == 0) return UNIVL_OK;
  UNIVL_CHECK_ARG(n_tensors <= 65535, "multi_cast: too many tensors");
  multi_cast_kernel<<<dim3(blocks_per_tensor, n_tensors), 256, 0, (cudaStream_t)stream>>>(device_table);
  UNIVL_CHECK_LAUNCH("multi_cast_f32_to_bf16");
  return UNIVL_OK;
}

static int launch_eltwise(const void* dy, const void* x, void* out, long long n, int mode, void* stream) {
  if (n == 0) return UNIVL_OK;
  long long blocks = (n + 511) / 512;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  eltwise_bf16_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const bf16*)dy, (const bf16*)x, (bf16*)out, n,
                                                                     mode);
  UNIVL_CHECK_LAUNCH("eltwise_bf16");
  return UNIVL_OK;
}
extern "C" int univl_gelu_bwd_bf16(const void* dy, const void* pre, void* out, long long n, void* stream) {
  UNIVL_CHECK_ARG(dy && pre && out && n >= 0, "gelu_bwd: bad arguments");
  return launch_eltwise(dy, pre, out, n, 0, stream);
}
extern "C" int univl_gelu_fwd_bf16(const void* x, void* out, long long n, void* stream) {
  UNIVL_CHECK_ARG(x && out && n >= 0, "gelu_fwd: bad arguments");
  return launch_eltwise(nullptr, x, out, n, 3, stream);
}
extern "C" int univl_tanh_fwd_bf16(const void* x, void* out, long long n, void* stream) {
  UNIVL_CHECK_ARG(x && out && n >= 0, "tanh_fwd: bad arguments");
  return launch_eltwise(nullptr, x, out, n, 1, stream);
}
extern "C" int univl_tanh_bwd_bf16(const void* dy, const void* y, void* out, long long n, void* stream) {
  UNIVL_CHECK_ARG(dy && y && out && n >= 0, "tanh_bwd: bad arguments");
  return launch_eltwise(dy, y, out, n, 2, stream);
}

extern "C" int univl_fill_f32(float* p, float value, long long n, void* stream) {
  UNIVL_CHECK_ARG(p && n >= 0, "fill: bad arguments");
  if (n == 0) return UNIVL_OK;
  if (value == 0.0f) {  // gradient-buffer clears (677 MB per step): the runtime's memset path, graph-capturable
    cudaError_t e = cudaMemsetAsync(p, 0, (size_t)n * sizeof(float), (cudaStream_t)stream);
    if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "fill memset: %s", cudaGetErrorString(e));
    return UNIVL_OK;
  }
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 16) blocks = device_sms() * 16;
  fill_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(p, value, n);
  UNIVL_CHECK_LAUNCH("fill_f32");
  return UNIVL_OK;
}
