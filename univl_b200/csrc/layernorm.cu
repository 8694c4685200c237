// univl_b200 — fused (dropout + residual +) LayerNorm, forward and backward.  HBM-bound.
//
// Reference semantics (modules/until_module.py:49-53): y = gamma * (z - mean) / sqrt(var_biased + eps) + beta with
// eps = 1e-12 INSIDE the sqrt.  The fused forms cover
//   BertSelfOutput / BertOutput (modules/module_bert.py:207-211, :246-250):  y = LN(dropout(x) + residual)
//   embeddings (module_bert.py:143-145 etc.):                               y = dropout(LN(z))        (drop_mode 2)
//   prediction-head transform (module_bert.py:308-312) and NormalizeVideo (modeling.py:88-92, fp32 input).
// One warp owns one row at a time (cols <= 1024, cols % 256 == 0 -> 1..4 16-byte vectors per lane); all statistics are
// fp32 and two-pass over registers, exactly the reference's mean -> centred variance order.  Backward regenerates the
// dropout mask from (seed, stream) and accumulates dgamma / dbeta / dbias column sums in registers across the rows a
// warp walks, then reduces through shared memory into one partial row per CTA; partials_reduce adds the rows in CTA
// order.
#include "common.cuh"

namespace univl {

constexpr int LN_WARPS = 8;
constexpr int LN_MAX_VEC = 4;  // cols <= 1024

__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// raw (still packed) 8-element vectors: what a software-pipelined row loop keeps in flight for the NEXT row
template <typename T> struct Raw8;
template <> struct Raw8<bf16> { uint4 u; };
template <> struct Raw8<float> { float4 a, b; };
__device__ __forceinline__ void raw_load(const bf16* p, Raw8<bf16>& r) {
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.u.x), "=r"(r.u.y), "=r"(r.u.z), "=r"(r.u.w) : "l"(p));
}
__device__ __forceinline__ void raw_load(const float* p, Raw8<float>& r) {
  r.a = __ldg(reinterpret_cast<const float4*>(p));
  r.b = __ldg(reinterpret_cast<const float4*>(p + 4));
}
__device__ __forceinline__ void raw_unpack(const Raw8<bf16>& r, float (&v)[8]) {
  const uint32_t w[4] = {r.u.x, r.u.y, r.u.z, r.u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}
__device__ __forceinline__ void raw_unpack(const Raw8<float>& r, float (&v)[8]) {
  v[0] = r.a.x; v[1] = r.a.y; v[2] = r.a.z; v[3] = r.a.w;
  v[4] = r.b.x; v[5] = r.b.y; v[6] = r.b.z; v[7] = r.b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]);
  u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]);
  u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

struct DropCfg {
  int mode;  // 0 none, 1 on x before the residual add, 2 on the LayerNorm output
  uint32_t threshold;
  float scale;  // 1/(1-p)
  uint64_t seed, stream;
  const unsigned long long* rng;  // device {seed, epoch}: resolved at kernel entry so launches are graph-replayable
};
__device__ __forceinline__ DropCfg resolve_drop(DropCfg d) {
  if (d.mode != 0 && d.rng != nullptr) {
    d.seed = d.rng[0];
    d.stream += d.rng[1] << 20;
  }
  return d;
}

// keep bits of 8 consecutive elements starting at flat index idx0 (idx0 % 8 == 0): one Philox call
__device__ __forceinline__ uint32_t keep8_mask(const DropCfg& d, uint64_t idx0) {
  return dropout_keep8(d.seed, d.stream, idx0, d.threshold);
}

// The row loop is software-pipelined: the raw vectors of the warp's NEXT row are requested before the current row's
// reductions, so every warp always has a full row of loads in flight (the un-pipelined loop spent 67% of its issue
// slots stalled on the long scoreboard: r01 ncu capture, 2.85 TB/s).
template <typename TIn, int NVEC>
__global__ void __launch_bounds__(LN_WARPS * 32, NVEC <= 3 ? 3 : 2)
layernorm_fwd_kernel(const TIn* __restrict__ x, const bf16* __restrict__ res, const float* __restrict__ gamma,
                     const float* __restrict__ beta, bf16* __restrict__ y, float* __restrict__ mean_out,
                     float* __restrict__ rstd_out, int rows, float eps, DropCfg drop_in) {
  pdl_trigger();
  pdl_wait();
  const DropCfg drop = resolve_drop(drop_in);
  constexpr int cols = NVEC * 256;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_cols = 1.0f / (float)cols;
  const long long stride = (long long)gridDim.x * LN_WARPS;
  long long row = (long long)blockIdx.x * LN_WARPS + warp;
  Raw8<TIn> nx[NVEC];
  Raw8<bf16> nr[NVEC];
  if (row < rows) {
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const long long off = row * cols + (i * 32 + lane) * 8;
      raw_load(x + off, nx[i]);
      if (res != nullptr) raw_load(res + off, nr[i]);
    }
  }
  for (; row < rows; row += stride) {
    float z[NVEC][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      raw_unpack(nx[i], z[i]);
      if (drop.mode == 1) {
        const uint32_t keep = keep8_mask(drop, (uint64_t)row * cols + c);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[i][j] = ((keep >> j) & 1u) ? z[i][j] * drop.scale : 0.f;
      }
      if (res != nullptr) {
        float r[8];
        raw_unpack(nr[i], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[i][j] += r[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += z[i][j];
    }
    const long long next = row + stride;
    if (next < rows) {
#pragma unroll
      for (int i = 0; i < NVEC; ++i) {
        const long long off = next * cols + (i * 32 + lane) * 8;
        raw_load(x + off, nx[i]);
        if (res != nullptr) raw_load(res + off, nr[i]);
      }
    }
    const float mean = warp_sum(s) * inv_cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = z[i][j] - mean;
        q += d * d;
      }
    const float var = warp_sum(q) * inv_cols;
    const float rstd = 1.0f / sqrtf(var + eps);
    if (lane == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      float g[8], b[8], o[8];
      load8(gamma + c, g);
      load8(beta + c, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j] * ((z[i][j] - mean) * rstd) + b[j];
      if (drop.mode == 2) {
        const uint32_t keep = keep8_mask(drop, (uint64_t)row * cols + c);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = ((keep >> j) & 1u) ? o[j] * drop.scale : 0.f;
      }
      store8(y + row * cols + c, o);
    }
  }
}

template <typename TIn>
static void launch_ln_fwd(int grid, cudaStream_t st, const TIn* x, const bf16* res, const float* gamma,
                          const float* beta, bf16* y, float* mean, float* rstd, int rows, int cols, float eps,
                          DropCfg drop) {
  const dim3 g(grid), b(LN_WARPS * 32);
  switch (cols >> 8) {
    case 1: launch_kernel(layernorm_fwd_kernel<TIn, 1>, g, b, 0, st, x, res, gamma, beta, y, mean, rstd, rows, eps, drop); break;
    case 2: launch_kernel(layernorm_fwd_kernel<TIn, 2>, g, b, 0, st, x, res, gamma, beta, y, mean, rstd, rows, eps, drop); break;
    case 3: launch_kernel(layernorm_fwd_kernel<TIn, 3>, g, b, 0, st, x, res, gamma, beta, y, mean, rstd, rows, eps, drop); break;
    default: launch_kernel(layernorm_fwd_kernel<TIn, 4>, g, b, 0, st, x, res, gamma, beta, y, mean, rstd, rows, eps, drop); break;
  }
}

// Backward.  dz = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy_eff * gamma.
//   dx_res   (bf16, may be null): dz                       — gradient w.r.t. the residual input (and x when no dropout)
//   dx_dense (bf16, may be null): dz * keep/(1-p)          — gradient w.r.t. x under drop_mode 1
//   dgamma, dbeta (fp32), dbias (fp32, optional) += column sums of dx_dense (or dz), summed in a fixed order

// one 8-wide vector of the row: z = pre-LayerNorm value, d = effective upstream gradient, keep = dropout bit mask
template <typename TIn>
__device__ __forceinline__ void ln_bwd_load(const bf16* dy, const bf16* dy2, const TIn* x, const bf16* res,
                                            long long off, const DropCfg& drop, float (&z)[8], float (&d)[8],
                                            uint32_t& keep) {
  load8(x + off, z);
  keep = 0xffu;
  if (drop.mode != 0) keep = keep8_mask(drop, (uint64_t)off);
  if (drop.mode == 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] = ((keep >> j) & 1u) ? z[j] * drop.scale : 0.f;
  }
  if (res != nullptr) {
    float r[8];
    load8(res + off, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] += r[j];
  }
  load8(dy + off, d);
  if (dy2 != nullptr) {
    float d2[8];
    load8(dy2 + off, d2);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] += d2[j];
  }
  if (drop.mode == 2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = ((keep >> j) & 1u) ? d[j] * drop.scale : 0.f;
  }
}

// Single sweep: the normalised row and g = dy * gamma stay in registers between the statistics and the dz phase, so each
// element is loaded, unpacked and (under dropout) Philox-masked exactly once.  (The earlier two-sweep form re-read the
// L1-resident row and regenerated the mask: 68 issued instructions per element, issue-bound at 2.4 TB/s.)
// The three column-sum accumulators (dgamma, dbeta, dbias partials: 3 x cols floats per warp) live in shared memory,
// each warp read-modify-writing only its own slice with conflict-free 16-byte accesses; holding them in registers cost
// 72 registers per thread and capped the kernel at 12 warps per SM, latency-bound at 40% of the HBM roofline.
constexpr int LNB_WARPS = 4;
__device__ __forceinline__ void acc8_add(float* p, const float (&v)[8]) {
  float4 a = *reinterpret_cast<float4*>(p), b = *reinterpret_cast<float4*>(p + 4);
  a.x += v[0]; a.y += v[1]; a.z += v[2]; a.w += v[3];
  b.x += v[4]; b.y += v[5]; b.z += v[6]; b.w += v[7];
  *reinterpret_cast<float4*>(p) = a;
  *reinterpret_cast<float4*>(p + 4) = b;
}
template <typename TIn, int NVEC>
__global__ void __launch_bounds__(LNB_WARPS * 32, NVEC <= 3 ? 5 : 3)
layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ dy2, const TIn* __restrict__ x,
                     const bf16* __restrict__ res, const float* __restrict__ gamma, const float* __restrict__ mean_in,
                     const float* __restrict__ rstd_in, bf16* __restrict__ dx_res, bf16* __restrict__ dx_dense,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int rows,
                     DropCfg drop_in) {
  pdl_trigger();
  pdl_wait();
  const DropCfg drop = resolve_drop(drop_in);
  extern __shared__ __align__(16) float lnb_acc[];  // [LNB_WARPS][3][cols]
  constexpr int cols = NVEC * 256;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_cols = 1.0f / (float)cols;
  const bool emit = dx_res != nullptr || dx_dense != nullptr || dbias != nullptr;
  float* my = lnb_acc + warp * 3 * cols;
  for (int k = lane * 4; k < 3 * cols; k += 128) *reinterpret_cast<float4*>(my + k) = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncwarp();

  for (long long row = (long long)blockIdx.x * LNB_WARPS + warp; row < rows; row += (long long)gridDim.x * LNB_WARPS) {
    const float mean = mean_in[row], rstd = rstd_in[row];
    const float nm = -mean * rstd;
    float xh[NVEC][8], g[NVEC][8];
    uint32_t keep[NVEC];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      float d[8], gm[8], dh[8];
      ln_bwd_load(dy, dy2, x, res, row * cols + c, drop, xh[i], d, keep[i]);
      load8(gamma + c, gm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float h = fmaf(xh[i][j], rstd, nm);
        const float gg = d[j] * gm[j];
        s1 += gg;
        s2 = fmaf(gg, h, s2);
        dh[j] = d[j] * h;
        xh[i][j] = h;
        g[i][j] = gg;
      }
      acc8_add(my + c, dh);
      acc8_add(my + cols + c, d);
    }
    if (!emit) continue;  // parameter gradients only
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float a = -s1 * inv_cols * rstd, b = -s2 * inv_cols * rstd;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      float dz[8], dd[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dz[j] = fmaf(xh[i][j], b, fmaf(g[i][j], rstd, a));
        dd[j] = (drop.mode == 1) ? (((keep[i] >> j) & 1u) ? dz[j] * drop.scale : 0.f) : dz[j];
      }
      if (dbias != nullptr) acc8_add(my + 2 * cols + c, dd);
      if (dx_res != nullptr) store8(dx_res + row * cols + c, dz);
      if (dx_dense != nullptr && dx_dense != dx_res) store8(dx_dense + row * cols + c, dd);
    }
  }
  // column sums: add the LNB_WARPS slices, one partial row per column and CTA
  __syncthreads();
  for (int which = 0; which < 3; ++which) {
    float* dst = which == 0 ? dgamma : which == 1 ? dbeta : dbias;
    if (dst == nullptr) continue;
    for (int e = threadIdx.x; e < cols; e += LNB_WARPS * 32) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < LNB_WARPS; ++w) t += lnb_acc[(w * 3 + which) * cols + e];
      dst[(long long)blockIdx.x * cols + e] = t;  // this CTA's partial (partials_reduce sums them in order)
    }
  }
}

template <typename TIn>
static int launch_ln_bwd(int grid, cudaStream_t st, const bf16* dy, const bf16* dy2, const TIn* x, const bf16* res,
                         const float* gamma, const float* mean, const float* rstd, bf16* dx_res, bf16* dx_dense,
                         float* dgamma_out, float* dbeta_out, float* dbias_out, int rows, int cols, DropCfg drop) {
  const size_t smem = (size_t)LNB_WARPS * 3 * cols * sizeof(float);
  // parameter gradients: per-CTA partial rows, summed in CTA order after the kernel
  float* outs[3] = {dgamma_out, dbeta_out, dbias_out};
  float* parts[3] = {nullptr, nullptr, nullptr};
  for (int w = 0; w < 3; ++w)
    if (outs[w] != nullptr)
      if (int rc = scratch_alloc((void**)&parts[w], (size_t)grid * cols * sizeof(float), st)) return rc;
  float *dgamma = parts[0], *dbeta = parts[1], *dbias = parts[2];
  switch (cols >> 8) {
    case 1: launch_kernel(layernorm_bwd_kernel<TIn, 1>, dim3(grid), dim3(LNB_WARPS * 32), smem, st, dy, dy2, x, res, gamma, mean, rstd, dx_res, dx_dense, dgamma, dbeta, dbias, rows, drop); break;
    case 2: launch_kernel(layernorm_bwd_kernel<TIn, 2>, dim3(grid), dim3(LNB_WARPS * 32), smem, st, dy, dy2, x, res, gamma, mean, rstd, dx_res, dx_dense, dgamma, dbeta, dbias, rows, drop); break;
    case 3: launch_kernel(layernorm_bwd_kernel<TIn, 3>, dim3(grid), dim3(LNB_WARPS * 32), smem, st, dy, dy2, x, res, gamma, mean, rstd, dx_res, dx_dense, dgamma, dbeta, dbias, rows, drop); break;
    default: launch_kernel(layernorm_bwd_kernel<TIn, 4>, dim3(grid), dim3(LNB_WARPS * 32), smem, st, dy, dy2, x, res, gamma, mean, rstd, dx_res, dx_dense, dgamma, dbeta, dbias, rows, drop); break;
  }
  UNIVL_CHECK_LAUNCH("layernorm_bwd");
  for (int w = 0; w < 3; ++w)
    if (parts[w] != nullptr)
      if (int rc = partials_reduce(parts[w], grid, 1, cols, outs[w], cols, st)) return rc;
  return UNIVL_OK;
}

static int check_ln_shape(const char* what, int rows, int cols) {
  UNIVL_CHECK_ARG(rows >= 0 && cols > 0 && (cols % 256) == 0 && cols <= 256 * LN_MAX_VEC,
                  "%s: cols must be a multiple of 256 and <= %d (got rows=%d cols=%d)", what, 256 * LN_MAX_VEC, rows,
                  cols);
  return UNIVL_OK;
}

static DropCfg make_drop(int mode, float p, const unsigned long long* rng, unsigned long long stream) {
  DropCfg d;
  d.mode = (p > 0.f) ? mode : 0;
  d.threshold = dropout_threshold16(p);
  d.scale = (p > 0.f) ? 1.0f / (1.0f - p) : 1.0f;
  d.seed = 0;
  d.stream = stream;
  d.rng = rng;
  return d;
}

static int lnb_grid(int rows) {
  long long blocks = ((long long)rows + LNB_WARPS - 1) / LNB_WARPS;
  const long long cap = (long long)device_sms() * 5;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}
static int ln_grid(int rows) {
  long long blocks = ((long long)rows + LN_WARPS - 1) / LN_WARPS;
  const long long cap = (long long)device_sms() * 8;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace univl

using namespace univl;

// y = LN(dropout(x) + res) [drop_mode 1]  or  dropout(LN(x + res)) [drop_mode 2];  x, res, y bf16; stats fp32.
extern "C" int univl_layernorm_fwd(const void* x, const void* res, const float* gamma, const float* beta, void* y,
                                   float* mean, float* rstd, int rows, int cols, float eps, float p_drop,
                                   int drop_mode, const unsigned long long* rng_state,
                                   unsigned long long stream_id, void* stream) {
  if (int rc = check_ln_shape("layernorm_fwd", rows, cols)) return rc;
  UNIVL_CHECK_ARG(x && gamma && beta && y, "layernorm_fwd: null pointer");
  UNIVL_CHECK_ARG(p_drop == 0.f || rng_state != nullptr, "layernorm_fwd: dropout needs rng_state");
  UNIVL_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f && drop_mode >= 0 && drop_mode <= 2, "layernorm_fwd: bad dropout");
  if (rows == 0) return UNIVL_OK;
  launch_ln_fwd<bf16>(ln_grid(rows), (cudaStream_t)stream, (const bf16*)x, (const bf16*)res, gamma, beta, (bf16*)y, mean,
                      rstd, rows, cols, eps, make_drop(drop_mode, p_drop, rng_state, stream_id));
  UNIVL_CHECK_LAUNCH("layernorm_fwd");
  return UNIVL_OK;
}

extern "C" int univl_layernorm_bwd(const void* dy, const void* dy2, const void* x, const void* res,
                                   const float* gamma, const float* mean, const float* rstd, void* dx_res,
                                   void* dx_dense, float* dgamma, float* dbeta, float* dbias, int rows, int cols,
                                   float p_drop, int drop_mode, const unsigned long long* rng_state,
                                   unsigned long long stream_id, void* stream) {
  if (int rc = check_ln_shape("layernorm_bwd", rows, cols)) return rc;
  UNIVL_CHECK_ARG(dy && x && gamma && mean && rstd, "layernorm_bwd: null pointer");
  UNIVL_CHECK_ARG(p_drop == 0.f || rng_state != nullptr, "layernorm_bwd: dropout needs rng_state");
  UNIVL_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f && drop_mode >= 0 && drop_mode <= 2, "layernorm_bwd: bad dropout");
  if (rows == 0) return UNIVL_OK;
  return launch_ln_bwd<bf16>(lnb_grid(rows), (cudaStream_t)stream, (const bf16*)dy, (const bf16*)dy2, (const bf16*)x,
                             (const bf16*)res, gamma, mean, rstd, (bf16*)dx_res, (bf16*)dx_dense, dgamma, dbeta, dbias,
                             rows, cols, make_drop(drop_mode, p_drop, rng_state, stream_id));
}

// fp32 input rows (NormalizeVideo, reference modules/modeling.py:88-92): y(bf16) = LN(x_f32); no dropout.
extern "C" int univl_layernorm_f32_fwd(const float* x, const float* gamma, const float* beta, void* y, float* mean,
                                       float* rstd, int rows, int cols, float eps, void* stream) {
  if (int rc = check_ln_shape("layernorm_f32_fwd", rows, cols)) return rc;
  UNIVL_CHECK_ARG(x && gamma && beta && y, "layernorm_f32_fwd: null pointer");
  if (rows == 0) return UNIVL_OK;
  launch_ln_fwd<float>(ln_grid(rows), (cudaStream_t)stream, x, (const bf16*)nullptr, gamma, beta, (bf16*)y, mean, rstd,
                       rows, cols, eps, make_drop(0, 0.f, nullptr, 0));
  UNIVL_CHECK_LAUNCH("layernorm_f32_fwd");
  return UNIVL_OK;
}

// parameter gradients only (the video features are inputs, not activations)
extern "C" int univl_layernorm_f32_bwd(const void* dy, const float* x, const float* gamma, const float* mean,
                                       const float* rstd, float* dgamma, float* dbeta, int rows, int cols,
                                       void* stream) {
  if (int rc = check_ln_shape("layernorm_f32_bwd", rows, cols)) return rc;
  UNIVL_CHECK_ARG(dy && x && gamma && mean && rstd && dgamma && dbeta, "layernorm_f32_bwd: null pointer");
  if (rows == 0) return UNIVL_OK;
  return launch_ln_bwd<float>(lnb_grid(rows), (cudaStream_t)stream, (const bf16*)dy, nullptr, x, nullptr, gamma, mean,
                              rstd, nullptr, nullptr, dgamma, dbeta, nullptr, rows, cols, make_drop(0, 0.f, nullptr, 0));
}
