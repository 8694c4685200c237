// univl_b200 — shared device helpers for the sm_90a kernels.
//
// Thin inline-PTX wrappers for the Hopper primitives the kernels use
// (mbarrier, TMA bulk-tensor copies, wgmma), plus small math and
// packing helpers.  Everything here is header-only and device-side except the
// error-string plumbing at the bottom.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace univl {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------
// error plumbing shared by all translation units (defined in api.cu)
// ----------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
int device_sms();        // SM count of the current device (api.cu)
int usable_sms();        // SM count minus univl_set_reserved_sms (api.cu)
// Deterministic cross-CTA sums: a kernel writes one partial row per contributor into stream-ordered scratch memory
// (cudaMallocAsync, capturable in CUDA graphs) instead of adding atomically; partials_reduce adds the rows to dst in
// contributor order and frees the scratch, so every run sums in the same order.  (api.cu)
int scratch_alloc(void** p, size_t bytes, cudaStream_t st);
// dst[r * ld + c] += sum over k in [0, nparts) of part[k * rows * cols + r * cols + c], k ascending; frees part
int partials_reduce(float* part, int nparts, long long rows, long long cols, float* dst, long long ld, cudaStream_t st);
#define UNIVL_OK 0
#define UNIVL_ERR_ARG -1
#define UNIVL_ERR_CUDA -2
#define UNIVL_ERR_UNSUPPORTED -3

#define UNIVL_CHECK_ARG(cond, ...)                                   \
  do {                                                               \
    if (!(cond)) return univl::set_error(UNIVL_ERR_ARG, __VA_ARGS__); \
  } while (0)

#define UNIVL_CHECK_LAUNCH(name)                                                          \
  do {                                                                                    \
    cudaError_t e__ = cudaGetLastError();                                                 \
    if (e__ != cudaSuccess)                                                               \
      return univl::set_error(UNIVL_ERR_CUDA, "%s launch: %s", name, cudaGetErrorString(e__)); \
  } while (0)

// ----------------------------------------------------------------------------
// programmatic dependent launch (PDL): every hot kernel is launched with the programmatic-stream-serialization
// attribute, calls pdl_trigger() on entry (the NEXT kernel's CTAs may become resident as soon as all of ours have
// started) and pdl_wait() before its first global-memory access (blocks until the previous kernel has completed and
// flushed).  Launch latency and per-CTA set-up of kernel N+1 overlap the tail of kernel N — the text / visual encoder
// layers are ~25 kernels of 5-15 us each.  Opt-in with UNIVL_PDL=1 (without the attribute the device calls are no-ops);
// measured neutral (1806 vs 1816 samples/s) under CUDA-graph replay, so it is off by default.
// ----------------------------------------------------------------------------
bool pdl_enabled();  // api.cu
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                        Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// ----------------------------------------------------------------------------
// generic helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// erf-GELU as the reference states it: x * 0.5 * (1 + erf(x / sqrt(2)))  (modules/until_module.py:28-33).
// erf is evaluated with Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, two orders below bf16 resolution) because the
// GEMM epilogue is instruction-bound: one MUFU.RCP + one MUFU.EX2 + a handful of FMAs instead of libdevice's branchy
// erff.  The same exponential exp(-x^2/2) serves the derivative's Gaussian term.
// Arranged for the fewest issue slots (11 FP + 2 MUFU forward, 15 + 2 for the derivative):
//   w(x) = 1 - Phi(|x|) = 0.5 * t * poly(t) * exp(-x^2/2),  t = 1 / (1 + p |x| / sqrt(2))      (A&S 7.1.26)
//   gelu(x)  = max(x, 0) - |x| * w(x)
//   gelu'(x) = Phi(x) + x * phi(x),   Phi(x) = x >= 0 ? 1 - w : w
__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// w = 1 - Phi(|x|) (in [0, 0.5]) and gauss = exp(-x^2 / 2)
__device__ __forceinline__ void erf_exp_terms(float x, float& w, float& gauss) {
  const float t = rcp_approx(fmaf(fabsf(x), 0.3275911f * 0.70710678118654752440f, 1.0f));
  gauss = ex2_approx((x * x) * (-0.5f * 1.44269504088896340736f));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  w = (poly * t) * gauss;
}
__device__ __forceinline__ float gelu_erf(float x) {
  float w, g;
  erf_exp_terms(x, w, g);
  return fmaf(-fabsf(x), w, fmaxf(x, 0.f));
}
// d/dx gelu_erf(x) = Phi(x) + x * phi(x)
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float w, g;
  erf_exp_terms(x, w, g);
  const float cdf = x >= 0.f ? 1.0f - w : w;
  return fmaf(x * 0.39894228040143267794f, g, cdf);
}

// ----------------------------------------------------------------------------
// Philox4x32-10 counter RNG (dropout masks are regenerated in backward from
// (seed, offset) — never stored).
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t ctr_hi, uint64_t ctr_lo) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32);
  uint32_t c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// Keep-mask for element `idx` of dropout stream (seed, stream): element idx uses
// 32 random bits: word (idx & 3) of philox(seed, stream, idx >> 2).
__device__ __forceinline__ bool dropout_keep(uint64_t seed, uint64_t stream, uint64_t idx,
                                             uint32_t keep_threshold) {
  const uint4 r = philox4x32(seed, stream, idx >> 2);
  const uint32_t w = (idx & 3) == 0 ? r.x : (idx & 3) == 1 ? r.y : (idx & 3) == 2 ? r.z : r.w;
  return w < keep_threshold;
}
// threshold such that P(keep) = 1 - p  (p in [0,1))
__host__ __device__ __forceinline__ uint32_t dropout_threshold(float p) {
  double keep = 1.0 - (double)p;
  if (keep >= 1.0) return 0xFFFFFFFFu;
  return (uint32_t)(keep * 4294967296.0);
}
// 16-bit variant: an element is kept iff its 16 random bits are < threshold16, so one Philox4x32 call (128 bits)
// decides 8 elements; P(keep) is exact to 2^-16, far below the sampling noise of any dropout mask.
__host__ __device__ __forceinline__ uint32_t dropout_threshold16(float p) {
  double keep = 1.0 - (double)p;
  if (keep >= 1.0) return 65536u;
  return (uint32_t)(keep * 65536.0 + 0.5);
}
// 16-bit word w (0..7) of a Philox output
__device__ __forceinline__ uint32_t philox_u16(const uint4& r, int w) {
  const uint32_t x = (w >> 1) == 0 ? r.x : (w >> 1) == 1 ? r.y : (w >> 1) == 2 ? r.z : r.w;
  return (w & 1) ? (x >> 16) : (x & 0xFFFFu);
}
// keep-mask (bit j = keep element idx0 + j) of 8 consecutive elements, idx0 % 8 == 0: ONE Philox call
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint64_t stream, uint64_t idx0, uint32_t thr16) {
  const uint4 r = philox4x32(seed, stream, idx0 >> 3);
  return ((r.x & 0xFFFFu) < thr16 ? 1u : 0u) | ((r.x >> 16) < thr16 ? 2u : 0u) | ((r.y & 0xFFFFu) < thr16 ? 4u : 0u) |
         ((r.y >> 16) < thr16 ? 8u : 0u) | ((r.z & 0xFFFFu) < thr16 ? 16u : 0u) | ((r.z >> 16) < thr16 ? 32u : 0u) |
         ((r.w & 0xFFFFu) < thr16 ? 64u : 0u) | ((r.w >> 16) < thr16 ? 128u : 0u);
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a pipeline bug must surface as a trap (launch failure), never as
// a hung GPU.  try_wait already suspends in hardware, so the spin count stays low
// in healthy runs; 1<<26 polls is many seconds.  No printf here: a function call inside the wgmma consumer loops makes
// ptxas serialise every wgmma (C7510), so the timeout is reported by the trap alone.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ----------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2D tiled loads into shared memory
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}


// ---- TMA stores (shared -> global) -----------------------------------------------------------------------------
// bulk tensor store / reduce of one staging box; coordinates {inner (column), outer (row)}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the most recent N bulk groups of this thread have finished READING their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------
// Hopper warpgroup MMA (wgmma) plumbing
// ----------------------------------------------------------------------------
// One lane of a fully converged warp (elect.sync), for the single-thread TMA issue of a producer warp.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving reads / writes of an accumulator across the asynchronous MMA region
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup (producer warpgroups give theirs to the MMA warpgroups)
template <int N>
__device__ __forceinline__ void regs_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void regs_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Shared-memory matrix descriptor of a 128B-swizzled operand (sm_90 GmmaDescriptor): start address, leading / stride
// byte offsets in 16-byte units, layout type 1 = SWIZZLE_128B.  K-major: SBO = 1024 (8 rows of 128 B), LBO unused.
// MN-major: LBO = distance between 64-element MN blocks, SBO = 1024 (8 k-rows of 128 B).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;  // layout_type = SWIZZLE_128B
  return d;
}

}  // namespace univl
