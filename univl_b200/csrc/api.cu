// univl_b200 — C-ABI plumbing shared by every kernel file: error strings and version.
#include "common.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

namespace univl {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("UNIVL_PDL");
    v = (e && e[0] == '1') ? 1 : 0;  // measured neutral on the FT-Align step (graph replay): opt-in
  }
  return v == 1;
}

// SMs a concurrently running collective kernel (NCCL) occupies while the kernels being enqueued run: persistent grids are
// sized to the SMs that are actually free, otherwise the CTAs that find no SM run as a second wave and double the time
// of every persistent kernel under the collective.  Read at enqueue time, so it is baked into captured graphs.
static int g_reserved_sms = 0;

int device_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0, n = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    sms = n;
  }
  return sms;
}

int usable_sms() {
  const int n = device_sms() - g_reserved_sms;
  return n < 8 ? 8 : n;
}

int scratch_alloc(void** p, size_t bytes, cudaStream_t st) {
  static bool pool_ready[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 64 && !pool_ready[dev]) {
    // keep freed scratch in the device's default pool instead of returning it at every synchronisation
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool_ready[dev] = true;
  }
  const cudaError_t e = cudaMallocAsync(p, bytes < 16 ? 16 : bytes, st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "scratch allocation of %zu bytes: %s", bytes, cudaGetErrorString(e));
  return UNIVL_OK;
}

// Every element's partial rows are added in row order, t = 0; t += row 0; t += row 1; ..., then dst += t: the same
// arithmetic, and so the same bits, as one thread walking the rows, on every launch and with any grid.  What is
// parallel is the reading.  A CTA owns 32 consecutive elements (a warp reads 128 contiguous bytes of a row); its 8
// warps load the rows in stages of 256 (32 loads in flight per lane) into a double-buffered shared-memory tile, and
// warp 0 adds each staged tile in row order while the next stage's loads are in flight.  The loads, not the serial
// adds, bound the time, and they no longer wait on each other.
constexpr int PR_WARPS = 8;
constexpr int PR_STAGE = 256;                      // rows per stage, PR_STAGE / PR_WARPS per lane
constexpr int PR_SMEM = 2 * PR_STAGE * 32 * 4;     // two staged tiles [PR_STAGE][32] fp32: 64 KB

__global__ void __launch_bounds__(PR_WARPS * 32)
partials_reduce_kernel(const float* __restrict__ part, int nparts, long long n, long long cols, float* __restrict__ dst,
                       long long ld) {
  extern __shared__ float pr_tile[];  // [2][PR_STAGE][32]
  constexpr int PER = PR_STAGE / PR_WARPS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long e = blockIdx.x * 32LL + lane;
  const bool ok = e < n;
  const int stages = (nparts + PR_STAGE - 1) / PR_STAGE;
  float v[PER];
  // stage s, row s * PR_STAGE + i * PR_WARPS + warp -> v[i]; rows past nparts are never added
  auto load = [&](int s) {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int k = s * PR_STAGE + i * PR_WARPS + warp;
      v[i] = ok && k < nparts ? __ldcs(part + (long long)k * n + e) : 0.f;
    }
  };
  if (stages > 0) load(0);
  float t = 0.f;
  for (int s = 0; s < stages; ++s) {
    // tile s & 1 was last read by warp 0 at stage s - 2, before it reached the barrier of stage s - 1
    float* tile = pr_tile + (s & 1) * PR_STAGE * 32;
#pragma unroll
    for (int i = 0; i < PER; ++i) tile[(i * PR_WARPS + warp) * 32 + lane] = v[i];
    __syncthreads();
    if (s + 1 < stages) load(s + 1);
    if (warp == 0) {
      const int kn = nparts - s * PR_STAGE < PR_STAGE ? nparts - s * PR_STAGE : PR_STAGE;
      for (int k = 0; k < kn; ++k) t += tile[k * 32 + lane];
    }
  }
  if (warp == 0 && ok) {
    const long long r = e / cols, c = e - r * cols;
    dst[r * ld + c] += t;
  }
}

static int partials_reduce_launch(const float* part, int nparts, long long rows, long long cols, float* dst, long long ld,
                                  cudaStream_t st) {
  const long long n = rows * cols;
  const long long blocks = n > 0 ? (n + 31) / 32 : 1;
  if (blocks > 0x7fffffffLL) return set_error(UNIVL_ERR_UNSUPPORTED, "partials_reduce: %lld elements", n);
  cudaError_t e = cudaFuncSetAttribute(partials_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PR_SMEM);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "partials_reduce smem attribute: %s", cudaGetErrorString(e));
  partials_reduce_kernel<<<(unsigned)blocks, PR_WARPS * 32, PR_SMEM, st>>>(part, nparts, n, cols, dst, ld);
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "partials_reduce launch: %s", cudaGetErrorString(e));
  return UNIVL_OK;
}

int partials_reduce(float* part, int nparts, long long rows, long long cols, float* dst, long long ld, cudaStream_t st) {
  const int rc = partials_reduce_launch(part, nparts, rows, cols, dst, ld, st);
  cudaFreeAsync(part, st);
  return rc;
}

}  // namespace univl

extern "C" int univl_set_reserved_sms(int n) {
  if (n < 0) return univl::set_error(UNIVL_ERR_ARG, "univl_set_reserved_sms: n = %d", n);
  univl::g_reserved_sms = n;
  return UNIVL_OK;
}
extern "C" int univl_partials_reduce(const float* part, int nparts, long long rows, long long cols, float* dst,
                                     long long ld, void* stream) {
  UNIVL_CHECK_ARG(part && dst && nparts >= 0 && rows >= 0 && cols > 0 && ld >= cols,
                  "partials_reduce: bad arguments nparts=%d rows=%lld cols=%lld ld=%lld", nparts, rows, cols, ld);
  return univl::partials_reduce_launch(part, nparts, rows, cols, dst, ld, (cudaStream_t)stream);
}
extern "C" const char* univl_last_error_string() { return univl::g_err; }
extern "C" int univl_abi_version() { return 1; }
