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

__global__ void __launch_bounds__(256)
partials_reduce_kernel(const float* __restrict__ part, int nparts, long long rows, long long cols, float* __restrict__ dst,
                       long long ld) {
  const long long n = rows * cols;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float t = 0.f;
    for (int k = 0; k < nparts; ++k) t += part[(long long)k * n + i];
    const long long r = i / cols, c = i - r * cols;
    dst[r * ld + c] += t;
  }
}

int partials_reduce(float* part, int nparts, long long rows, long long cols, float* dst, long long ld, cudaStream_t st) {
  const long long n = rows * cols;
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8LL) blocks = device_sms() * 8LL;
  if (blocks < 1) blocks = 1;
  partials_reduce_kernel<<<(int)blocks, 256, 0, st>>>(part, nparts, rows, cols, dst, ld);
  const cudaError_t e = cudaGetLastError();
  cudaFreeAsync(part, st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "partials_reduce launch: %s", cudaGetErrorString(e));
  return UNIVL_OK;
}

}  // namespace univl

extern "C" int univl_set_reserved_sms(int n) {
  if (n < 0) return univl::set_error(UNIVL_ERR_ARG, "univl_set_reserved_sms: n = %d", n);
  univl::g_reserved_sms = n;
  return UNIVL_OK;
}
extern "C" const char* univl_last_error_string() { return univl::g_err; }
extern "C" int univl_abi_version() { return 1; }
