// univl_b200 — fused multi-tensor BertAdam over flat fp32 buffers (SURVEY.md §8f#1).  HBM-bound: one read of
// p/g/m/v, one write of p/m/v plus the bf16 weight copy the GEMMs consume — 3 launches for ~300 tensors instead
// of the reference's Python loop of ~10 launches per tensor.
//
// Reference semantics restated (modules/optimization.py:103-167, driver main_task_retrieval.py:347):
//   driver : clip_grad_norm_(all parameters, 1.0)             -> g *= min(1, 1 / (||g||_all + 1e-6))
//   step   : per tensor clip_grad_norm_(p, max_grad_norm)     -> g *= min(1, max / (||g_t|| + 1e-6))
//            m = b1 m + (1-b1) g ;  v = b2 v + (1-b2) g^2     (NO bias correction)
//            update = m / (sqrt(v) + e) + weight_decay * p    (e OUTSIDE the sqrt, decoupled decay)
//            p -= lr * schedule(step / t_total, warmup) * update ;  step += 1
//   warmup_linear(x, w) = x / w if x < w else max((x - 1) / (w - 1), 0)      (optimization.py:37-43)
// The step counter lives in device memory so the whole update is CUDA-graph capturable.  It is ONE counter for all
// tensors, where the reference keeps a `step` per parameter and advances it only when that parameter has a gradient:
// a tensor that is skipped on some steps (below) is scheduled here at the optimizer's step count, in the reference at
// its own, smaller one.  Both agree whenever every tensor receives a gradient on every step.
#include "common.cuh"

namespace univl {

struct AdamSeg {  // one per CHUNK of a tensor (<= 64K elements: one CTA each), 32 bytes
  long long offset;
  int count;
  int tensor;  // index into the per-tensor sum-of-squares array
  float lr;
  float weight_decay;
  float pad0, pad1;
};

struct AdamCfg {
  float b1, b2, eps;
  float max_grad_norm;     // per-tensor clip (<= 0 disables)
  float global_clip_norm;  // all-parameter clip (<= 0 disables)
  float warmup;            // fraction of t_total, < 0 = none
  long long t_total;       // < 0 = constant lr
  float grad_scale;        // e.g. 1 / world_size after a sum all-reduce
};

// gradients arrive as fp32 (the buffer backward accumulates into) or as the bf16 all-reduce payload (univl_b200/ddp.py),
// which the optimizer then reads directly instead of through an expanded fp32 copy
__device__ __forceinline__ float4 load_grad4(const float* g, long long e) {
  return *reinterpret_cast<const float4*>(g + e);
}
__device__ __forceinline__ float4 load_grad4(const bf16* g, long long e) {
  const uint2 u = *reinterpret_cast<const uint2*>(g + e);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float load_grad(const float* g, long long e) { return g[e]; }
__device__ __forceinline__ float load_grad(const bf16* g, long long e) { return __bfloat162float(g[e]); }

template <typename G>
__global__ void __launch_bounds__(256)
adam_sumsq_kernel(const G* __restrict__ g, const AdamSeg* __restrict__ segs, float* __restrict__ part,
                  float grad_scale) {
  __shared__ float red[8];
  const AdamSeg s = segs[blockIdx.x];
  float acc = 0.f;
  // OR of the gradients' bits: some element is nonzero iff the OR has a magnitude bit set (-0 counts as zero).  A bit
  // test, not `x != 0.f`: under --use_fast_math comparisons flush denormals, and a denormal gradient is a gradient.
  unsigned bits = 0u;
  for (int i = threadIdx.x * 4; i < s.count; i += blockDim.x * 4) {
    if (i + 4 <= s.count) {
      const float4 x = load_grad4(g, s.offset + i);
      acc += (x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w) * grad_scale * grad_scale;
      bits |= __float_as_uint(x.x) | __float_as_uint(x.y) | __float_as_uint(x.z) | __float_as_uint(x.w);
    } else {
      for (int j = i; j < s.count; ++j) {
        const float x = load_grad(g, s.offset + j);
        acc += x * x * grad_scale * grad_scale;
        bits |= __float_as_uint(x);
      }
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  const int any_nz = __syncthreads_or((bits & 0x7fffffffu) != 0u);
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    // this chunk's share; adam_tensor_sums_kernel adds a tensor's chunks in order.  A chunk with a nonzero gradient
    // whose squares all flushed stores -0: adding it changes no sum, and its sign bit still says "has a gradient".
    part[blockIdx.x] = (any_nz && t == 0.f) ? -0.f : t;
  }
}

// per-chunk sums of squares -> sumsq[tensor], each tensor's chunks added in chunk order; tensor_nz[tensor] = some
// chunk of it has a nonzero gradient (a partial that is not +0)
__global__ void __launch_bounds__(256)
adam_tensor_sums_kernel(const float* __restrict__ part, const AdamSeg* __restrict__ segs, int n_chunks,
                        float* __restrict__ sumsq, int* __restrict__ tensor_nz, int n_tensors) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n_tensors) return;
  float t = 0.f;
  unsigned nz = 0u;
  for (int c = 0; c < n_chunks; ++c)
    if (segs[c].tensor == i) {
      const float x = part[c];
      t += x;
      nz |= __float_as_uint(x);
    }
  sumsq[i] = t;
  tensor_nz[i] = nz != 0u;
}

// sumsq[n_tensors] -> sumsq[n_tensors] holds the total
__global__ void adam_total_kernel(float* __restrict__ sumsq, int n_tensors) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n_tensors; i += blockDim.x) acc += sumsq[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    sumsq[n_tensors] = t;
  }
}

template <typename G>
__global__ void __launch_bounds__(256)
adam_update_kernel(float* __restrict__ p, const G* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                   bf16* __restrict__ p_bf16, const AdamSeg* __restrict__ segs, const float* __restrict__ sumsq,
                   const int* __restrict__ tensor_nz, int n_tensors, const long long* __restrict__ step,
                   AdamCfg cfg) {
  const AdamSeg s = segs[blockIdx.x];
  // a tensor whose gradient is identically zero received none this step (unused poolers etc.): the reference
  // skips parameters with `p.grad is None` entirely — no moment update, no weight decay (optimization.py:115-116).
  // Decided from the nonzero flags, not from sumsq == 0: squares below the fp32 normal range flush to zero (fast-math
  // FTZ), so gradients under ~1e-19 in magnitude sum to 0 yet must still move the moments and apply weight decay.
  if (!tensor_nz[s.tensor]) return;
  float cg = 1.f;
  if (cfg.global_clip_norm > 0.f) cg = fminf(1.f, cfg.global_clip_norm / (sqrtf(sumsq[n_tensors]) + 1e-6f));
  float ct = 1.f;
  if (cfg.max_grad_norm > 0.f) ct = fminf(1.f, cfg.max_grad_norm / (cg * sqrtf(sumsq[s.tensor]) + 1e-6f));
  const float gmul = cfg.grad_scale * cg * ct;
  float sched = 1.f;
  if (cfg.t_total > 0) {
    const float x = (float)((double)(*step) / (double)cfg.t_total);
    sched = (cfg.warmup >= 0.f && x < cfg.warmup) ? x / cfg.warmup : fmaxf((x - 1.f) / (cfg.warmup - 1.f), 0.f);
  }
  const float lr = s.lr * sched;
  // chunk offsets are multiples of 64 elements: 16-byte vector accesses are aligned
  for (int i = threadIdx.x * 4; i < s.count; i += blockDim.x * 4) {
    const long long e = s.offset + i;
    if (i + 4 <= s.count) {
      const float4 g4 = load_grad4(g, e);
      float4 m4 = *reinterpret_cast<const float4*>(m + e);
      float4 v4 = *reinterpret_cast<const float4*>(v + e);
      float4 p4 = *reinterpret_cast<const float4*>(p + e);
      const float gg[4] = {g4.x * gmul, g4.y * gmul, g4.z * gmul, g4.w * gmul};
      float mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w}, pp[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mm[j] = cfg.b1 * mm[j] + (1.f - cfg.b1) * gg[j];
        vv[j] = cfg.b2 * vv[j] + (1.f - cfg.b2) * gg[j] * gg[j];
        pp[j] -= lr * (mm[j] / (sqrtf(vv[j]) + cfg.eps) + s.weight_decay * pp[j]);
      }
      *reinterpret_cast<float4*>(m + e) = make_float4(mm[0], mm[1], mm[2], mm[3]);
      *reinterpret_cast<float4*>(v + e) = make_float4(vv[0], vv[1], vv[2], vv[3]);
      *reinterpret_cast<float4*>(p + e) = make_float4(pp[0], pp[1], pp[2], pp[3]);
      if (p_bf16 != nullptr) {
        uint2 u;
        u.x = pack_bf16x2(pp[0], pp[1]);
        u.y = pack_bf16x2(pp[2], pp[3]);
        *reinterpret_cast<uint2*>(p_bf16 + e) = u;
      }
    } else {
      for (int j = i; j < s.count; ++j) {
        const long long ee = s.offset + j;
        const float gr = load_grad(g, ee) * gmul;
        const float mm = cfg.b1 * m[ee] + (1.f - cfg.b1) * gr;
        const float vv = cfg.b2 * v[ee] + (1.f - cfg.b2) * gr * gr;
        float pp = p[ee];
        pp -= lr * (mm / (sqrtf(vv) + cfg.eps) + s.weight_decay * pp);
        m[ee] = mm; v[ee] = vv; p[ee] = pp;
        if (p_bf16 != nullptr) p_bf16[ee] = __float2bfloat16(pp);
      }
    }
  }
}

__global__ void adam_step_inc_kernel(long long* step) { *step += 1; }

}  // namespace univl

using namespace univl;

// One optimizer step over flat buffers.  segs: device array of n_chunks {int64 offset, int32 count, int32 tensor,
// float lr, float weight_decay, -, -} — one CTA per chunk (chunks of <= 64K elements, offsets multiples of 64);
// scratch: n_tensors + 1 floats (left holding each tensor's and the total sum of squares of the scaled gradients);
// step: device int64 (incremented).  p_bf16 (same element offsets as p) may be null.
template <typename G>
static int adam_step(float* p, const G* g, float* m, float* v, void* p_bf16, const void* segs, int n_chunks,
                     int n_tensors, float* scratch, long long* step, const AdamCfg& cfg, void* stream) {
  UNIVL_CHECK_ARG(p && g && m && v && segs && scratch && step, "bert_adam_step: null pointer");
  UNIVL_CHECK_ARG(n_tensors > 0 && n_chunks >= n_tensors, "bert_adam_step: bad tensor / chunk count");
  cudaStream_t st = (cudaStream_t)stream;
  const AdamSeg* s = reinterpret_cast<const AdamSeg*>(segs);
  // one allocation: per-chunk sums [n_chunks], then per-tensor "has a gradient" flags [n_tensors]
  float* part;
  if (int rc = scratch_alloc((void**)&part, (size_t)(n_chunks + n_tensors) * sizeof(float), st)) return rc;
  int* tensor_nz = reinterpret_cast<int*>(part + n_chunks);
  adam_sumsq_kernel<G><<<n_chunks, 256, 0, st>>>(g, s, part, cfg.grad_scale);
  adam_tensor_sums_kernel<<<(n_tensors + 255) / 256, 256, 0, st>>>(part, s, n_chunks, scratch, tensor_nz, n_tensors);
  adam_total_kernel<<<1, 256, 0, st>>>(scratch, n_tensors);
  adam_update_kernel<G><<<n_chunks, 256, 0, st>>>(p, g, m, v, (bf16*)p_bf16, s, scratch, tensor_nz, n_tensors, step,
                                                  cfg);
  cudaFreeAsync(part, st);
  adam_step_inc_kernel<<<1, 1, 0, st>>>(step);
  UNIVL_CHECK_LAUNCH("bert_adam_step");
  return UNIVL_OK;
}

extern "C" int univl_bert_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, const void* segs,
                                    int n_chunks, int n_tensors, float* scratch, long long* step, float b1, float b2,
                                    float eps, float max_grad_norm, float global_clip_norm, float warmup,
                                    long long t_total, float grad_scale, void* stream) {
  AdamCfg cfg{b1, b2, eps, max_grad_norm, global_clip_norm, warmup, t_total, grad_scale};
  return adam_step<float>(p, g, m, v, p_bf16, segs, n_chunks, n_tensors, scratch, step, cfg, stream);
}

// Same step with the gradients read from a bf16 buffer (same element offsets as p): the summed all-reduce payload of
// univl_b200.ddp.FlatGradReducer(compress="bf16"), consumed without expanding it to fp32 first.
extern "C" int univl_bert_adam_step_bf16grad(float* p, const void* g_bf16, float* m, float* v, void* p_bf16,
                                             const void* segs, int n_chunks, int n_tensors, float* scratch,
                                             long long* step, float b1, float b2, float eps, float max_grad_norm,
                                             float global_clip_norm, float warmup, long long t_total,
                                             float grad_scale, void* stream) {
  AdamCfg cfg{b1, b2, eps, max_grad_norm, global_clip_norm, warmup, t_total, grad_scale};
  return adam_step<bf16>(p, reinterpret_cast<const bf16*>(g_bf16), m, v, p_bf16, segs, n_chunks, n_tensors, scratch,
                         step, cfg, stream);
}
