// univl_b200 — pooling, similarity and loss kernels (the "tail" of UniVL.forward).  All fp32 math.
//
//   masked mean pooling (+ L2 normalise)       reference modules/modeling.py:327-339, :386-388
//   text x video similarity matrix              reference modules/modeling.py:389
//   MaxMarginRankingLoss / CrossEn / MILNCELoss reference modules/until_module.py:182-251
//   cross pooler tanh + similarity_dense        reference modules/module_cross.py:281-287, modeling.py:371
//   CrossEntropyLoss(ignore_index=-1) on vocab logits and the MFM NCE   reference modules/modeling.py:253,273-297
// Every loss kernel also emits d(loss)/d(input) for an upstream gradient of 1; autograd's scalar is applied by
// univl_scale_f32 (reads the scalar from device memory — no host sync).
#include "common.cuh"

namespace univl {

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < nw; ++w) t += red[w];
  return t;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int w = 0; w < nw; ++w) t = fmaxf(t, red[w]);
  return t;
}

// ------------------------------------------------------------------------------------------------------------
// masked mean pooling
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
meanpool_fwd_kernel(const bf16* __restrict__ x, const long long* __restrict__ mask, float* __restrict__ out,
                    float* __restrict__ norm_out, int S, int H, int skip_first, int guard_zero, int l2norm) {
  __shared__ float red[32];
  const int n = blockIdx.x;
  float den = 0.f;
  for (int s = 0; s < S; ++s) den += (mask[(long long)n * S + s] != 0 && !(skip_first && s == 0)) ? 1.f : 0.f;
  if (guard_zero && den == 0.f) den = 1.f;
  float sq = 0.f;
  float u[4];
  int nc = 0;
  for (int c = threadIdx.x; c < H; c += blockDim.x, ++nc) {
    float acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const bool on = mask[(long long)n * S + s] != 0 && !(skip_first && s == 0);
      if (on) acc += __bfloat162float(x[((long long)n * S + s) * H + c]);
    }
    acc = acc / den;
    u[nc] = acc;
    sq += acc * acc;
  }
  float nrm = 1.f;
  if (l2norm) {
    nrm = fmaxf(sqrtf(block_sum(sq, red)), 1e-12f);  // F.normalize eps
  }
  if (threadIdx.x == 0 && norm_out) norm_out[n] = nrm;
  nc = 0;
  for (int c = threadIdx.x; c < H; c += blockDim.x, ++nc) out[(long long)n * H + c] = u[nc] / nrm;
}

__global__ void __launch_bounds__(256)
meanpool_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ norm,
                    const long long* __restrict__ mask, bf16* __restrict__ dx, int S, int H, int skip_first,
                    int guard_zero, int l2norm) {
  __shared__ float red[32];
  const int n = blockIdx.x;
  float den = 0.f;
  for (int s = 0; s < S; ++s) den += (mask[(long long)n * S + s] != 0 && !(skip_first && s == 0)) ? 1.f : 0.f;
  if (guard_zero && den == 0.f) den = 1.f;
  float dot = 0.f;
  if (l2norm)
    for (int c = threadIdx.x; c < H; c += blockDim.x) dot += y[(long long)n * H + c] * dy[(long long)n * H + c];
  if (l2norm) dot = block_sum(dot, red);
  const float nrm = l2norm ? norm[n] : 1.f;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float du = dy[(long long)n * H + c];
    if (l2norm) du = (du - y[(long long)n * H + c] * dot) / nrm;
    du /= den;
    for (int s = 0; s < S; ++s) {
      const bool on = mask[(long long)n * S + s] != 0 && !(skip_first && s == 0);
      dx[((long long)n * S + s) * H + c] = __float2bfloat16(on ? du : 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// sim = T V^T  (tiny)
// ------------------------------------------------------------------------------------------------------------
__global__ void sim_fwd_kernel(const float* __restrict__ t, const float* __restrict__ v, float* __restrict__ sim,
                               int Bt, int Bv, int H) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= Bt * Bv) return;
  const int i = gw / Bv, j = gw % Bv;
  float acc = 0.f;
  for (int c = lane; c < H; c += 32) acc += t[(long long)i * H + c] * v[(long long)j * H + c];
  acc = warp_sum(acc);
  if (lane == 0) sim[gw] = acc;
}
// dt[i,:] = sum_j dsim[i,j] v[j,:] ; dv[j,:] = sum_i dsim[i,j] t[i,:]
__global__ void sim_bwd_kernel(const float* __restrict__ dsim, const float* __restrict__ t,
                               const float* __restrict__ v, float* __restrict__ dt, float* __restrict__ dv, int Bt,
                               int Bv, int H) {
  const int r = blockIdx.x;
  if (r < Bt) {
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      float acc = 0.f;
      for (int j = 0; j < Bv; ++j) acc += dsim[(long long)r * Bv + j] * v[(long long)j * H + c];
      dt[(long long)r * H + c] = acc;
    }
  } else {
    const int j = r - Bt;
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      float acc = 0.f;
      for (int i = 0; i < Bt; ++i) acc += dsim[(long long)i * Bv + j] * t[(long long)i * H + c];
      dv[(long long)j * H + c] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// losses on a [B, B] similarity matrix (single CTA)
// ------------------------------------------------------------------------------------------------------------
// mean_ij w_ij * ( relu(m + s_ij - s_ii) + relu(m + s_ij - s_jj) ), diagonal included (until_module.py:245-251)
__global__ void __launch_bounds__(256)
maxmargin_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int B, float margin,
                 int n_pair, float w_same, float w_diff) {
  __shared__ float red[32];
  const float inv = 1.0f / ((float)B * (float)B);
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) dsim[e] = 0.f;
  __syncthreads();
  float acc = 0.f;
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
    const int i = e / B, j = e % B;
    const float w = (n_pair > 0) ? ((i / n_pair == j / n_pair) ? w_same : w_diff) : 1.f;
    const float s = sim[e];
    const float a = margin + s - sim[i * B + i];
    const float c = margin + s - sim[j * B + j];
    float gs = 0.f;
    if (a > 0.f) { acc += w * a; gs += w * inv; }
    if (c > 0.f) { acc += w * c; gs += w * inv; }
    dsim[e] = gs;
  }
  __syncthreads();
  // the diagonal s_kk appears in every term of row k (a) and column k (c): add those in a fixed order
  for (int k = threadIdx.x; k < B; k += blockDim.x) {
    const float skk = sim[k * B + k];
    float t = 0.f;
    for (int j = 0; j < B; ++j) {
      const float w = (n_pair > 0) ? ((k / n_pair == j / n_pair) ? w_same : w_diff) : 1.f;
      if (margin + sim[k * B + j] - skk > 0.f) t -= w * inv;
    }
    for (int i = 0; i < B; ++i) {
      const float w = (n_pair > 0) ? ((i / n_pair == k / n_pair) ? w_same : w_diff) : 1.f;
      if (margin + sim[i * B + k] - skk > 0.f) t -= w * inv;
    }
    dsim[k * B + k] += t;
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) *loss = acc * inv;
}

// -mean_i log_softmax(sim[i,:])[i]   (until_module.py:186-191)
__global__ void __launch_bounds__(256)
crossen_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int B) {
  __shared__ float red[32];
  float acc = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = warp; i < B; i += nw) {
    float m = -INFINITY;
    for (int j = lane; j < B; j += 32) m = fmaxf(m, sim[i * B + j]);
    m = warp_max(m);
    float l = 0.f;
    for (int j = lane; j < B; j += 32) l += expf(sim[i * B + j] - m);
    l = warp_sum(l);
    const float lse = m + logf(l);
    for (int j = lane; j < B; j += 32)
      dsim[i * B + j] = (expf(sim[i * B + j] - lse) - (i == j ? 1.f : 0.f)) / (float)B;
    if (lane == 0) acc += lse - sim[i * B + i];
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) *loss = acc / (float)B;
}

// MIL-NCE (until_module.py:201-221) on sim [N, N], N = bs * P.  For each picked row r = k*P + P/2:
//   loss_r = logsumexp_{all c}(row) - logsumexp_{c in pos(r)}(row),
//   row = [ sim[c, r] for c < N ] ++ [ sim[r, c] - 1e12 * same_block(r, c) for c < N ],  pos(r) = first half, same block.
__global__ void __launch_bounds__(256)
milnce_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int bs, int P) {
  __shared__ float red[32];
  const int N = bs * P;
  for (int e = threadIdx.x; e < N * N; e += blockDim.x) dsim[e] = 0.f;
  __syncthreads();
  float acc = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int k = warp; k < bs; k += nw) {
    const int r = k * P + P / 2;
    float m = -INFINITY, mp = -INFINITY;
    for (int c = lane; c < 2 * N; c += 32) {
      const bool first = c < N;
      const int cc = first ? c : c - N;
      const bool same = (cc / P) == k;
      const float x = first ? sim[cc * N + r] : sim[r * N + cc] + (same ? -1e12f : 0.f);
      m = fmaxf(m, x);
      if (first && same) mp = fmaxf(mp, x);
    }
    m = warp_max(m);
    mp = warp_max(mp);
    float l = 0.f, lp = 0.f;
    for (int c = lane; c < 2 * N; c += 32) {
      const bool first = c < N;
      const int cc = first ? c : c - N;
      const bool same = (cc / P) == k;
      const float x = first ? sim[cc * N + r] : sim[r * N + cc] + (same ? -1e12f : 0.f);
      l += expf(x - m);
      if (first && same) lp += expf(x - mp);
    }
    l = warp_sum(l);
    lp = warp_sum(lp);
    const float lse = m + logf(l), lsep = mp + logf(lp);
    if (lane == 0) acc += lse - lsep;
    for (int c = lane; c < 2 * N; c += 32) {
      const bool first = c < N;
      const int cc = first ? c : c - N;
      const bool same = (cc / P) == k;
      const float x = first ? sim[cc * N + r] : sim[r * N + cc] + (same ? -1e12f : 0.f);
      float gr = expf(x - lse);
      if (first && same) gr -= expf(x - lsep);
      gr /= (float)bs;
      atomicAdd(first ? &dsim[cc * N + r] : &dsim[r * N + cc], gr);
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) *loss = acc / (float)bs;
}

// ------------------------------------------------------------------------------------------------------------
// softmax cross-entropy over wide rows (vocab logits / MFM frame logits)
// ------------------------------------------------------------------------------------------------------------
// target_mode 0: target = labels[r]; 1: target = r.  Row is scored iff labels[r] != ignore_index.
// Optional pairwise mask (MFM): logit += (1 - vm[r] * vm[c]) * -1e8   (modeling.py:286-288).
__global__ void __launch_bounds__(256)
xent_fwd_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                const long long* __restrict__ vm, float* __restrict__ lse_out, float* __restrict__ loss_sum,
                float* __restrict__ count, int V, int target_mode, long long ignore_index) {
  __shared__ float red[32];
  const int r = blockIdx.x;
  const long long lab = labels[r];
  if (lab == ignore_index) {
    if (threadIdx.x == 0) lse_out[r] = 0.f;
    return;
  }
  const float* row = logits + (long long)r * ld;
  const float vr = vm ? (vm[r] != 0 ? 1.f : 0.f) : 1.f;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    float x = row[c];
    if (vm) x += (1.0f - vr * (vm[c] != 0 ? 1.f : 0.f)) * -1e8f;
    m = fmaxf(m, x);
  }
  m = block_max(m, red);
  float l = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    float x = row[c];
    if (vm) x += (1.0f - vr * (vm[c] != 0 ? 1.f : 0.f)) * -1e8f;
    l += expf(x - m);
  }
  l = block_sum(l, red);
  if (threadIdx.x == 0) {
    const float lse = m + logf(l);
    lse_out[r] = lse;
    const long long tgt = target_mode == 0 ? lab : r;
    float xt = row[tgt];
    if (vm) xt += (1.0f - vr * (vm[tgt] != 0 ? 1.f : 0.f)) * -1e8f;
    atomicAdd(loss_sum, lse - xt);
    atomicAdd(count, 1.f);
  }
}

// dlogits(bf16)[r, c] = g/count * (softmax - onehot) for scored rows, 0 elsewhere; columns [V, ld_d) zero-filled
__global__ void __launch_bounds__(256)
xent_bwd_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                const long long* __restrict__ vm, const float* __restrict__ lse_in, const float* __restrict__ count,
                const float* __restrict__ gscale, bf16* __restrict__ dlogits, long long ld_d, int V, int target_mode,
                long long ignore_index) {
  const int r = blockIdx.x;
  const long long lab = labels[r];
  bf16* drow = dlogits + (long long)r * ld_d;
  if (lab == ignore_index) {
    for (int c = threadIdx.x; c < ld_d; c += blockDim.x) drow[c] = __float2bfloat16(0.f);
    return;
  }
  const float* row = logits + (long long)r * ld;
  const float vr = vm ? (vm[r] != 0 ? 1.f : 0.f) : 1.f;
  const float lse = lse_in[r];
  const float g = (gscale ? *gscale : 1.f) / *count;
  const long long tgt = target_mode == 0 ? lab : r;
  for (int c = threadIdx.x; c < ld_d; c += blockDim.x) {
    float d = 0.f;
    if (c < V) {
      float x = row[c];
      if (vm) x += (1.0f - vr * (vm[c] != 0 ? 1.f : 0.f)) * -1e8f;
      d = (expf(x - lse) - (c == tgt ? 1.f : 0.f)) * g;
    }
    drow[c] = __float2bfloat16(d);
  }
}

__global__ void finalize_mean_kernel(const float* __restrict__ sum, const float* __restrict__ count,
                                     float* __restrict__ out) {
  *out = *sum / *count;  // 0/0 -> NaN exactly like the reference's mean of an empty selection (modeling.py:295-296)
}

// ------------------------------------------------------------------------------------------------------------
// cross pooler activation + similarity_dense:  logit[r] = tanh(u[r,:]) . w + b
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pooler_sim_fwd_kernel(const bf16* __restrict__ u, const float* __restrict__ w, const float* __restrict__ b,
                      float* __restrict__ out, int N, int H) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= N) return;
  float acc = 0.f;
  for (int c = lane; c < H; c += 32) acc += tanhf(__bfloat162float(u[(long long)row * H + c])) * w[c];
  acc = warp_sum(acc);
  if (lane == 0) out[row] = acc + b[0];
}
__global__ void __launch_bounds__(256)
pooler_sim_bwd_kernel(const bf16* __restrict__ u, const float* __restrict__ w, const float* __restrict__ dout,
                      bf16* __restrict__ du, float* __restrict__ dw, float* __restrict__ db, int N, int H) {
  // one CTA handles a slab of rows; threads own columns; dw / db receive this CTA's partial row (summed in CTA order)
  const int rows_per = (N + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per, r1 = min(N, r0 + rows_per);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const float wc = w[c];
    float acc = 0.f;
    for (int r = r0; r < r1; ++r) {
      const float th = tanhf(__bfloat162float(u[(long long)r * H + c]));
      const float g = dout[r];
      acc += g * th;
      du[(long long)r * H + c] = __float2bfloat16(g * wc * (1.f - th * th));
    }
    dw[(long long)blockIdx.x * H + c] = acc;
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int r = r0; r < r1; ++r) s += dout[r];
    db[blockIdx.x] = s;
  }
}

__global__ void scale_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, long long n,
                                 const float* __restrict__ g) {
  const float s = *g;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i] * s;
}

}  // namespace univl

using namespace univl;

extern "C" int univl_meanpool_fwd(const void* x, const long long* mask, float* out, float* norm_out, int N, int S,
                                  int H, int skip_first, int guard_zero, int l2norm, void* stream) {
  UNIVL_CHECK_ARG(x && mask && out && N >= 0 && S > 0 && H > 0 && H <= 1024, "meanpool_fwd: bad arguments");
  UNIVL_CHECK_ARG(!l2norm || norm_out, "meanpool_fwd: norm_out required with l2norm");
  if (N == 0) return UNIVL_OK;
  meanpool_fwd_kernel<<<N, 256, 0, (cudaStream_t)stream>>>((const bf16*)x, mask, out, norm_out, S, H, skip_first,
                                                           guard_zero, l2norm);
  UNIVL_CHECK_LAUNCH("meanpool_fwd");
  return UNIVL_OK;
}
extern "C" int univl_meanpool_bwd(const float* dy, const float* y, const float* norm, const long long* mask, void* dx,
                                  int N, int S, int H, int skip_first, int guard_zero, int l2norm, void* stream) {
  UNIVL_CHECK_ARG(dy && y && mask && dx && N >= 0 && S > 0 && H > 0, "meanpool_bwd: bad arguments");
  if (N == 0) return UNIVL_OK;
  meanpool_bwd_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(dy, y, norm, mask, (bf16*)dx, S, H, skip_first, guard_zero,
                                                           l2norm);
  UNIVL_CHECK_LAUNCH("meanpool_bwd");
  return UNIVL_OK;
}
extern "C" int univl_sim_matmul_fwd(const float* t, const float* v, float* sim, int Bt, int Bv, int H, void* stream) {
  UNIVL_CHECK_ARG(t && v && sim && Bt > 0 && Bv > 0 && H > 0, "sim_matmul_fwd: bad arguments");
  const long long threads = (long long)Bt * Bv * 32;
  sim_fwd_kernel<<<(int)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(t, v, sim, Bt, Bv, H);
  UNIVL_CHECK_LAUNCH("sim_matmul_fwd");
  return UNIVL_OK;
}
extern "C" int univl_sim_matmul_bwd(const float* dsim, const float* t, const float* v, float* dt, float* dv, int Bt,
                                    int Bv, int H, void* stream) {
  UNIVL_CHECK_ARG(dsim && t && v && dt && dv && Bt > 0 && Bv > 0 && H > 0, "sim_matmul_bwd: bad arguments");
  sim_bwd_kernel<<<Bt + Bv, 256, 0, (cudaStream_t)stream>>>(dsim, t, v, dt, dv, Bt, Bv, H);
  UNIVL_CHECK_LAUNCH("sim_matmul_bwd");
  return UNIVL_OK;
}
// n_pair <= 0 disables the block weighting (weights 1)
extern "C" int univl_maxmargin_loss(const float* sim, float* loss, float* dsim, int B, float margin, int n_pair,
                                    float w_same, float w_diff, void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && B > 0 && B <= 4096, "maxmargin_loss: bad arguments");
  maxmargin_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(sim, loss, dsim, B, margin, n_pair, w_same, w_diff);
  UNIVL_CHECK_LAUNCH("maxmargin_loss");
  return UNIVL_OK;
}
extern "C" int univl_crossen_loss(const float* sim, float* loss, float* dsim, int B, void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && B > 0, "crossen_loss: bad arguments");
  crossen_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(sim, loss, dsim, B);
  UNIVL_CHECK_LAUNCH("crossen_loss");
  return UNIVL_OK;
}
extern "C" int univl_milnce_loss(const float* sim, float* loss, float* dsim, int batch_size, int n_pair,
                                 void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && batch_size > 0 && n_pair > 0, "milnce_loss: bad arguments");
  milnce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(sim, loss, dsim, batch_size, n_pair);
  UNIVL_CHECK_LAUNCH("milnce_loss");
  return UNIVL_OK;
}
// loss = mean over scored rows of (logsumexp(row) - row[target]);  scratch: lse[T], sum_count[2] (zeroed here)
extern "C" int univl_softmax_xent_fwd(const float* logits, long long ld, const long long* labels,
                                      const long long* pair_mask, float* lse, float* sum_count, float* loss, int T,
                                      int V, int target_mode, long long ignore_index, void* stream) {
  UNIVL_CHECK_ARG(logits && labels && lse && sum_count && loss && T > 0 && V > 0 && ld >= V,
                  "softmax_xent_fwd: bad arguments");
  UNIVL_CHECK_ARG(target_mode == 0 || target_mode == 1, "softmax_xent_fwd: bad target_mode");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(sum_count, 0, 2 * sizeof(float), st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "softmax_xent_fwd memset: %s", cudaGetErrorString(e));
  xent_fwd_kernel<<<T, 256, 0, st>>>(logits, ld, labels, pair_mask, lse, sum_count, sum_count + 1, V, target_mode,
                                     ignore_index);
  finalize_mean_kernel<<<1, 1, 0, st>>>(sum_count, sum_count + 1, loss);
  UNIVL_CHECK_LAUNCH("softmax_xent_fwd");
  return UNIVL_OK;
}
extern "C" int univl_softmax_xent_bwd(const float* logits, long long ld, const long long* labels,
                                      const long long* pair_mask, const float* lse, const float* sum_count,
                                      const float* gscale, void* dlogits, long long ld_d, int T, int V,
                                      int target_mode, long long ignore_index, void* stream) {
  UNIVL_CHECK_ARG(logits && labels && lse && sum_count && dlogits && T > 0 && V > 0 && ld_d >= V,
                  "softmax_xent_bwd: bad arguments");
  xent_bwd_kernel<<<T, 256, 0, (cudaStream_t)stream>>>(logits, ld, labels, pair_mask, lse, sum_count + 1, gscale,
                                                       (bf16*)dlogits, ld_d, V, target_mode, ignore_index);
  UNIVL_CHECK_LAUNCH("softmax_xent_bwd");
  return UNIVL_OK;
}
extern "C" int univl_pooler_sim_fwd(const void* u, const float* w, const float* b, float* out, int N, int H,
                                    void* stream) {
  UNIVL_CHECK_ARG(u && w && b && out && N > 0 && H > 0, "pooler_sim_fwd: bad arguments");
  pooler_sim_fwd_kernel<<<(N * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>((const bf16*)u, w, b, out, N, H);
  UNIVL_CHECK_LAUNCH("pooler_sim_fwd");
  return UNIVL_OK;
}
extern "C" int univl_pooler_sim_bwd(const void* u, const float* w, const float* dout, void* du, float* dw, float* db,
                                    int N, int H, void* stream) {
  UNIVL_CHECK_ARG(u && w && dout && du && dw && db && N > 0 && H > 0, "pooler_sim_bwd: bad arguments");
  int blocks = (N + 15) / 16;
  if (blocks > device_sms()) blocks = device_sms();
  cudaStream_t st = (cudaStream_t)stream;
  float *pw, *pb;
  if (int rc = scratch_alloc((void**)&pw, (size_t)blocks * H * sizeof(float), st)) return rc;
  if (int rc = scratch_alloc((void**)&pb, (size_t)blocks * sizeof(float), st)) return rc;
  pooler_sim_bwd_kernel<<<blocks, 256, 0, st>>>((const bf16*)u, w, dout, (bf16*)du, pw, pb, N, H);
  UNIVL_CHECK_LAUNCH("pooler_sim_bwd");
  if (int rc = partials_reduce(pw, blocks, 1, H, dw, H, st)) return rc;
  return partials_reduce(pb, blocks, 1, 1, db, 1, st);
}
// dst[i] = src[i] * (*gscale)   — applies autograd's upstream scalar without a host round trip
extern "C" int univl_scale_f32(float* dst, const float* src, long long n, const float* gscale, void* stream) {
  UNIVL_CHECK_ARG(dst && src && gscale && n >= 0, "scale_f32: bad arguments");
  if (n == 0) return UNIVL_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > device_sms() * 8) blocks = device_sms() * 8;
  scale_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(dst, src, n, gscale);
  UNIVL_CHECK_LAUNCH("scale_f32");
  return UNIVL_OK;
}
