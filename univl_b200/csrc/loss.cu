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
// The rows sequence n pools, in the order they are added: row k < count() is x row row(k), pooled when on(k).
// Padded: the S rows of the [N, S] layout, on where the mask is set.  Packed: the sequence's valid rows alone
// (cu[n] .. cu[n + 1] - 1, ascending source position), so it adds the same values in the same order as the padded
// layout, which skips its masked rows.
struct PaddedPoolRows {
  const long long* mask;
  int S, skip_first;
  long long n;
  __device__ int count() const { return S; }
  __device__ bool on(int k) const { return mask[n * S + k] != 0 && !(skip_first && k == 0); }
  __device__ long long row(int k) const { return n * S + k; }
};
struct PackedPoolRows {
  const int* idx;  // source token of every packed row (i * S + s)
  int S, skip_first, first, last;
  __device__ int count() const { return last - first; }
  __device__ bool on(int k) const { return !(skip_first && idx[first + k] % S == 0); }
  __device__ long long row(int k) const { return (long long)first + k; }
};

template <class Rows>
__device__ __forceinline__ void meanpool_row(const bf16* __restrict__ x, const Rows& rows, float* __restrict__ out,
                                             float* __restrict__ norm_out, long long n, int H, int guard_zero,
                                             int l2norm, float* red) {
  const int count = rows.count();
  float den = 0.f;
  for (int k = 0; k < count; ++k) den += rows.on(k) ? 1.f : 0.f;
  if (guard_zero && den == 0.f) den = 1.f;
  float sq = 0.f;
  float u[4];
  int nc = 0;
  for (int c = threadIdx.x; c < H; c += blockDim.x, ++nc) {
    float acc = 0.f;
    for (int k = 0; k < count; ++k)
      if (rows.on(k)) acc += __bfloat162float(x[rows.row(k) * H + c]);
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
  for (int c = threadIdx.x; c < H; c += blockDim.x, ++nc) out[n * H + c] = u[nc] / nrm;
}

__global__ void __launch_bounds__(256)
meanpool_fwd_kernel(const bf16* __restrict__ x, const long long* __restrict__ mask, float* __restrict__ out,
                    float* __restrict__ norm_out, int S, int H, int skip_first, int guard_zero, int l2norm) {
  __shared__ float red[32];
  const PaddedPoolRows rows{mask, S, skip_first, (long long)blockIdx.x};
  meanpool_row(x, rows, out, norm_out, blockIdx.x, H, guard_zero, l2norm, red);
}

__global__ void __launch_bounds__(256)
meanpool_packed_fwd_kernel(const bf16* __restrict__ x, const int* __restrict__ cu, const int* __restrict__ idx,
                           float* __restrict__ out, int S, int H, int skip_first, int guard_zero, int l2norm) {
  __shared__ float red[32];
  const PackedPoolRows rows{idx, S, skip_first, cu[blockIdx.x], cu[blockIdx.x + 1]};
  meanpool_row(x, rows, out, (float*)nullptr, blockIdx.x, H, guard_zero, l2norm, red);
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
// sim = T V^T  (tiny); with G groups the block diagonal sim[g] = T[g Bt : (g+1) Bt] V[g Bv : (g+1) Bv]^T, [G, Bt, Bv]
// ------------------------------------------------------------------------------------------------------------
__global__ void sim_fwd_kernel(const float* __restrict__ t, const float* __restrict__ v, float* __restrict__ sim,
                               int Bt, int Bv, int H, int groups) {
  // 64-bit: a matrix of more than 2^27 entries has more than 2^32 threads
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)groups * Bt * Bv) return;
  const int g = (int)(gw / ((long long)Bt * Bv));
  const long long e = gw - (long long)g * Bt * Bv;
  const int i = g * Bt + (int)(e / Bv), j = g * Bv + (int)(e % Bv);
  const float acc = sim_dot(t + (long long)i * H, v + (long long)j * H, H, lane);
  if (lane == 0) sim[gw] = acc;
}
// dt[i,:] = sum_j dsim[i,j] v[j,:] ; dv[j,:] = sum_i dsim[i,j] t[i,:]   (within group blockIdx.x / (Bt + Bv))
__global__ void sim_bwd_kernel(const float* __restrict__ dsim, const float* __restrict__ t,
                               const float* __restrict__ v, float* __restrict__ dt, float* __restrict__ dv, int Bt,
                               int Bv, int H) {
  const int g = blockIdx.x / (Bt + Bv), r = blockIdx.x - g * (Bt + Bv);
  dsim += (long long)g * Bt * Bv;
  t += (long long)g * Bt * H;
  dt += (long long)g * Bt * H;
  v += (long long)g * Bv * H;
  dv += (long long)g * Bv * H;
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
// losses on a [B, B] similarity matrix, one CTA per group of a [G, B, B] stack.  With G = 1 the CTA writes the loss
// itself; with G > 1 it writes its group's loss to parts[g] (group_mean_kernel averages them in group order) and scales
// its dsim by 1/G, the gradient of the mean over groups.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void group_scale_dsim(float* dsim, int n) {
  if (gridDim.x == 1) return;
  __syncthreads();
  const float s = 1.0f / (float)gridDim.x;
  for (int e = threadIdx.x; e < n; e += blockDim.x) dsim[e] *= s;
}
__global__ void group_mean_kernel(const float* __restrict__ parts, int groups, float* __restrict__ out) {
  float acc = 0.f;
  for (int g = 0; g < groups; ++g) acc += parts[g];
  *out = acc / (float)groups;
}
// mean_ij w_ij * ( relu(m + s_ij - s_ii) + relu(m + s_ij - s_jj) ), diagonal included (until_module.py:245-251)
__global__ void __launch_bounds__(256)
maxmargin_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int B, float margin,
                 int n_pair, float w_same, float w_diff) {
  __shared__ float red[32];
  sim += (long long)blockIdx.x * B * B;
  dsim += (long long)blockIdx.x * B * B;
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
  if (threadIdx.x == 0) loss[blockIdx.x] = acc * inv;
  group_scale_dsim(dsim, B * B);
}

// -mean_i log_softmax(sim[i,:])[i]   (until_module.py:186-191)
__global__ void __launch_bounds__(256)
crossen_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int B) {
  __shared__ float red[32];
  sim += (long long)blockIdx.x * B * B;
  dsim += (long long)blockIdx.x * B * B;
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
  if (threadIdx.x == 0) loss[blockIdx.x] = acc / (float)B;
  group_scale_dsim(dsim, B * B);
}

// MIL-NCE (until_module.py:201-221) on sim [N, N], N = bs * P.  For each picked row r = k*P + P/2:
//   loss_r = logsumexp_{all c}(row) - logsumexp_{c in pos(r)}(row),
//   row = [ sim[c, r] for c < N ] ++ [ sim[r, c] - 1e12 * same_block(r, c) for c < N ],  pos(r) = first half, same block.
__global__ void __launch_bounds__(256)
milnce_kernel(const float* __restrict__ sim, float* __restrict__ loss, float* __restrict__ dsim, int bs, int P) {
  __shared__ float red[32];
  const int N = bs * P;
  sim += (long long)blockIdx.x * N * N;
  dsim += (long long)blockIdx.x * N * N;
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
      // Order-independent: a cell receives at most two addends onto its 0 — (r, r) from both halves of row r, and
      // (r1, r2) from the picked rows r1 and r2 — and 0 + a + b has the same bits as 0 + b + a.
      atomicAdd(first ? &dsim[cc * N + r] : &dsim[r * N + cc], gr);
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) loss[blockIdx.x] = acc / (float)bs;
  group_scale_dsim(dsim, N * N);
}

// ------------------------------------------------------------------------------------------------------------
// softmax cross-entropy over wide rows (vocab logits / MFM frame logits)
// ------------------------------------------------------------------------------------------------------------
// target_mode 0: target = labels[r]; 1: target = r.  Row is scored iff labels[r] != ignore_index.
// Optional pairwise mask (MFM): logit += (1 - vm[r] * vm[c]) * -1e8   (modeling.py:286-288).
// G groups of R = T / G consecutive rows (micro-batches) keep their own sum and count (xent_sum_kernel).  In
// target_mode 1 a row of group g holds logits against its own group's R frames only (the MFM NCE of one micro-batch):
// its target is r - g R and its mask columns are vm[g R + c].
__global__ void __launch_bounds__(256)
xent_fwd_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                const long long* __restrict__ vm, float* __restrict__ lse_out, float* __restrict__ term, int V,
                int target_mode, long long ignore_index, int rows_per_group) {
  __shared__ float red[32];
  const int r = blockIdx.x;
  const long long lab = labels[r];
  if (lab == ignore_index) {
    if (threadIdx.x == 0) lse_out[r] = term[r] = 0.f;
    return;
  }
  const int g = r / rows_per_group;
  const long long off = target_mode == 1 ? (long long)g * rows_per_group : 0;
  const float* row = logits + (long long)r * ld;
  const float vr = vm ? (vm[r] != 0 ? 1.f : 0.f) : 1.f;
  if (vm) vm += off;
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
    const long long tgt = target_mode == 0 ? lab : r - off;
    float xt = row[tgt];
    if (vm) xt += (1.0f - vr * (vm[tgt] != 0 ? 1.f : 0.f)) * -1e8f;
    term[r] = lse - xt;
  }
}

// dlogits(bf16)[r, c] = (g / G) / count[group] * (softmax - onehot) for scored rows, 0 elsewhere; columns [V, ld_d)
// zero-filled
__global__ void __launch_bounds__(256)
xent_bwd_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                const long long* __restrict__ vm, const float* __restrict__ lse_in, const float* __restrict__ count,
                const float* __restrict__ gscale, bf16* __restrict__ dlogits, long long ld_d, int V, int target_mode,
                long long ignore_index, int rows_per_group, int groups) {
  const int r = blockIdx.x;
  const long long lab = labels[r];
  bf16* drow = dlogits + (long long)r * ld_d;
  if (lab == ignore_index) {
    for (int c = threadIdx.x; c < ld_d; c += blockDim.x) drow[c] = __float2bfloat16(0.f);
    return;
  }
  const int grp = r / rows_per_group;
  const long long off = target_mode == 1 ? (long long)grp * rows_per_group : 0;
  const float* row = logits + (long long)r * ld;
  const float vr = vm ? (vm[r] != 0 ? 1.f : 0.f) : 1.f;
  if (vm) vm += off;
  const float lse = lse_in[r];
  // (gscale / G) / count: the bits of the reference loop's (loss / G).backward() on this row's micro-batch alone
  const float g = ((gscale ? *gscale : 1.f) / (float)groups) / count[grp];
  const long long tgt = target_mode == 0 ? lab : r - off;
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

// One CTA: sum[g] and count[g] of each group's per-row terms (xent_fwd_kernel), each thread adding its rows in row order
// and block_sum combining the threads in a fixed order, so the loss has the same bits on every launch.  Then the mean
// over groups of sum[g] / count[g]; 0/0 -> NaN exactly like the reference's mean of an empty selection
// (modeling.py:295-296), so a group without a scored row makes the loss NaN, as that micro-batch's loss would be.
__global__ void __launch_bounds__(256)
xent_sum_kernel(const float* __restrict__ term, const long long* __restrict__ labels, long long ignore_index,
                int rows_per_group, int groups, float* __restrict__ sum, float* __restrict__ count,
                float* __restrict__ out) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int g = 0; g < groups; ++g) {
    const long long r0 = (long long)g * rows_per_group;
    float s = 0.f, n = 0.f;
    for (int r = threadIdx.x; r < rows_per_group; r += blockDim.x) {
      s += term[r0 + r];
      n += labels[r0 + r] != ignore_index ? 1.f : 0.f;
    }
    s = block_sum(s, red);
    n = block_sum(n, red);
    if (threadIdx.x == 0) {
      sum[g] = s;
      count[g] = n;
      acc = g == 0 ? s / n : acc + s / n;
    }
  }
  if (threadIdx.x == 0) *out = groups > 1 ? acc / (float)groups : acc;
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
extern "C" int univl_meanpool_packed_fwd(const void* x, const int* cu, const int* idx, float* out, int N, int S, int H,
                                         int skip_first, int guard_zero, int l2norm, void* stream) {
  // x and idx are read only for the rows the sequences hold: both may be null when there are none
  UNIVL_CHECK_ARG(cu && out && N >= 0 && S > 0 && H > 0 && H <= 1024, "meanpool_packed_fwd: bad arguments");
  if (N == 0) return UNIVL_OK;
  meanpool_packed_fwd_kernel<<<N, 256, 0, (cudaStream_t)stream>>>((const bf16*)x, cu, idx, out, S, H, skip_first,
                                                                  guard_zero, l2norm);
  UNIVL_CHECK_LAUNCH("meanpool_packed_fwd");
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
extern "C" int univl_sim_matmul_fwd(const float* t, const float* v, float* sim, int Bt, int Bv, int H, int groups,
                                    void* stream) {
  UNIVL_CHECK_ARG(t && v && sim && Bt > 0 && Bv > 0 && H > 0 && groups > 0, "sim_matmul_fwd: bad arguments");
  const long long threads = (long long)groups * Bt * Bv * 32;
  sim_fwd_kernel<<<(int)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(t, v, sim, Bt, Bv, H, groups);
  UNIVL_CHECK_LAUNCH("sim_matmul_fwd");
  return UNIVL_OK;
}
extern "C" int univl_sim_matmul_bwd(const float* dsim, const float* t, const float* v, float* dt, float* dv, int Bt,
                                    int Bv, int H, int groups, void* stream) {
  UNIVL_CHECK_ARG(dsim && t && v && dt && dv && Bt > 0 && Bv > 0 && H > 0 && groups > 0,
                  "sim_matmul_bwd: bad arguments");
  sim_bwd_kernel<<<groups * (Bt + Bv), 256, 0, (cudaStream_t)stream>>>(dsim, t, v, dt, dv, Bt, Bv, H);
  UNIVL_CHECK_LAUNCH("sim_matmul_bwd");
  return UNIVL_OK;
}
// one CTA per group; G > 1 collects the group losses in scratch and averages them in group order
template <typename Launch>
static int group_loss(float* loss, int groups, cudaStream_t st, const char* name, Launch launch) {
  if (groups == 1) {
    launch(loss);
    UNIVL_CHECK_LAUNCH(name);
    return UNIVL_OK;
  }
  float* parts;
  if (int rc = scratch_alloc((void**)&parts, (size_t)groups * sizeof(float), st)) return rc;
  launch(parts);
  group_mean_kernel<<<1, 1, 0, st>>>(parts, groups, loss);
  const cudaError_t e = cudaGetLastError();
  cudaFreeAsync(parts, st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "%s launch: %s", name, cudaGetErrorString(e));
  return UNIVL_OK;
}
// n_pair <= 0 disables the block weighting (weights 1)
extern "C" int univl_maxmargin_loss(const float* sim, float* loss, float* dsim, int B, float margin, int n_pair,
                                    float w_same, float w_diff, int groups, void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && B > 0 && B <= 4096 && groups > 0, "maxmargin_loss: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  return group_loss(loss, groups, st, "maxmargin_loss", [&](float* out) {
    maxmargin_kernel<<<groups, 256, 0, st>>>(sim, out, dsim, B, margin, n_pair, w_same, w_diff);
  });
}
extern "C" int univl_crossen_loss(const float* sim, float* loss, float* dsim, int B, int groups, void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && B > 0 && groups > 0, "crossen_loss: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  return group_loss(loss, groups, st, "crossen_loss", [&](float* out) {
    crossen_kernel<<<groups, 256, 0, st>>>(sim, out, dsim, B);
  });
}
extern "C" int univl_milnce_loss(const float* sim, float* loss, float* dsim, int batch_size, int n_pair, int groups,
                                 void* stream) {
  UNIVL_CHECK_ARG(sim && loss && dsim && batch_size > 0 && n_pair > 0 && groups > 0, "milnce_loss: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  return group_loss(loss, groups, st, "milnce_loss", [&](float* out) {
    milnce_kernel<<<groups, 256, 0, st>>>(sim, out, dsim, batch_size, n_pair);
  });
}
// loss = mean over groups of the mean over the group's scored rows of (logsumexp(row) - row[target]);
// outputs besides the loss: lse[T], sum_count[2 * groups] (sums, then counts)
extern "C" int univl_softmax_xent_fwd(const float* logits, long long ld, const long long* labels,
                                      const long long* pair_mask, float* lse, float* sum_count, float* loss, int T,
                                      int V, int target_mode, long long ignore_index, int groups, void* stream) {
  UNIVL_CHECK_ARG(logits && labels && lse && sum_count && loss && T > 0 && V > 0 && ld >= V,
                  "softmax_xent_fwd: bad arguments");
  UNIVL_CHECK_ARG(target_mode == 0 || target_mode == 1, "softmax_xent_fwd: bad target_mode");
  UNIVL_CHECK_ARG(groups > 0 && T % groups == 0, "softmax_xent_fwd: %d groups must divide T=%d", groups, T);
  UNIVL_CHECK_ARG(target_mode == 0 || groups == 1 || V == T / groups,
                  "softmax_xent_fwd: grouped target_mode 1 needs V = T / groups");
  cudaStream_t st = (cudaStream_t)stream;
  // per-row terms in scratch, not in lse: ProjXentFn keeps lse for the backward
  float* term;
  if (int rc = scratch_alloc((void**)&term, (size_t)T * sizeof(float), st)) return rc;
  xent_fwd_kernel<<<T, 256, 0, st>>>(logits, ld, labels, pair_mask, lse, term, V, target_mode, ignore_index,
                                     T / groups);
  xent_sum_kernel<<<1, 256, 0, st>>>(term, labels, ignore_index, T / groups, groups, sum_count, sum_count + groups,
                                     loss);
  const cudaError_t e = cudaGetLastError();
  cudaFreeAsync(term, st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "softmax_xent_fwd launch: %s", cudaGetErrorString(e));
  return UNIVL_OK;
}
extern "C" int univl_softmax_xent_bwd(const float* logits, long long ld, const long long* labels,
                                      const long long* pair_mask, const float* lse, const float* sum_count,
                                      const float* gscale, void* dlogits, long long ld_d, int T, int V,
                                      int target_mode, long long ignore_index, int groups, void* stream) {
  UNIVL_CHECK_ARG(logits && labels && lse && sum_count && dlogits && T > 0 && V > 0 && ld_d >= V,
                  "softmax_xent_bwd: bad arguments");
  UNIVL_CHECK_ARG(groups > 0 && T % groups == 0, "softmax_xent_bwd: %d groups must divide T=%d", groups, T);
  xent_bwd_kernel<<<T, 256, 0, (cudaStream_t)stream>>>(logits, ld, labels, pair_mask, lse, sum_count + groups, gscale,
                                                       (bf16*)dlogits, ld_d, V, target_mode, ignore_index,
                                                       T / groups, groups);
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
