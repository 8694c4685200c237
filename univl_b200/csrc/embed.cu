// univl_b200 — embedding front-ends fused with their LayerNorm (+ dropout).  HBM-bound, one warp per token row.
//
//   text    : y = dropout(LN(word[id] + pos[s] + type[t]))       reference modules/module_bert.py:132-146,
//             (type table optional: the caption decoder has none)           modules/module_decoder.py:309-320
//   sources : y = dropout(LN(src(row) + pos[s] (+ type[s >= Wa])))
//             visual embeddings (src = Linear(1024->768) output)  reference modules/module_visual.py:118-131
//             cross  embeddings (src = concat(text_i, video_j))   reference modules/module_cross.py:123-138 with
//             modules/modeling.py:315-325; in all-pairs mode sequence p = (i, j) = (p / Nb, p % Nb) reads text i and
//             video j in place — the `repeat`ed [B*B, W+F, H] input of modeling.py:358-367 is never materialised.
// The tables are the fp32 master parameters (no bf16 copy is needed for a gather).  Backward recomputes the pre-LN
// row and runs the LayerNorm backward: each row's table gradient goes to scratch memory and is summed per table row in
// row order (keyed_rows_sum_kernel); the activation gradients are direct bf16 writes (summed in registers over the
// pairs that share a source row).
#include "common.cuh"

namespace univl {

constexpr int EMB_WARPS = 8;
constexpr int EMB_H = 768;
constexpr int EMB_VEC = EMB_H / 256;  // 3 vectors of 8 per lane

struct EmbDrop {
  uint32_t threshold;
  float scale;
  uint64_t seed, stream;
  int on;
  const unsigned long long* rng;  // device {seed, epoch}, resolved at kernel entry (graph-replayable)
};
__device__ __forceinline__ EmbDrop resolve_emb_drop(EmbDrop d) {
  if (d.on && d.rng != nullptr) {
    d.seed = d.rng[0];
    d.stream += d.rng[1] << 20;
  }
  return d;
}

__device__ __forceinline__ void ld8f(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void ld8h(const bf16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}
__device__ __forceinline__ void st8h(bf16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void emb_keep8(const EmbDrop& d, uint64_t idx0, bool (&k)[8]) {
  const uint32_t m = dropout_keep8(d.seed, d.stream, idx0, d.threshold);
#pragma unroll
  for (int j = 0; j < 8; ++j) k[j] = (m >> j) & 1u;
}

// z (registers) -> mean/rstd -> y ; shared by both forward kernels
__device__ __forceinline__ void ln_row_fwd(float (&z)[EMB_VEC][8], const float* gamma, const float* beta, bf16* yrow,
                                           float* mean_out, float* rstd_out, long long row, float eps,
                                           const EmbDrop& drop, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += z[i][j];
  const float mean = warp_sum(s) * (1.0f / EMB_H);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = z[i][j] - mean;
      q += d * d;
    }
  const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / EMB_H) + eps);
  if (lane == 0) {
    mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i) {
    const int c = (i * 32 + lane) * 8;
    float g[8], b[8], o[8];
    ld8f(gamma + c, g);
    ld8f(beta + c, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = g[j] * ((z[i][j] - mean) * rstd) + b[j];
    if (drop.on) {
      bool k[8];
      emb_keep8(drop, (uint64_t)row * EMB_H + c, k);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = k[j] ? o[j] * drop.scale : 0.f;
    }
    st8h(yrow + c, o);
  }
}

// dy (bf16 row, after-dropout gradient) -> dz in registers; accumulates dgamma/dbeta partials
__device__ __forceinline__ void ln_row_bwd(const float (&z)[EMB_VEC][8], const bf16* dyrow, const float* gamma,
                                           float mean, float rstd, long long row, const EmbDrop& drop, int lane,
                                           float (&dz)[EMB_VEC][8], float (&acc_g)[EMB_VEC][8],
                                           float (&acc_b)[EMB_VEC][8]) {
  float xh[EMB_VEC][8], g[EMB_VEC][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i) {
    const int c = (i * 32 + lane) * 8;
    float d[8], gm[8];
    ld8h(dyrow + c, d);
    if (drop.on) {
      bool k[8];
      emb_keep8(drop, (uint64_t)row * EMB_H + c, k);
#pragma unroll
      for (int j = 0; j < 8; ++j) d[j] = k[j] ? d[j] * drop.scale : 0.f;
    }
    ld8f(gamma + c, gm);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      xh[i][j] = (z[i][j] - mean) * rstd;
      g[i][j] = d[j] * gm[j];
      s1 += g[i][j];
      s2 += g[i][j] * xh[i][j];
      acc_g[i][j] += d[j] * xh[i][j];
      acc_b[i][j] += d[j];
    }
  }
  s1 = warp_sum(s1) * (1.0f / EMB_H);
  s2 = warp_sum(s2) * (1.0f / EMB_H);
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dz[i][j] = rstd * (g[i][j] - s1 - xh[i][j] * s2);
}

__device__ __forceinline__ void flush_colsums(float (&acc)[EMB_VEC][8], float* dst, float (*red)[257], int warp,
                                              int lane) {
  for (int i = 0; i < EMB_VEC; ++i) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[i][j];
    __syncthreads();
    for (int e = threadIdx.x; e < 256; e += EMB_WARPS * 32) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < EMB_WARPS; ++w) t += red[w][e];
      dst[((long long)blockIdx.y * gridDim.x + blockIdx.x) * EMB_H + i * 256 + e] = t;  // this CTA's partial row
    }
  }
}

// Table gradients (word / position / type rows): every row's gradient dz and its table keys go to scratch memory and
// keyed_rows_sum_kernel adds, per key, the rows in row order — the same sums in the same order on every run.
__device__ __forceinline__ void st8f(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
// dst[key * H + c] += sum of src[r * H + c] over the rows r whose key is `key` (ascending r); key < 0: no table row
__global__ void __launch_bounds__(256)
keyed_rows_sum_kernel(const float* __restrict__ src, const int* __restrict__ key, long long rows, float* __restrict__ dst) {
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int k = key[r];
    if (k < 0) continue;
    bool earlier = false;  // the first row with key k owns the sum; the block stops at the first chunk that shows one
    for (long long q0 = 0; q0 < r && !earlier; q0 += blockDim.x) {
      const long long q = q0 + threadIdx.x;
      earlier = __syncthreads_or(q < r && key[q] == k) != 0;
    }
    if (earlier) continue;
    for (int c = threadIdx.x; c < EMB_H; c += blockDim.x) {
      float t = 0.f;
      for (long long q = r; q < rows; ++q)
        if (key[q] == k) t += src[q * EMB_H + c];
      dst[(long long)k * EMB_H + c] += t;
    }
  }
}

// rows [0, n_rows) are walked as  first + k * stride  with stride = the largest multiple of `period` that the launched
// warps cover, so a warp's position index (row % period) never changes; surplus warps idle
__device__ __forceinline__ long long period_stride(long long launched_warps, int period) {
  return launched_warps >= period ? (launched_warps / period) * period : launched_warps;
}

// ------------------------------------------------------------------------------------------------------------
// text embeddings
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(EMB_WARPS * 32)
embed_text_fwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ type_ids,
                      const float* __restrict__ word, const float* __restrict__ pos, const float* __restrict__ type,
                      const float* __restrict__ gamma, const float* __restrict__ beta, bf16* __restrict__ y,
                      float* __restrict__ mean_out, float* __restrict__ rstd_out, int n_seq, int S, int vocab,
                      float eps, EmbDrop drop_in) {
  const EmbDrop drop = resolve_emb_drop(drop_in);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)n_seq * S;
  for (long long row = (long long)blockIdx.x * EMB_WARPS + warp; row < rows; row += (long long)gridDim.x * EMB_WARPS) {
    const int s = (int)(row % S);
    long long id = ids[row];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const long long t = (type != nullptr && type_ids != nullptr) ? (type_ids[row] != 0 ? 1 : 0) : 0;
    float z[EMB_VEC][8];
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      float a[8], b[8];
      ld8f(word + id * EMB_H + c, a);
      ld8f(pos + (long long)s * EMB_H + c, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] = a[j] + b[j];
      if (type != nullptr) {
        float tt[8];
        ld8f(type + t * EMB_H + c, tt);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[i][j] += tt[j];
      }
    }
    ln_row_fwd(z, gamma, beta, y + row * EMB_H, mean_out, rstd_out, row, eps, drop, lane);
  }
}

__global__ void __launch_bounds__(EMB_WARPS * 32)
embed_text_bwd_kernel(const bf16* __restrict__ dy, const long long* __restrict__ ids,
                      const long long* __restrict__ type_ids, const float* __restrict__ word,
                      const float* __restrict__ pos, const float* __restrict__ type, const float* __restrict__ gamma,
                      const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float* __restrict__ zrows,
                      int* __restrict__ keys, int want_type, float* __restrict__ dgamma, float* __restrict__ dbeta,
                      int n_seq, int S, int vocab, EmbDrop drop_in) {
  const EmbDrop drop = resolve_emb_drop(drop_in);
  __shared__ float red[EMB_WARPS][257];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)n_seq * S;
  float acc_g[EMB_VEC][8], acc_b[EMB_VEC][8];
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc_g[i][j] = acc_b[i][j] = 0.f;
  const long long stride = period_stride((long long)gridDim.x * EMB_WARPS, S);
  long long row = (long long)blockIdx.x * EMB_WARPS + warp;
  if (row >= stride) row = rows;
  for (; row < rows; row += stride) {
    const int s = (int)(row % S);
    long long id = ids[row];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const long long t = (type != nullptr && type_ids != nullptr) ? (type_ids[row] != 0 ? 1 : 0) : 0;
    float z[EMB_VEC][8], dz[EMB_VEC][8];
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) {
      const int c = (i * 32 + lane) * 8;
      float a[8], b[8];
      ld8f(word + id * EMB_H + c, a);
      ld8f(pos + (long long)s * EMB_H + c, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] = a[j] + b[j];
      if (type != nullptr) {
        float tt[8];
        ld8f(type + t * EMB_H + c, tt);
#pragma unroll
        for (int j = 0; j < 8; ++j) z[i][j] += tt[j];
      }
    }
    ln_row_bwd(z, dy + row * EMB_H, gamma, mean_in[row], rstd_in[row], row, drop, lane, dz, acc_g, acc_b);
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) st8f(zrows + row * EMB_H + (i * 32 + lane) * 8, dz[i]);
    if (lane == 0) {  // table rows this token's gradient belongs to: word id, position, type
      keys[row] = (int)id;
      keys[rows + row] = s;
      keys[2 * rows + row] = want_type ? (int)t : -1;
    }
  }
  flush_colsums(acc_g, dgamma, red, warp, lane);
  flush_colsums(acc_b, dbeta, red, warp, lane);
}

// ------------------------------------------------------------------------------------------------------------
// activation-source embeddings (visual / cross)
// ------------------------------------------------------------------------------------------------------------
struct SrcCfg {
  const bf16* a;  // [Na, Wa, H]
  const bf16* b;  // [Nb, Fb, H] or null (Fb = 0)
  int Na, Wa, Nb, Fb;
  int all_pairs;  // 0: sequence p reads (a[p], b[p]); 1: p = i * Nb + j reads (a[i], b[j])
};

// Shared by both source kernels: one warp owns one SOURCE row (text row of a, or video row of b; blockIdx.y selects).
// Every output sequence that reads this row (1 in aligned mode; Nb or Na in all-pairs mode) sees the SAME pre-LN
// vector z = src + pos (+ type), hence the same mean / rstd / normalised row: LayerNorm runs once per source row and
// only the dropout mask differs between the fan-out rows.
struct SrcRow {
  long long owner;  // i (text) or j (video)
  int s;            // position inside the concatenated sequence
  int fan;          // number of output sequences reading this row
};
__device__ __forceinline__ SrcRow src_row_info(const SrcCfg& c, int which, long long sr) {
  const int len = which == 0 ? c.Wa : c.Fb;
  SrcRow r;
  r.owner = sr / len;
  r.s = (int)(sr % len) + (which == 0 ? 0 : c.Wa);
  r.fan = c.all_pairs ? (which == 0 ? c.Nb : c.Na) : 1;
  return r;
}
__device__ __forceinline__ long long src_out_row(const SrcCfg& c, int which, const SrcRow& r, int f) {
  const long long p = c.all_pairs ? (which == 0 ? r.owner * c.Nb + f : (long long)f * c.Nb + r.owner) : r.owner;
  return p * (c.Wa + c.Fb) + r.s;
}
__device__ __forceinline__ void src_load_z(const SrcCfg& c, int which, long long sr, const SrcRow& r,
                                           const float* pos, const float* type, int lane, float (&z)[EMB_VEC][8]) {
  const bf16* xr = (which == 0 ? c.a : c.b) + sr * EMB_H;
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i) {
    const int col = (i * 32 + lane) * 8;
    float a[8], b[8];
    ld8h(xr + col, a);
    ld8f(pos + (long long)r.s * EMB_H + col, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) z[i][j] = a[j] + b[j];
    if (type != nullptr) {
      float tt[8];
      ld8f(type + (which == 0 ? 0 : EMB_H) + col, tt);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] += tt[j];
    }
  }
}

__global__ void __launch_bounds__(EMB_WARPS * 32)
embed_src_fwd_kernel(SrcCfg src, const float* __restrict__ pos, const float* __restrict__ type,
                     const float* __restrict__ gamma, const float* __restrict__ beta, bf16* __restrict__ y,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out, float eps, EmbDrop drop_in) {
  const EmbDrop drop = resolve_emb_drop(drop_in);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int which = blockIdx.y;
  const long long n_src_rows = which == 0 ? (long long)src.Na * src.Wa : (long long)src.Nb * src.Fb;
  for (long long sr = (long long)blockIdx.x * EMB_WARPS + warp; sr < n_src_rows;
       sr += (long long)gridDim.x * EMB_WARPS) {
    const SrcRow r = src_row_info(src, which, sr);
    float z[EMB_VEC][8];
    src_load_z(src, which, sr, r, pos, type, lane, z);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += z[i][j];
    const float mean = warp_sum(sum) * (1.0f / EMB_H);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = z[i][j] - mean;
        q += d * d;
      }
    const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / EMB_H) + eps);
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) {
      const int col = (i * 32 + lane) * 8;
      float g[8], b[8];
      ld8f(gamma + col, g);
      ld8f(beta + col, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] = g[j] * ((z[i][j] - mean) * rstd) + b[j];
    }
    for (int f = 0; f < r.fan; ++f) {
      const long long row = src_out_row(src, which, r, f);
      if (lane == 0) {
        mean_out[row] = mean;
        rstd_out[row] = rstd;
      }
#pragma unroll
      for (int i = 0; i < EMB_VEC; ++i) {
        const int col = (i * 32 + lane) * 8;
        float o[8];
        uint32_t keep = 0xffu;
        if (drop.on) keep = dropout_keep8(drop.seed, drop.stream, (uint64_t)row * EMB_H + col, drop.threshold);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = ((keep >> j) & 1u) ? z[i][j] * drop.scale : 0.f;
        st8h(y + row * EMB_H + col, o);
      }
    }
  }
}

// Backward: LayerNorm backward is linear in the upstream gradient and z / mean / rstd are shared by the fan-out rows,
// so the (dropout-masked) dy rows are first SUMMED over the fan-out — SRC_BATCH rows of 16-byte loads in flight per lane —
// and one LayerNorm backward runs on the sum.  Deterministic, no atomics on activations.
constexpr int SRC_BATCH = 2;
__global__ void __launch_bounds__(EMB_WARPS * 32)
embed_src_bwd_kernel(const bf16* __restrict__ dy, SrcCfg src, const float* __restrict__ pos,
                     const float* __restrict__ type, const float* __restrict__ gamma,
                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in, bf16* __restrict__ da,
                     bf16* __restrict__ db, float* __restrict__ zrows, int* __restrict__ keys, int want_type,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, EmbDrop drop_in) {
  const EmbDrop drop = resolve_emb_drop(drop_in);
  __shared__ float red[EMB_WARPS][257];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int which = blockIdx.y;  // 0: rows of a, 1: rows of b
  const long long n_src_rows = which == 0 ? (long long)src.Na * src.Wa : (long long)src.Nb * src.Fb;
  float acc_g[EMB_VEC][8], acc_b[EMB_VEC][8];
#pragma unroll
  for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc_g[i][j] = acc_b[i][j] = 0.f;
  const long long rows_a = (long long)src.Na * src.Wa;
  const long long n_rows = rows_a + (src.Fb > 0 ? (long long)src.Nb * src.Fb : 0);
  const long long stride = period_stride((long long)gridDim.x * EMB_WARPS, which == 0 ? src.Wa : src.Fb);
  long long sr = (long long)blockIdx.x * EMB_WARPS + warp;
  if (sr >= stride) sr = n_src_rows;
  for (; sr < n_src_rows; sr += stride) {
    const SrcRow r = src_row_info(src, which, sr);
    float D[EMB_VEC][8];
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) D[i][j] = 0.f;
    for (int f0 = 0; f0 < r.fan; f0 += SRC_BATCH) {
      uint4 raw[SRC_BATCH][EMB_VEC];
      long long rows[SRC_BATCH];
#pragma unroll
      for (int u = 0; u < SRC_BATCH; ++u) {
        rows[u] = src_out_row(src, which, r, min(f0 + u, r.fan - 1));
#pragma unroll
        for (int i = 0; i < EMB_VEC; ++i)
          raw[u][i] = *reinterpret_cast<const uint4*>(dy + rows[u] * EMB_H + (i * 32 + lane) * 8);
      }
#pragma unroll
      for (int u = 0; u < SRC_BATCH; ++u) {
        if (f0 + u >= r.fan) continue;
#pragma unroll
        for (int i = 0; i < EMB_VEC; ++i) {
          const int col = (i * 32 + lane) * 8;
          uint32_t keep = 0xffu;
          if (drop.on) keep = dropout_keep8(drop.seed, drop.stream, (uint64_t)rows[u] * EMB_H + col, drop.threshold);
          const uint32_t w[4] = {raw[u][i].x, raw[u][i].y, raw[u][i].z, raw[u][i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 v = unpack_bf16x2(w[j]);
            if ((keep >> (2 * j)) & 1u) D[i][2 * j] += v.x;
            if ((keep >> (2 * j + 1)) & 1u) D[i][2 * j + 1] += v.y;
          }
        }
      }
    }
    if (drop.on) {
#pragma unroll
      for (int i = 0; i < EMB_VEC; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) D[i][j] *= drop.scale;
    }
    // one LayerNorm backward on the summed gradient
    const long long row0 = src_out_row(src, which, r, 0);
    const float mean = mean_in[row0], rstd = rstd_in[row0];
    float z[EMB_VEC][8];
    src_load_z(src, which, sr, r, pos, type, lane, z);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) {
      float gm[8];
      ld8f(gamma + (i * 32 + lane) * 8, gm);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (z[i][j] - mean) * rstd;
        const float g = D[i][j] * gm[j];
        s1 += g;
        s2 = fmaf(g, xh, s2);
        acc_g[i][j] = fmaf(D[i][j], xh, acc_g[i][j]);
        acc_b[i][j] += D[i][j];
        z[i][j] = xh;
        D[i][j] = g;
      }
    }
    s1 = warp_sum(s1) * (1.0f / EMB_H);
    s2 = warp_sum(s2) * (1.0f / EMB_H);
    bf16* dst = (which == 0 ? da : db);
    const long long zr = (which == 0 ? 0 : rows_a) + sr;  // row of the table-gradient scratch
#pragma unroll
    for (int i = 0; i < EMB_VEC; ++i) {
      const int col = (i * 32 + lane) * 8;
      float dz[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[j] = rstd * (D[i][j] - s1 - z[i][j] * s2);
      if (dst != nullptr) st8h(dst + sr * EMB_H + col, dz);
      st8f(zrows + zr * EMB_H + col, dz);
    }
    if (lane == 0) {  // table rows: position r.s, type = which source
      keys[zr] = r.s;
      keys[n_rows + zr] = want_type ? which : -1;
    }
  }
  flush_colsums(acc_g, dgamma, red, warp, lane);
  flush_colsums(acc_b, dbeta, red, warp, lane);
}

struct EmbTables {
  float* t[3];  // word, position, type gradients (each nullable); keys holds one slot of `rows` keys per non-null table
};
// table gradients from the per-row scratch (keyed, in row order) and LayerNorm gamma / beta from the per-CTA partials;
// frees the scratch
static int emb_table_grads(float* zrows, int* keys, long long rows, EmbTables tabs, float* pg, float* pb, int parts,
                           float* dgamma, float* dbeta, cudaStream_t st) {
  long long blocks = rows < device_sms() * 8LL ? rows : device_sms() * 8LL;
  int k_used = 0;
  for (int k = 0; k < 3; ++k) {
    if (tabs.t[k] == nullptr) continue;
    keyed_rows_sum_kernel<<<(int)(blocks < 1 ? 1 : blocks), 256, 0, st>>>(zrows, keys + (long long)k_used * rows, rows,
                                                                           tabs.t[k]);
    ++k_used;
  }
  UNIVL_CHECK_LAUNCH("embed table gradients");
  cudaFreeAsync(zrows, st);
  cudaFreeAsync(keys, st);
  if (int rc = partials_reduce(pg, parts, 1, EMB_H, dgamma, EMB_H, st)) return rc;
  return partials_reduce(pb, parts, 1, EMB_H, dbeta, EMB_H, st);
}

static EmbDrop make_emb_drop(float p, const unsigned long long* rng, unsigned long long stream) {
  EmbDrop d;
  d.on = p > 0.f;
  d.threshold = dropout_threshold16(p);
  d.scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  d.seed = 0;
  d.stream = stream;
  d.rng = rng;
  return d;
}
// backward kernels: ~2 rows per warp so the register-held table sums amortise their flush (4 rows per warp left the
// all-pairs source kernel with 5 warps per SM: 127 us, latency-bound)
static int emb_bwd_grid(long long rows) {
  long long blocks = (rows + EMB_WARPS * 2 - 1) / (EMB_WARPS * 2);
  const long long cap = (long long)device_sms() * 4;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}
static int emb_grid(long long rows) {
  long long blocks = (rows + EMB_WARPS - 1) / EMB_WARPS;
  const long long cap = (long long)device_sms() * 8;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace univl

using namespace univl;

extern "C" int univl_embed_text_fwd(const long long* ids, const long long* type_ids, const float* word,
                                    const float* pos, const float* type, const float* gamma, const float* beta,
                                    void* y, float* mean, float* rstd, int n_seq, int S, int H, int vocab, float eps,
                                    float p_drop, const unsigned long long* rng_state, unsigned long long stream_id,
                                    void* stream) {
  UNIVL_CHECK_ARG(H == EMB_H, "embed_text_fwd: hidden size must be %d (got %d)", EMB_H, H);
  UNIVL_CHECK_ARG(ids && word && pos && gamma && beta && y && mean && rstd, "embed_text_fwd: null pointer");
  UNIVL_CHECK_ARG(n_seq >= 0 && S > 0 && vocab > 0, "embed_text_fwd: bad shape");
  if (n_seq == 0) return UNIVL_OK;
  embed_text_fwd_kernel<<<emb_grid((long long)n_seq * S), EMB_WARPS * 32, 0, (cudaStream_t)stream>>>(
      ids, type_ids, word, pos, type, gamma, beta, (bf16*)y, mean, rstd, n_seq, S, vocab, eps,
      make_emb_drop(p_drop, rng_state, stream_id));
  UNIVL_CHECK_LAUNCH("embed_text_fwd");
  return UNIVL_OK;
}

extern "C" int univl_embed_text_bwd(const void* dy, const long long* ids, const long long* type_ids,
                                    const float* word, const float* pos, const float* type, const float* gamma,
                                    const float* mean, const float* rstd, float* dword, float* dpos, float* dtype,
                                    float* dgamma, float* dbeta, int n_seq, int S, int H, int vocab, float p_drop,
                                    const unsigned long long* rng_state, unsigned long long stream_id, void* stream) {
  UNIVL_CHECK_ARG(H == EMB_H, "embed_text_bwd: hidden size must be %d (got %d)", EMB_H, H);
  UNIVL_CHECK_ARG(dy && ids && word && pos && gamma && mean && rstd && dword && dpos && dgamma && dbeta,
                  "embed_text_bwd: null pointer");
  if (n_seq == 0) return UNIVL_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = (long long)n_seq * S;
  const int grid = emb_bwd_grid(rows);
  float *zrows, *pg, *pb;
  int* keys;
  if (int rc = scratch_alloc((void**)&zrows, (size_t)rows * EMB_H * sizeof(float), st)) return rc;
  if (int rc = scratch_alloc((void**)&keys, (size_t)3 * rows * sizeof(int), st)) return rc;
  if (int rc = scratch_alloc((void**)&pg, (size_t)grid * EMB_H * sizeof(float), st)) return rc;
  if (int rc = scratch_alloc((void**)&pb, (size_t)grid * EMB_H * sizeof(float), st)) return rc;
  embed_text_bwd_kernel<<<grid, EMB_WARPS * 32, 0, st>>>(
      (const bf16*)dy, ids, type_ids, word, pos, type, gamma, mean, rstd, zrows, keys, dtype != nullptr ? 1 : 0, pg, pb,
      n_seq, S, vocab, make_emb_drop(p_drop, rng_state, stream_id));
  UNIVL_CHECK_LAUNCH("embed_text_bwd");
  return emb_table_grads(zrows, keys, rows, {dword, dpos, dtype}, pg, pb, grid, dgamma, dbeta, st);
}

extern "C" int univl_embed_src_fwd(const void* a, const void* b, const float* pos, const float* type,
                                   const float* gamma, const float* beta, void* y, float* mean, float* rstd, int Na,
                                   int Wa, int Nb, int Fb, int all_pairs, int H, float eps, float p_drop,
                                   const unsigned long long* rng_state, unsigned long long stream_id, void* stream) {
  UNIVL_CHECK_ARG(H == EMB_H, "embed_src_fwd: hidden size must be %d (got %d)", EMB_H, H);
  UNIVL_CHECK_ARG(a && pos && gamma && beta && y && mean && rstd, "embed_src_fwd: null pointer");
  UNIVL_CHECK_ARG(Na >= 0 && Wa > 0 && Fb >= 0 && (Fb == 0 || (b != nullptr && Nb > 0)), "embed_src_fwd: bad shape");
  UNIVL_CHECK_ARG(all_pairs || Fb == 0 || Na == Nb, "embed_src_fwd: aligned mode needs Na == Nb");
  SrcCfg src{(const bf16*)a, (const bf16*)b, Na, Wa, Fb == 0 ? 1 : Nb, Fb, all_pairs && Fb > 0};
  const long long n_seq = src.all_pairs ? (long long)Na * Nb : Na;
  if (n_seq == 0) return UNIVL_OK;
  const long long rows_a = (long long)Na * Wa, rows_b = (long long)(Fb == 0 ? 0 : Nb) * Fb;
  dim3 grid(emb_grid(rows_a > rows_b ? rows_a : rows_b), Fb == 0 ? 1 : 2);
  embed_src_fwd_kernel<<<grid, EMB_WARPS * 32, 0, (cudaStream_t)stream>>>(
      src, pos, type, gamma, beta, (bf16*)y, mean, rstd, eps, make_emb_drop(p_drop, rng_state, stream_id));
  UNIVL_CHECK_LAUNCH("embed_src_fwd");
  return UNIVL_OK;
}

extern "C" int univl_embed_src_bwd(const void* dy, const void* a, const void* b, const float* pos, const float* type,
                                   const float* gamma, const float* mean, const float* rstd, void* da, void* db,
                                   float* dpos, float* dtype, float* dgamma, float* dbeta, int Na, int Wa, int Nb,
                                   int Fb, int all_pairs, int H, float p_drop, const unsigned long long* rng_state,
                                   unsigned long long stream_id, void* stream) {
  UNIVL_CHECK_ARG(H == EMB_H, "embed_src_bwd: hidden size must be %d (got %d)", EMB_H, H);
  UNIVL_CHECK_ARG(dy && a && pos && gamma && mean && rstd && dpos && dgamma && dbeta, "embed_src_bwd: null pointer");
  UNIVL_CHECK_ARG(Fb == 0 || b != nullptr, "embed_src_bwd: missing second source");
  SrcCfg src{(const bf16*)a, (const bf16*)b, Na, Wa, Fb == 0 ? 1 : Nb, Fb, all_pairs && Fb > 0};
  if (Na == 0) return UNIVL_OK;
  const long long rows_a = (long long)Na * Wa, rows_b = (long long)(Fb == 0 ? 0 : Nb) * Fb;
  dim3 grid(emb_bwd_grid(rows_a > rows_b ? rows_a : rows_b), Fb == 0 ? 1 : 2);
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = rows_a + rows_b;
  const int parts = (int)(grid.x * grid.y);
  float *zrows, *pg, *pb;
  int* keys;
  if (int rc = scratch_alloc((void**)&zrows, (size_t)rows * EMB_H * sizeof(float), st)) return rc;
  if (int rc = scratch_alloc((void**)&keys, (size_t)2 * rows * sizeof(int), st)) return rc;
  if (int rc = scratch_alloc((void**)&pg, (size_t)parts * EMB_H * sizeof(float), st)) return rc;
  if (int rc = scratch_alloc((void**)&pb, (size_t)parts * EMB_H * sizeof(float), st)) return rc;
  embed_src_bwd_kernel<<<grid, EMB_WARPS * 32, 0, st>>>(
      (const bf16*)dy, src, pos, type, gamma, mean, rstd, (bf16*)da, (bf16*)db, zrows, keys, dtype != nullptr ? 1 : 0,
      pg, pb, make_emb_drop(p_drop, rng_state, stream_id));
  UNIVL_CHECK_LAUNCH("embed_src_bwd");
  return emb_table_grads(zrows, keys, rows, {nullptr, dpos, dtype}, pg, pb, parts, dgamma, dbeta, st);
}
