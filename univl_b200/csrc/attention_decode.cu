// univl_b200 — single-query attention over indexed key rows: one decoder token per query row.
//
// Incremental caption decoding (caption.PrefixDecodeCache) attends with one query token per hypothesis, to keys that
// are rows of a shared K|V buffer picked by an int32 list: the self-attention cache's rows of the hypothesis' ancestors
// (one plane of rows per position, so reordering beams copies no K/V) or the valid rows of the hypothesis' own
// cross-encoder output.  With Sq = 1 the work is one pass over the listed K/V rows: bandwidth-bound, no tensor cores.
//
// One CTA per query row, all 12 heads.  A warp reads a whole K|V row (3 KB) in 16-byte vectors, each lane holding 8
// dims of 3 heads (vector j of lane l is vector l + 32 j of the row: head l / 8 + 4 j), so every row is loaded once for
// all heads; the 8 lanes of a head reduce its dot product with three shuffles.  Warp w takes keys w, w + 8, ... in
// chunks of DEC_CHUNK with an online softmax, one rescale per chunk.  The 8 warps' partial (max, sum, context) are then
// merged through shared memory in warp order: no floating-point atomics and no dependence on the SM count, so the bits
// depend on the inputs alone.
#include "common.cuh"

namespace univl {

constexpr int DEC_WARPS = 8;
constexpr int DEC_THREADS = DEC_WARPS * 32;
constexpr int DEC_HEADS = 12;
constexpr int DEC_H = DEC_HEADS * 64;     // 768 columns: 96 16-byte vectors, 3 per lane
constexpr int DEC_CHUNK = 4;              // keys per warp between rescales (24 16-byte loads in flight per lane)

__device__ __forceinline__ void bf16x8_to_f32(const uint4& u, float (&f)[8]) {
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}

__global__ void __launch_bounds__(DEC_THREADS)
attention_decode_kernel(const bf16* __restrict__ q, long long ldq, const bf16* __restrict__ kv, long long ldkv,
                        const int* __restrict__ key_rows, long long ld_rows, const int* __restrict__ n_keys,
                        const int* __restrict__ list_of_query, bf16* __restrict__ o, long long ldo,
                        float* __restrict__ lse, float scale) {
  __shared__ float s_acc[DEC_WARPS][DEC_H];
  __shared__ float s_m[DEC_WARPS][DEC_HEADS];
  __shared__ float s_l[DEC_WARPS][DEC_HEADS];
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x;
  const int list = list_of_query != nullptr ? list_of_query[r] : r;
  const int n = n_keys[list];
  if (n <= 0) return;
  const int* rows = key_rows + (long long)list * ld_rows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // the query, pre-multiplied by the scale (a power of two for head dim 64: exact)
  float qf[3][8];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const uint4 u = *reinterpret_cast<const uint4*>(q + (long long)r * ldq + (lane + 32 * j) * 8);
    bf16x8_to_f32(u, qf[j]);
#pragma unroll
    for (int e = 0; e < 8; ++e) qf[j][e] *= scale;
  }
  float m[3], l[3], acc[3][8];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    m[j] = -INFINITY;
    l[j] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[j][e] = 0.f;
  }

  for (int k0 = warp; k0 < n; k0 += DEC_WARPS * DEC_CHUNK) {
    uint4 kr[DEC_CHUNK][3], vr[DEC_CHUNK][3];
#pragma unroll
    for (int c = 0; c < DEC_CHUNK; ++c) {
      const int k = k0 + c * DEC_WARPS;
      if (k < n) {
        const bf16* row = kv + (long long)rows[k] * ldkv;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          kr[c][j] = *reinterpret_cast<const uint4*>(row + (lane + 32 * j) * 8);
          vr[c][j] = *reinterpret_cast<const uint4*>(row + DEC_H + (lane + 32 * j) * 8);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 3; ++j) kr[c][j] = vr[c][j] = make_uint4(0, 0, 0, 0);
      }
    }
    float s[DEC_CHUNK][3];
#pragma unroll
    for (int c = 0; c < DEC_CHUNK; ++c) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        float kf[8];
        bf16x8_to_f32(kr[c][j], kf);
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(qf[j][e], kf[e], d);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 4);
        s[c][j] = k0 + c * DEC_WARPS < n ? d : -INFINITY;
      }
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float mx = m[j];
#pragma unroll
      for (int c = 0; c < DEC_CHUNK; ++c) mx = fmaxf(mx, s[c][j]);
      const float corr = __expf(m[j] - mx);  // 0 on the first chunk (m = -inf), 1 when the maximum holds
      m[j] = mx;
      l[j] *= corr;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[j][e] *= corr;
#pragma unroll
      for (int c = 0; c < DEC_CHUNK; ++c) {
        const float p = __expf(s[c][j] - mx);  // 0 for a key past the end
        float vf[8];
        bf16x8_to_f32(vr[c][j], vf);
        l[j] += p;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[j][e] = fmaf(p, vf[e], acc[j][e]);
      }
    }
  }

  // per-warp partials to shared memory (a warp without keys leaves m = -inf, l = 0, acc = 0)
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int vec = lane + 32 * j;
#pragma unroll
    for (int e = 0; e < 8; ++e) s_acc[warp][vec * 8 + e] = acc[j][e];
    if ((lane & 7) == 0) {
      s_m[warp][vec >> 3] = m[j];
      s_l[warp][vec >> 3] = l[j];
    }
  }
  __syncthreads();
  // merge in warp order; every thread owns column pairs (2c, 2c + 1) of one head
  for (int c = threadIdx.x; c < DEC_H / 2; c += DEC_THREADS) {
    const int h = (2 * c) >> 6;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) M = fmaxf(M, s_m[w][h]);
    float L = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int w = 0; w < DEC_WARPS; ++w) {
      const float f = __expf(s_m[w][h] - M);  // 0 for a warp without keys
      L = fmaf(s_l[w][h], f, L);
      o0 = fmaf(s_acc[w][2 * c], f, o0);
      o1 = fmaf(s_acc[w][2 * c + 1], f, o1);
    }
    const float inv = 1.f / L;
    *reinterpret_cast<uint32_t*>(o + (long long)r * ldo + 2 * c) = pack_bf16x2(o0 * inv, o1 * inv);
    if (lse != nullptr && (2 * c & 63) == 0) lse[(long long)r * DEC_HEADS + h] = M + __logf(L);
  }
}

}  // namespace univl

using namespace univl;

extern "C" int univl_attention_decode_fwd(const void* q, long long ldq, const void* kv, long long ldkv,
                                          const int* key_rows, long long ld_rows, const int* n_keys,
                                          const int* list_of_query, int n_q, int heads, void* o, long long ldo,
                                          float* lse, float scale, void* stream) {
  UNIVL_CHECK_ARG(heads == DEC_HEADS, "attention_decode_fwd: heads must be 12 (got %d)", heads);
  UNIVL_CHECK_ARG(n_q >= 0, "attention_decode_fwd: bad n_q=%d", n_q);
  UNIVL_CHECK_ARG(q != nullptr && (ldq % 8) == 0 && ((uintptr_t)q & 15) == 0,
                  "attention_decode_fwd: q must be 16-byte aligned with a row stride that is a multiple of 8");
  UNIVL_CHECK_ARG(kv != nullptr && (ldkv % 8) == 0 && ldkv >= 2 * DEC_H && ((uintptr_t)kv & 15) == 0,
                  "attention_decode_fwd: kv must be 16-byte aligned with a row stride >= 1536 that is a multiple of 8");
  UNIVL_CHECK_ARG(key_rows != nullptr && n_keys != nullptr && ld_rows >= 0,
                  "attention_decode_fwd: null key_rows / n_keys or negative ld_rows");
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0 && ldo >= DEC_H && ((uintptr_t)o & 3) == 0,
                  "attention_decode_fwd: bad output (4-byte aligned, even row stride >= 768)");
  if (n_q == 0) return UNIVL_OK;
  launch_kernel(attention_decode_kernel, dim3(n_q), dim3(DEC_THREADS), 0, (cudaStream_t)stream, (const bf16*)q, ldq,
                (const bf16*)kv, ldkv, key_rows, ld_rows, n_keys, list_of_query, (bf16*)o, ldo, lse, scale);
  UNIVL_CHECK_LAUNCH("attention_decode_fwd");
  return UNIVL_OK;
}
