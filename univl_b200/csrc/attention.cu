// univl_b200 — multi-head attention core for short sequences (S <= 256), forward and backward.
//
// Reference semantics (modules/module_bert.py:176-196, module_decoder.py:225-245):
//   scores = Q K^T / sqrt(d)  THEN  + additive mask (-10000 for masked keys — NOT -inf: a fully masked row keeps the
//   softmax of its raw scores);  P = softmax(scores);  P = dropout(P);  ctx = P V;  heads merged back to [T, H].
// The decoder's self-attention mask is (key padded OR key index > query index) -> -10000 ONCE (module_decoder.py:395).
//
// d = 64, whole K/V of one (sequence, head) live in shared memory, so softmax is exact two-pass (max+sum, then
// normalised P) and nothing of the [B, h, S, S] score tensor ever reaches HBM.  Tensor work uses warp-level
// mma.sync m16n8k16 bf16 (the S x S x 64 products are ~4 % of a layer's FLOPs; the projections around them run on
// wgmma — see gemm_wgmma.cu).  One CTA per (sequence, head); each warp owns 16 query rows (or 16 key rows in the
// dK/dV pass of backward) at a time.  Backward recomputes P from Q, K and the saved log-sum-exp, flash-style, with
// no atomics: dQ is produced by query-row tasks, dK/dV by key-row tasks that recompute the transposed tiles.
// Dropout masks are Philox(seed, stream, element) and regenerated identically in every pass.
#include <stdlib.h>

#include "common.cuh"

namespace univl {

constexpr int HD = 64;        // head dim
constexpr int LDS = 72;       // smem row stride in elements (144 B: conflict-free ldmatrix)
constexpr int ATT_FWD_WARPS = 8;   // upper bounds; the launch uses one warp per 16-row task up to these
constexpr int ATT_BWD_WARPS = 12;

struct AttnParams {
  const bf16 *q, *k, *v;
  long long ldq, ldk, ldv;
  bf16* o;
  long long ldo;
  float* lse;  // [n_seq, heads, Sq]
  const long long* mask_a;  // [Na, Wa]
  const long long* mask_b;  // [Nb, Fb] or null
  int Wa, Fb, Nb, all_pairs;
  int n_seq, heads, Sq, Sk, causal;
  float scale;
  uint32_t drop_threshold;
  float drop_scale;
  int drop_on;
  uint64_t seed, stream;
  const unsigned long long* rng;  // device {seed, epoch}, resolved at kernel entry (graph-replayable)
  // backward only
  const bf16* d_o;
  long long lddo;
  bf16 *dq, *dk, *dv;
  long long lddq, lddk, lddv;
  int share_tiles;  // backward: 1 = query-major pass shares P_drop / dS with the key-major pass through smem
  int rng_rowmajor; // backward: dropout layout of the fused QKV+attention forward kernel (fused_attn.cu), see tile_rng_rowmajor
  float *dbq, *dbk, *dbv;  // backward, optional: projection-bias gradients += column sums of dq / dk / dv  [heads*64]
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// copy `rows` x 64 bf16 (head slice) into smem [rows16][LDS], zero-filling rows >= rows
__device__ __forceinline__ void load_head_tile(bf16* dst, const bf16* src, long long ld, int rows, int rows16) {
  for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    bf16* d = dst + r * LDS + c * 8;
    if (r < rows) cp_async16(d, src + (long long)r * ld + c * 8);
    else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
  }
}

// additive key mask for this sequence into smem: 0 / -10000 for real keys, -inf for padding beyond Sk
__device__ __forceinline__ void build_key_mask(float* madd, const AttnParams& p, int seq, int Sk16) {
  const long long i = p.all_pairs ? seq / p.Nb : seq;
  const long long j = p.all_pairs ? seq % p.Nb : seq;
  for (int c = threadIdx.x; c < Sk16; c += blockDim.x) {
    float m;
    if (c >= p.Sk) m = -INFINITY;
    else {
      long long v = 1;
      if (p.mask_a != nullptr) {
        if (c < p.Wa) v = p.mask_a[i * p.Wa + c];
        else if (p.mask_b != nullptr) v = p.mask_b[j * p.Fb + (c - p.Wa)];
      }
      m = v != 0 ? 0.f : -10000.f;
    }
    madd[c] = m;
  }
}

// A-operand fragments (16 rows x 64 dims) of smem matrix X starting at row r0
__device__ __forceinline__ void load_a_frags(const bf16* X, int r0, int lane, uint32_t (&a)[4][4]) {
  const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) ldsm_x4(smem_u32(X + row * LDS + kc * 16 + (lane >> 4) * 8), a[kc]);
}

// C[16 x 16] = A(16 x 64) * Y^T where Y rows n0..n0+15 are the "n" index (keys or queries), contraction over dims
__device__ __forceinline__ void mma_a_yT(const uint32_t (&a)[4][4], const bf16* Y, int n0, int lane, float (&c)[2][4]) {
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) c[nb][e] = 0.f;
  const int row = n0 + (lane & 7) + (lane >> 4) * 8;
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    uint32_t b[4];
    ldsm_x4(smem_u32(Y + row * LDS + kc * 16 + ((lane >> 3) & 1) * 8), b);
    mma16816(c[0], a[kc], b[0], b[1]);
    mma16816(c[1], a[kc], b[2], b[3]);
  }
}

// acc[16 x 64] += P(16 x 16, bf16 A-fragments) * Z where Z rows k0..k0+15 are the contraction index
__device__ __forceinline__ void mma_p_z(const uint32_t (&pa)[4], const bf16* Z, int k0, int lane, float (&acc)[8][4]) {
  const int row = k0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int nd = 0; nd < 4; ++nd) {
    uint32_t b[4];
    ldsm_x4_t(smem_u32(Z + row * LDS + nd * 16 + (lane >> 4) * 8), b);
    mma16816(acc[2 * nd], pa, b[0], b[1]);
    mma16816(acc[2 * nd + 1], pa, b[2], b[3]);
  }
}

// Dropout randoms are laid out to match the mma fragment: for the 16 x 16 tile (query block qb, key block kb) the
// element (i, j) uses 16-bit word w = (j & 1) | ((i >> 3) & 1) << 1 | ((j >> 3) & 1) << 2 of
// Philox(seed, stream, ((bh * nQb + qb) * nKb + kb) * 32 + lane_f),  lane_f = (i & 7) << 2 | (j & 7) >> 1.
// In the query-major passes (forward, dQ) lane_f is the thread's own lane and its 8 tile elements are the 8 words of
// ONE call; the key-major pass (dK/dV) needs two calls per tile.
__device__ __forceinline__ uint4 tile_rng(const AttnParams& p, long long bh, int qb, int kb, int nQb, int nKb,
                                          int lane_f) {
  return philox4x32(p.seed, p.stream, (uint64_t)(((bh * nQb + qb) * (long long)nKb + kb) * 32 + lane_f));
}

// Row-major dropout layout (written by fused_attn.cu's forward): element (bh, query i, key j) is 16-bit word (j & 7) of
// Philox(seed, stream, (bh * Sq + i) * (Sk / 8) + j / 8).  In the mma fragment a thread (g, t) holds, of the 16 x 16 tile
// (q0, kb), rows i0 = q0 + g and i1 = i0 + 8 and keys kb*16 + nb*8 + 2t + {0, 1}: the two keys are the halves of 32-bit
// word t of the (row, nb) call.  The four lanes of a quad share the four calls (row i0 / i1) x (nb 0 / 1): lane t computes
// call c = t and the quad exchanges words with three XOR shuffles.  Returns w[rsel * 2 + nb] = word t of that call.
__device__ __forceinline__ void tile_rng_rowmajor(const AttnParams& p, long long bh, int q0, int kb, int lane,
                                                  uint32_t (&w)[4]) {
  const int g = lane >> 2, t = lane & 3;
  const int row = q0 + g + ((t >> 1) ? 8 : 0);
  const uint4 r = philox4x32(p.seed, p.stream,
                             (uint64_t)(bh * p.Sq + row) * (uint64_t)(p.Sk >> 3) + (uint64_t)(kb * 2 + (t & 1)));
  uint32_t got[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int want = t ^ k;  // component the partner lane (t ^ k) needs from this lane's call
    const uint32_t send = want == 0 ? r.x : want == 1 ? r.y : want == 2 ? r.z : r.w;
    got[k] = __shfl_xor_sync(0xffffffffu, send, k);  // = word t of call (t ^ k)
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int k = c ^ t;
    w[c] = k == 0 ? got[0] : k == 1 ? got[1] : k == 2 ? got[2] : got[3];
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------
// NKB > 0: the whole score row (<= NKB 16-key blocks) stays in registers — one QK^T pass, exact softmax, 2 * NKB
// independent accumulator chains for the tensor pipe.  NKB == 0: 16-key chunks with a stats pre-pass (any Sk <= 256).
template <int NKB>
__global__ void __launch_bounds__(ATT_FWD_WARPS * 32)  // (capping S=96 at 112 registers for 3 CTAs/SM measured 6% slower)
attention_fwd_kernel(const AttnParams p_in) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = p_in;
  if (p.drop_on && p.rng != nullptr) {
    p.seed = p.rng[0];
    p.stream += p.rng[1] << 20;
  }
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sQ = reinterpret_cast<bf16*>(smem_att);
  bf16* sK = sQ + Sq16 * LDS;
  bf16* sV = sK + Sk16 * LDS;
  float* madd = reinterpret_cast<float*>(sV + Sk16 * LDS);

  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  load_head_tile(sQ, p.q + (long long)seq * p.Sq * p.ldq + h * HD, p.ldq, p.Sq, Sq16);
  load_head_tile(sK, p.k + (long long)seq * p.Sk * p.ldk + h * HD, p.ldk, p.Sk, Sk16);
  load_head_tile(sV, p.v + (long long)seq * p.Sk * p.ldv + h * HD, p.ldv, p.Sk, Sk16);
  build_key_mask(madd, p, seq, Sk16);
  cp_async_wait_all();
  __syncthreads();

  for (int q0 = warp * 16; q0 < Sq16; q0 += (int)(blockDim.x >> 5) * 16) {
    uint32_t qa[4][4];
    load_a_frags(sQ, q0, lane, qa);
    const int i0 = q0 + g, i1 = q0 + g + 8;
    if constexpr (NKB > 0) {
      const int nkb = Sk16 >> 4;
      float s[NKB][2][4];
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) mma_a_yT(qa, sK, kb * 16, lane, s[kb]);
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) {
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = kb * 16 + nb * 8 + 2 * t + e;
              const float ma = madd[j];
              float a0 = ma, a1 = ma;
              if (p.causal) {
                if (j > i0 && a0 == 0.f) a0 = -10000.f;
                if (j > i1 && a1 == 0.f) a1 = -10000.f;
              }
              s[kb][nb][e] = s[kb][nb][e] * p.scale + a0;
              s[kb][nb][2 + e] = s[kb][nb][2 + e] * p.scale + a1;
              mx0 = fmaxf(mx0, s[kb][nb][e]);
              mx1 = fmaxf(mx1, s[kb][nb][2 + e]);
            }
        }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) {
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              s[kb][nb][e] = __expf(s[kb][nb][e] - mx0);
              s[kb][nb][2 + e] = __expf(s[kb][nb][2 + e] - mx1);
              sum0 += s[kb][nb][e];
              sum1 += s[kb][nb][2 + e];
            }
        }
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
      const float r0 = 1.0f / sum0, r1 = 1.0f / sum1;
      float o[8][4];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[nb][e] = 0.f;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) {
          uint4 rnd = make_uint4(0, 0, 0, 0);
          if (p.drop_on) rnd = tile_rng(p, bh, q0 >> 4, kb, Sq16 >> 4, Sk16 >> 4, lane);
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float p0 = s[kb][nb][e] * r0, p1 = s[kb][nb][2 + e] * r1;
              if (p.drop_on) {
                p0 = philox_u16(rnd, e | (nb << 2)) < p.drop_threshold ? p0 * p.drop_scale : 0.f;
                p1 = philox_u16(rnd, e | 2 | (nb << 2)) < p.drop_threshold ? p1 * p.drop_scale : 0.f;
              }
              s[kb][nb][e] = p0;
              s[kb][nb][2 + e] = p1;
            }
          uint32_t pa[4];
          pa[0] = pack_bf16x2(s[kb][0][0], s[kb][0][1]);
          pa[1] = pack_bf16x2(s[kb][0][2], s[kb][0][3]);
          pa[2] = pack_bf16x2(s[kb][1][0], s[kb][1][1]);
          pa[3] = pack_bf16x2(s[kb][1][2], s[kb][1][3]);
          mma_p_z(pa, sV, kb * 16, lane, o);
        }
      bf16* orow0 = p.o + ((long long)seq * p.Sq + i0) * p.ldo + h * HD;
      bf16* orow1 = p.o + ((long long)seq * p.Sq + i1) * p.ldo + h * HD;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        if (i0 < p.Sq) *reinterpret_cast<uint32_t*>(orow0 + nb * 8 + 2 * t) = pack_bf16x2(o[nb][0], o[nb][1]);
        if (i1 < p.Sq) *reinterpret_cast<uint32_t*>(orow1 + nb * 8 + 2 * t) = pack_bf16x2(o[nb][2], o[nb][3]);
      }
      if (t == 0 && p.lse != nullptr) {
        if (i0 < p.Sq) p.lse[bh * p.Sq + i0] = mx0 + __logf(sum0);
        if (i1 < p.Sq) p.lse[bh * p.Sq + i1] = mx1 + __logf(sum1);
      }
      continue;
    }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    // pass 1: row max and sum of exponentials
    for (int j0 = 0; j0 < Sk16; j0 += 16) {
      float s[2][4];
      mma_a_yT(qa, sK, j0, lane, s);
      float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = j0 + nb * 8 + 2 * t + e;
          float ma = madd[j];
          float a0 = ma, a1 = ma;
          if (p.causal) {
            if (j > i0 && a0 == 0.f) a0 = -10000.f;
            if (j > i1 && a1 == 0.f) a1 = -10000.f;
          }
          s[nb][e] = s[nb][e] * p.scale + a0;
          s[nb][2 + e] = s[nb][2 + e] * p.scale + a1;
          cm0 = fmaxf(cm0, s[nb][e]);
          cm1 = fmaxf(cm1, s[nb][2 + e]);
        }
      cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1));
      cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
      cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1));
      cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
      const float n0 = fmaxf(m0, cm0), n1 = fmaxf(m1, cm1);
      float e0 = 0.f, e1 = 0.f;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          e0 += __expf(s[nb][e] - n0);
          e1 += __expf(s[nb][2 + e] - n1);
        }
      e0 += __shfl_xor_sync(0xffffffffu, e0, 1);
      e0 += __shfl_xor_sync(0xffffffffu, e0, 2);
      e1 += __shfl_xor_sync(0xffffffffu, e1, 1);
      e1 += __shfl_xor_sync(0xffffffffu, e1, 2);
      l0 = l0 * __expf(m0 - n0) + e0;
      l1 = l1 * __expf(m1 - n1) + e1;
      m0 = n0;
      m1 = n1;
    }
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    // pass 2: normalised probabilities -> P V
    float o[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[nb][e] = 0.f;
    for (int j0 = 0; j0 < Sk16; j0 += 16) {
      float s[2][4];
      mma_a_yT(qa, sK, j0, lane, s);
      uint4 rnd = make_uint4(0, 0, 0, 0);
      if (p.drop_on) rnd = tile_rng(p, bh, q0 >> 4, j0 >> 4, Sq16 >> 4, Sk16 >> 4, lane);
#pragma unroll
      for (int nb = 0; nb < 2; ++nb) {
        const int jb = j0 + nb * 8 + 2 * t;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = jb + e;
          float ma = madd[j];
          float a0 = ma, a1 = ma;
          if (p.causal) {
            if (j > i0 && a0 == 0.f) a0 = -10000.f;
            if (j > i1 && a1 == 0.f) a1 = -10000.f;
          }
          float p0 = __expf(s[nb][e] * p.scale + a0 - m0) * inv0;
          float p1 = __expf(s[nb][2 + e] * p.scale + a1 - m1) * inv1;
          if (p.drop_on) {
            p0 = philox_u16(rnd, e | (nb << 2)) < p.drop_threshold ? p0 * p.drop_scale : 0.f;
            p1 = philox_u16(rnd, e | 2 | (nb << 2)) < p.drop_threshold ? p1 * p.drop_scale : 0.f;
          }
          s[nb][e] = p0;
          s[nb][2 + e] = p1;
        }
      }
      uint32_t pa[4];
      pa[0] = pack_bf16x2(s[0][0], s[0][1]);
      pa[1] = pack_bf16x2(s[0][2], s[0][3]);
      pa[2] = pack_bf16x2(s[1][0], s[1][1]);
      pa[3] = pack_bf16x2(s[1][2], s[1][3]);
      mma_p_z(pa, sV, j0, lane, o);
    }
    // store context rows (heads merged: column h*64 + d) and the row log-sum-exp
    bf16* orow0 = p.o + ((long long)seq * p.Sq + i0) * p.ldo + h * HD;
    bf16* orow1 = p.o + ((long long)seq * p.Sq + i1) * p.ldo + h * HD;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      if (i0 < p.Sq) *reinterpret_cast<uint32_t*>(orow0 + nb * 8 + 2 * t) = pack_bf16x2(o[nb][0], o[nb][1]);
      if (i1 < p.Sq) *reinterpret_cast<uint32_t*>(orow1 + nb * 8 + 2 * t) = pack_bf16x2(o[nb][2], o[nb][3]);
    }
    if (t == 0 && p.lse != nullptr) {
      if (i0 < p.Sq) p.lse[bh * p.Sq + i0] = m0 + __logf(l0);
      if (i1 < p.Sq) p.lse[bh * p.Sq + i1] = m1 + __logf(l1);
    }
  }
}

// ---- backward tasks ---------------------------------------------------------------------------------------------
struct BwdSmem {
  const bf16 *sQ, *sdO, *sK, *sV;
  const float *madd, *sLse, *sD;
  bf16 *sP, *sdS;  // SHARE mode: dropped probabilities / dS, [Sq16][ldp]
  int ldp;
  float* csum;     // per-task column sums of dq [nQ][64], dk [nK][64], dv [nK][64] (bias gradients), or null
  int nQ, nK;
};

// column sums of a 16 x 64 accumulator tile (rows g / g+8 of the fragment layout) into this task's own 64-float slot:
// butterfly over the 8 row groups (every lane ends up with the totals), then row group nb stores column block nb.  No
// atomics: the slots are summed over the tasks at the end of the kernel.  (Shared-memory float atomics from four lanes
// per warp cost 5.8 us per CTA: measured 893 vs 653 us on the cross-encoder shape.)
__device__ __forceinline__ void tile_colsum(const float (&acc)[8][4], float* slot, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    float c0 = acc[nb][0] + acc[nb][2], c1 = acc[nb][1] + acc[nb][3];
#pragma unroll
    for (int m = 4; m < 32; m <<= 1) {
      c0 += __shfl_xor_sync(0xffffffffu, c0, m);
      c1 += __shfl_xor_sync(0xffffffffu, c1, m);
    }
    if (g == nb) *reinterpret_cast<float2*>(slot + nb * 8 + 2 * t) = make_float2(c0, c1);
  }
}
template <bool SHARE>
__device__ __forceinline__ void bwd_dq_task(const AttnParams& p, const BwdSmem& sm, int task, int lane, int seq, int h,
                                            long long bh, int Sq16, int Sk16) {
  const bf16 *sQ = sm.sQ, *sdO = sm.sdO, *sK = sm.sK, *sV = sm.sV;
  const float *madd = sm.madd, *sLse = sm.sLse, *sD = sm.sD;
  bf16 *sP = sm.sP, *sdS = sm.sdS;
  const int ldp = sm.ldp;
  (void)sP; (void)sdS; (void)ldp;  // used only when SHARE
  // ---------------- dQ for 16 query rows ----------------
  const int q0 = task * 16;
  const int g = lane >> 2, t = lane & 3;
  uint32_t qa[4][4], da[4][4];
  load_a_frags(sQ, q0, lane, qa);
  load_a_frags(sdO, q0, lane, da);
  const int i0 = q0 + g, i1 = q0 + g + 8;
  const float lse0 = sLse[i0], lse1 = sLse[i1], D0 = sD[i0], D1 = sD[i1];
  float acc[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nb][e] = 0.f;
  for (int j0 = 0; j0 < Sk16; j0 += 16) {
    float s[2][4], dp[2][4];
    mma_a_yT(qa, sK, j0, lane, s);
    mma_a_yT(da, sV, j0, lane, dp);
    uint4 rnd = make_uint4(0, 0, 0, 0);
    uint32_t rw[4] = {0, 0, 0, 0};
    if (p.drop_on) {
      if (p.rng_rowmajor) tile_rng_rowmajor(p, bh, q0, j0 >> 4, lane, rw);
      else rnd = tile_rng(p, bh, q0 >> 4, j0 >> 4, Sq16 >> 4, Sk16 >> 4, lane);
    }
#pragma unroll
    for (int nb = 0; nb < 2; ++nb) {
      const int jb = j0 + nb * 8 + 2 * t;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = jb + e;
        float ma = madd[j];
        float a0 = ma, a1 = ma;
        if (p.causal) {
          if (j > i0 && a0 == 0.f) a0 = -10000.f;
          if (j > i1 && a1 == 0.f) a1 = -10000.f;
        }
        const float p0 = __expf(s[nb][e] * p.scale + a0 - lse0);
        const float p1 = __expf(s[nb][2 + e] * p.scale + a1 - lse1);
        float g0 = dp[nb][e], g1 = dp[nb][2 + e];
        float pk0 = p0, pk1 = p1;
        if (p.drop_on) {
          const uint32_t u0 = p.rng_rowmajor ? (e ? rw[nb] >> 16 : rw[nb] & 0xFFFFu) : philox_u16(rnd, e | (nb << 2));
          const uint32_t u1 = p.rng_rowmajor ? (e ? rw[2 + nb] >> 16 : rw[2 + nb] & 0xFFFFu)
                                             : philox_u16(rnd, e | 2 | (nb << 2));
          const bool kp0 = u0 < p.drop_threshold;
          const bool kp1 = u1 < p.drop_threshold;
          g0 = kp0 ? g0 * p.drop_scale : 0.f;
          g1 = kp1 ? g1 * p.drop_scale : 0.f;
          pk0 = kp0 ? p0 * p.drop_scale : 0.f;
          pk1 = kp1 ? p1 * p.drop_scale : 0.f;
        }
        s[nb][e] = p0 * (g0 - D0) * p.scale;
        s[nb][2 + e] = p1 * (g1 - D1) * p.scale;
        dp[nb][e] = pk0;  // dP is consumed: reuse its registers for the dropped probabilities
        dp[nb][2 + e] = pk1;
      }
      if (SHARE) {
        *reinterpret_cast<uint32_t*>(sP + i0 * ldp + jb) = pack_bf16x2(dp[nb][0], dp[nb][1]);
        *reinterpret_cast<uint32_t*>(sP + i1 * ldp + jb) = pack_bf16x2(dp[nb][2], dp[nb][3]);
        *reinterpret_cast<uint32_t*>(sdS + i0 * ldp + jb) = pack_bf16x2(s[nb][0], s[nb][1]);
        *reinterpret_cast<uint32_t*>(sdS + i1 * ldp + jb) = pack_bf16x2(s[nb][2], s[nb][3]);
      }
    }
    uint32_t pa[4];
    pa[0] = pack_bf16x2(s[0][0], s[0][1]);
    pa[1] = pack_bf16x2(s[0][2], s[0][3]);
    pa[2] = pack_bf16x2(s[1][0], s[1][1]);
    pa[3] = pack_bf16x2(s[1][2], s[1][3]);
    mma_p_z(pa, sK, j0, lane, acc);
  }
  if (sm.csum != nullptr) tile_colsum(acc, sm.csum + task * 64, lane);
  bf16* r0 = p.dq + ((long long)seq * p.Sq + i0) * p.lddq + h * HD;
  bf16* r1 = p.dq + ((long long)seq * p.Sq + i1) * p.lddq + h * HD;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    if (i0 < p.Sq) *reinterpret_cast<uint32_t*>(r0 + nb * 8 + 2 * t) = pack_bf16x2(acc[nb][0], acc[nb][1]);
    if (i1 < p.Sq) *reinterpret_cast<uint32_t*>(r1 + nb * 8 + 2 * t) = pack_bf16x2(acc[nb][2], acc[nb][3]);
  }
}

// key-major pass that recomputes the transposed score / dP tiles (any S <= 256)
__device__ __forceinline__ void bwd_dkdv_task_recompute(const AttnParams& p, const BwdSmem& sm, int task, int lane,
                                                        int seq, int h, long long bh, int Sq16, int Sk16) {
  const bf16 *sQ = sm.sQ, *sdO = sm.sdO, *sK = sm.sK, *sV = sm.sV;
  const float *madd = sm.madd, *sLse = sm.sLse, *sD = sm.sD;
  // ---------------- dK, dV for 16 key rows (transposed tiles) ----------------
  const int k0 = task * 16;
  const int g = lane >> 2, t = lane & 3;
  uint32_t ka[4][4], va[4][4];
  load_a_frags(sK, k0, lane, ka);
  load_a_frags(sV, k0, lane, va);
  const int j0r = k0 + g, j1r = k0 + g + 8;
  const float ma0 = madd[j0r], ma1 = madd[j1r];
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  for (int q0 = 0; q0 < Sq16; q0 += 16) {
    float st[2][4], dpt[2][4];
    mma_a_yT(ka, sQ, q0, lane, st);    // S^T tile: rows = keys, cols = queries
    mma_a_yT(va, sdO, q0, lane, dpt);  // dP^T tile
    float pd[2][4];
    uint4 rnd[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
    if (p.drop_on) {
      rnd[0] = tile_rng(p, bh, q0 >> 4, k0 >> 4, Sq16 >> 4, Sk16 >> 4, ((2 * t) << 2) | (g >> 1));
      rnd[1] = tile_rng(p, bh, q0 >> 4, k0 >> 4, Sq16 >> 4, Sk16 >> 4, ((2 * t + 1) << 2) | (g >> 1));
    }
#pragma unroll
    for (int nb = 0; nb < 2; ++nb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = q0 + nb * 8 + 2 * t + e;
        const float lse = sLse[i], D = sD[i];
        float a0 = ma0, a1 = ma1;
        if (p.causal) {
          if (j0r > i && a0 == 0.f) a0 = -10000.f;
          if (j1r > i && a1 == 0.f) a1 = -10000.f;
        }
        const float p0 = __expf(st[nb][e] * p.scale + a0 - lse);
        const float p1 = __expf(st[nb][2 + e] * p.scale + a1 - lse);
        float g0 = dpt[nb][e], g1 = dpt[nb][2 + e];
        float pk0 = p0, pk1 = p1;
        if (p.drop_on) {
          // element (query i, key j): word (j & 1) | ((i >> 3) & 1) << 1 | ((j >> 3) & 1) << 2 ; j = g (+8)
          const bool kp0 = philox_u16(rnd[e], (g & 1) | (nb << 1)) < p.drop_threshold;
          const bool kp1 = philox_u16(rnd[e], (g & 1) | (nb << 1) | 4) < p.drop_threshold;
          g0 = kp0 ? g0 * p.drop_scale : 0.f;
          g1 = kp1 ? g1 * p.drop_scale : 0.f;
          pk0 = kp0 ? p0 * p.drop_scale : 0.f;
          pk1 = kp1 ? p1 * p.drop_scale : 0.f;
        }
        pd[nb][e] = pk0;
        pd[nb][2 + e] = pk1;
        st[nb][e] = p0 * (g0 - D) * p.scale;
        st[nb][2 + e] = p1 * (g1 - D) * p.scale;
      }
    uint32_t pa[4], sa[4];
    pa[0] = pack_bf16x2(pd[0][0], pd[0][1]);
    pa[1] = pack_bf16x2(pd[0][2], pd[0][3]);
    pa[2] = pack_bf16x2(pd[1][0], pd[1][1]);
    pa[3] = pack_bf16x2(pd[1][2], pd[1][3]);
    sa[0] = pack_bf16x2(st[0][0], st[0][1]);
    sa[1] = pack_bf16x2(st[0][2], st[0][3]);
    sa[2] = pack_bf16x2(st[1][0], st[1][1]);
    sa[3] = pack_bf16x2(st[1][2], st[1][3]);
    mma_p_z(pa, sdO, q0, lane, dv);
    mma_p_z(sa, sQ, q0, lane, dk);
  }
  if (sm.csum != nullptr) {
    tile_colsum(dk, sm.csum + (sm.nQ + task) * 64, lane);
    tile_colsum(dv, sm.csum + (sm.nQ + sm.nK + task) * 64, lane);
  }
  bf16* kr0 = p.dk + ((long long)seq * p.Sk + j0r) * p.lddk + h * HD;
  bf16* kr1 = p.dk + ((long long)seq * p.Sk + j1r) * p.lddk + h * HD;
  bf16* vr0 = p.dv + ((long long)seq * p.Sk + j0r) * p.lddv + h * HD;
  bf16* vr1 = p.dv + ((long long)seq * p.Sk + j1r) * p.lddv + h * HD;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    if (j0r < p.Sk) {
      *reinterpret_cast<uint32_t*>(kr0 + nb * 8 + 2 * t) = pack_bf16x2(dk[nb][0], dk[nb][1]);
      *reinterpret_cast<uint32_t*>(vr0 + nb * 8 + 2 * t) = pack_bf16x2(dv[nb][0], dv[nb][1]);
    }
    if (j1r < p.Sk) {
      *reinterpret_cast<uint32_t*>(kr1 + nb * 8 + 2 * t) = pack_bf16x2(dk[nb][2], dk[nb][3]);
      *reinterpret_cast<uint32_t*>(vr1 + nb * 8 + 2 * t) = pack_bf16x2(dv[nb][2], dv[nb][3]);
    }
  }
}

// key-major pass on the tiles the query-major pass left in shared memory: dV = P_drop^T dO, dK = dS^T Q.  The A
// operand of both products is a transposed 16 x 16 block of a [query][key] matrix = ldmatrix.trans.
__device__ __forceinline__ void bwd_dkdv_task_shared(const AttnParams& p, const BwdSmem& sm, int task, int lane, int seq,
                                                     int h, int Sq16) {
  const int k0 = task * 16;
  const int g = lane >> 2, t = lane & 3;
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  // matrix m of the x4 load: query half (m >> 1), key half (m & 1)
  const int row_in = (lane & 7) + ((lane >> 4) & 1) * 8;
  const int col = k0 + ((lane >> 3) & 1) * 8;
  for (int q0 = 0; q0 < Sq16; q0 += 16) {
    uint32_t pa[4], sa[4];
    ldsm_x4_t(smem_u32(sm.sP + (q0 + row_in) * sm.ldp + col), pa);
    ldsm_x4_t(smem_u32(sm.sdS + (q0 + row_in) * sm.ldp + col), sa);
    mma_p_z(pa, sm.sdO, q0, lane, dv);
    mma_p_z(sa, sm.sQ, q0, lane, dk);
  }
  const int j0r = k0 + g, j1r = k0 + g + 8;
  if (sm.csum != nullptr) {
    tile_colsum(dk, sm.csum + (sm.nQ + task) * 64, lane);
    tile_colsum(dv, sm.csum + (sm.nQ + sm.nK + task) * 64, lane);
  }
  bf16* kr0 = p.dk + ((long long)seq * p.Sk + j0r) * p.lddk + h * HD;
  bf16* kr1 = p.dk + ((long long)seq * p.Sk + j1r) * p.lddk + h * HD;
  bf16* vr0 = p.dv + ((long long)seq * p.Sk + j0r) * p.lddv + h * HD;
  bf16* vr1 = p.dv + ((long long)seq * p.Sk + j1r) * p.lddv + h * HD;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    if (j0r < p.Sk) {
      *reinterpret_cast<uint32_t*>(kr0 + nb * 8 + 2 * t) = pack_bf16x2(dk[nb][0], dk[nb][1]);
      *reinterpret_cast<uint32_t*>(vr0 + nb * 8 + 2 * t) = pack_bf16x2(dv[nb][0], dv[nb][1]);
    }
    if (j1r < p.Sk) {
      *reinterpret_cast<uint32_t*>(kr1 + nb * 8 + 2 * t) = pack_bf16x2(dk[nb][2], dk[nb][3]);
      *reinterpret_cast<uint32_t*>(vr1 + nb * 8 + 2 * t) = pack_bf16x2(dv[nb][2], dv[nb][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ATT_BWD_WARPS * 32)
attention_bwd_kernel(const AttnParams p_in) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = p_in;
  if (p.drop_on && p.rng != nullptr) {
    p.seed = p.rng[0];
    p.stream += p.rng[1] << 20;
  }
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sQ = reinterpret_cast<bf16*>(smem_att);
  bf16* sdO = sQ + Sq16 * LDS;
  bf16* sK = sdO + Sq16 * LDS;
  bf16* sV = sK + Sk16 * LDS;
  float* madd = reinterpret_cast<float*>(sV + Sk16 * LDS);
  float* sLse = madd + Sk16;
  float* sD = sLse + Sq16;
  float* csum = sD + Sq16;  // [Sq16/16 + 2 * Sk16/16][64]

  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  (void)lane;

  load_head_tile(sQ, p.q + (long long)seq * p.Sq * p.ldq + h * HD, p.ldq, p.Sq, Sq16);
  load_head_tile(sdO, p.d_o + (long long)seq * p.Sq * p.lddo + h * HD, p.lddo, p.Sq, Sq16);
  load_head_tile(sK, p.k + (long long)seq * p.Sk * p.ldk + h * HD, p.ldk, p.Sk, Sk16);
  load_head_tile(sV, p.v + (long long)seq * p.Sk * p.ldv + h * HD, p.ldv, p.Sk, Sk16);
  build_key_mask(madd, p, seq, Sk16);
  cp_async_wait_all();
  __syncthreads();
  // D_i = sum_d dO[i,d] * O[i,d]   (8 lanes per row, 8 dims each); LSE rows (+inf on padding -> P = 0)
  for (int idx = threadIdx.x; idx < Sq16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    float part = 0.f;
    if (r < p.Sq) {
      const uint4 uo = *reinterpret_cast<const uint4*>(p.o + ((long long)seq * p.Sq + r) * p.ldo + h * HD + c * 8);
      const uint4 ud = *reinterpret_cast<const uint4*>(sdO + r * LDS + c * 8);
      const uint32_t wo[4] = {uo.x, uo.y, uo.z, uo.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = unpack_bf16x2(wo[j]), b = unpack_bf16x2(wd[j]);
        part += a.x * b.x + a.y * b.y;
      }
    }
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    part += __shfl_xor_sync(0xffffffffu, part, 4);
    if (c == 0) {
      sD[r] = part;
      sLse[r] = r < p.Sq ? p.lse[bh * p.Sq + r] : INFINITY;
    }
  }
  __syncthreads();

  const int nQ = Sq16 >> 4, nK = Sk16 >> 4;
  const int nw = (int)(blockDim.x >> 5);
  BwdSmem sm{sQ, sdO, sK, sV, madd, sLse, sD, nullptr, nullptr, Sk16 + 8, p.dbq != nullptr ? csum : nullptr, nQ, nK};
  if (p.share_tiles) {
    // S <= 128: the query-major pass leaves P_drop and dS in shared memory; the key-major pass only multiplies
    sm.sP = reinterpret_cast<bf16*>(csum + (nQ + 2 * nK) * 64);
    sm.sdS = sm.sP + Sq16 * sm.ldp;
    for (int task = warp; task < nQ; task += nw) bwd_dq_task<true>(p, sm, task, lane, seq, h, bh, Sq16, Sk16);
    __syncthreads();
    for (int task = warp; task < nK; task += nw) bwd_dkdv_task_shared(p, sm, task, lane, seq, h, Sq16);
  } else {
    for (int task = warp; task < nQ + nK; task += nw) {
      if (task < nQ) bwd_dq_task<false>(p, sm, task, lane, seq, h, bh, Sq16, Sk16);
      else bwd_dkdv_task_recompute(p, sm, task - nQ, lane, seq, h, bh, Sq16, Sk16);
    }
  }
  if (p.dbq != nullptr) {
    __syncthreads();
    for (int e = threadIdx.x; e < 192; e += blockDim.x) {
      const int kind = e >> 6, col = e & 63;
      const float* src = csum + (kind == 0 ? 0 : kind == 1 ? nQ : nQ + nK) * 64 + col;
      const int n = kind == 0 ? nQ : nK;
      float v = 0.f;
      for (int k = 0; k < n; ++k) v += src[k * 64];
      float* dst = kind == 0 ? p.dbq : kind == 1 ? p.dbk : p.dbv;
      dst[(long long)seq * p.heads * HD + h * HD + col] = v;  // this sequence's partial row
    }
  }
}

static int fill_common(AttnParams& p, const void* q, long long ldq, const void* k, long long ldk, const void* v,
                       long long ldv, const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb,
                       int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal, float scale, float p_drop,
                       const unsigned long long* rng_state, unsigned long long stream_id) {
  UNIVL_CHECK_ARG(q && k && v, "attention: null q/k/v");
  UNIVL_CHECK_ARG(n_seq >= 0 && heads > 0 && Sq > 0 && Sk > 0 && Sq <= 256 && Sk <= 256,
                  "attention: unsupported shape n_seq=%d heads=%d Sq=%d Sk=%d (S <= 256)", n_seq, heads, Sq, Sk);
  UNIVL_CHECK_ARG((ldq % 8) == 0 && (ldk % 8) == 0 && (ldv % 8) == 0, "attention: row strides must be multiples of 8");
  UNIVL_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0,
                  "attention: q/k/v must be 16-byte aligned");
  UNIVL_CHECK_ARG(mask_a == nullptr || Wa + Fb == Sk, "attention: mask parts (%d + %d) must cover Sk=%d", Wa, Fb, Sk);
  UNIVL_CHECK_ARG(!(Fb > 0 && mask_a != nullptr && mask_b == nullptr), "attention: missing second mask part");
  UNIVL_CHECK_ARG(!all_pairs || Nb > 0, "attention: all_pairs needs Nb > 0");
  UNIVL_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "attention: bad dropout probability");
  p.q = (const bf16*)q; p.k = (const bf16*)k; p.v = (const bf16*)v;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv;
  p.mask_a = mask_a; p.mask_b = mask_b; p.Wa = Wa; p.Fb = Fb; p.Nb = Nb > 0 ? Nb : 1; p.all_pairs = all_pairs;
  p.n_seq = n_seq; p.heads = heads; p.Sq = Sq; p.Sk = Sk; p.causal = causal; p.scale = scale;
  p.drop_on = p_drop > 0.f;
  p.drop_threshold = dropout_threshold16(p_drop);
  p.drop_scale = p_drop > 0.f ? 1.0f / (1.0f - p_drop) : 1.0f;
  UNIVL_CHECK_ARG(p_drop == 0.f || rng_state != nullptr, "attention: dropout needs rng_state");
  p.seed = 0; p.stream = stream_id; p.rng = rng_state;
  return UNIVL_OK;
}

}  // namespace univl

using namespace univl;

// ctx[T, heads*64] = softmax(Q K^T * scale + mask) V per (sequence, head).  q/k/v point at column 0 of head 0; head h
// reads columns [h*64, h*64+64).  Key mask = concat(mask_a[i, :Wa], mask_b[j, :Fb]) (int64 0/1) with (i, j) = (seq, seq)
// or, if all_pairs, (seq / Nb, seq % Nb); null mask_a = no padding mask.
extern "C" int univl_attention_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                   long long ldv, void* o, long long ldo, float* lse, const long long* mask_a,
                                   const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs, int n_seq, int heads,
                                   int Sq, int Sk, int causal, float scale, float p_drop, const unsigned long long* rng_state,
                                   unsigned long long stream_id, void* stream) {
  AttnParams p = {};
  if (int rc = fill_common(p, q, ldq, k, ldk, v, ldv, mask_a, mask_b, Wa, Fb, Nb, all_pairs, n_seq, heads, Sq, Sk,
                           causal, scale, p_drop, rng_state, stream_id))
    return rc;
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_fwd: bad output");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  const int Sq16 = (Sq + 15) & ~15, Sk16 = (Sk + 15) & ~15;
  const size_t smem = (size_t)(Sq16 + 2 * Sk16) * LDS * 2 + (size_t)Sk16 * 4;
  const int nkb = Sk16 / 16;
  void (*kern)(const AttnParams) = nkb <= 3 ? attention_fwd_kernel<3>
                                   : nkb <= 6 ? attention_fwd_kernel<6>
                                   : nkb <= 8 ? attention_fwd_kernel<8> : attention_fwd_kernel<0>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "attention_fwd smem attribute: %s", cudaGetErrorString(e));
  // warps per CTA: one per 16-row task up to 3, else two tasks per warp — smaller CTAs, more of them resident per SM, so
  // the load phase of one overlaps the math of the others (S = 96: 3-warp CTAs measured +0.8% on the whole step)
  const int fwd_tasks = Sq16 / 16;
  int fwd_warps = fwd_tasks <= 3 ? fwd_tasks : (fwd_tasks + 1) / 2;
  if (fwd_warps > ATT_FWD_WARPS) fwd_warps = ATT_FWD_WARPS;
  {
    static int cap = -1;  // tuning: UNIVL_ATT_FWD_WARPS=n caps the warps per CTA (more, smaller CTAs per SM)
    if (cap < 0) {
      const char* e = getenv("UNIVL_ATT_FWD_WARPS");
      cap = e ? atoi(e) : 0;
    }
    if (cap > 0 && fwd_warps > cap) fwd_warps = cap;
  }
  launch_kernel(kern, dim3(n_seq * heads), dim3(fwd_warps * 32), smem, (cudaStream_t)stream, p);
  UNIVL_CHECK_LAUNCH("attention_fwd");
  return UNIVL_OK;
}

extern "C" int univl_attention_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                   long long ldv, const void* o, long long ldo, const float* lse, const void* d_o,
                                   long long lddo, void* dq, long long lddq, void* dk, long long lddk, void* dv,
                                   long long lddv, const long long* mask_a, const long long* mask_b, int Wa, int Fb,
                                   int Nb, int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal, float scale,
                                   float p_drop, const unsigned long long* rng_state, unsigned long long stream_id,
                                   int rng_layout, float* dbq, float* dbk, float* dbv, void* stream) {
  AttnParams p = {};
  if (int rc = fill_common(p, q, ldq, k, ldk, v, ldv, mask_a, mask_b, Wa, Fb, Nb, all_pairs, n_seq, heads, Sq, Sk,
                           causal, scale, p_drop, rng_state, stream_id))
    return rc;
  UNIVL_CHECK_ARG(o && lse && d_o && dq && dk && dv, "attention_bwd: null pointer");
  UNIVL_CHECK_ARG((ldo % 8) == 0 && (lddo % 8) == 0 && (lddq % 2) == 0 && (lddk % 2) == 0 && (lddv % 2) == 0,
                  "attention_bwd: bad strides");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)const_cast<void*>(o); p.ldo = ldo; p.lse = const_cast<float*>(lse);
  p.d_o = (const bf16*)d_o; p.lddo = lddo;
  p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  UNIVL_CHECK_ARG((dbq == nullptr) == (dbk == nullptr) && (dbq == nullptr) == (dbv == nullptr),
                  "attention_bwd: bias-gradient pointers must be all set or all null");
  const int Sq16 = (Sq + 15) & ~15, Sk16 = (Sk + 15) & ~15;
  size_t smem = (size_t)(2 * Sq16 + 2 * Sk16) * LDS * 2 + (size_t)(Sk16 + 2 * Sq16 + (Sq16 / 16 + 2 * (Sk16 / 16)) * 64) * 4;
  p.share_tiles = (Sq16 <= 128 && Sk16 <= 128) ? 1 : 0;
  // rng_layout 1: masks were drawn by the fused QKV+attention forward kernel (row-major layout).  That kernel only runs
  // self-attention with S % 16 == 0, S <= 128, where the backward is always in tile-sharing mode.
  UNIVL_CHECK_ARG(rng_layout == 0 || rng_layout == 1, "attention_bwd: unknown rng_layout %d", rng_layout);
  UNIVL_CHECK_ARG(rng_layout == 0 || (p.share_tiles && Sq == Sk && (Sk % 16) == 0),
                  "attention_bwd: rng_layout 1 needs self-attention with S %% 16 == 0 and S <= 128");
  p.rng_rowmajor = rng_layout;
  if (p.share_tiles) smem += (size_t)2 * Sq16 * (Sk16 + 8) * 2;
  cudaError_t e = cudaFuncSetAttribute(attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "attention_bwd smem attribute: %s", cudaGetErrorString(e));
  int tasks = Sq16 / 16 + Sk16 / 16;
  if (p.share_tiles) tasks = Sq16 / 16 > Sk16 / 16 ? Sq16 / 16 : Sk16 / 16;  // the two passes run one after the other
  const int bwd_warps = tasks < ATT_BWD_WARPS ? tasks : ATT_BWD_WARPS;
  // bias gradients: one partial row per sequence, summed in sequence order after the kernel
  cudaStream_t st = (cudaStream_t)stream;
  float* outs[3] = {dbq, dbk, dbv};
  float* parts[3] = {nullptr, nullptr, nullptr};
  if (dbq != nullptr)
    for (int w = 0; w < 3; ++w)
      if (int rc = scratch_alloc((void**)&parts[w], (size_t)n_seq * heads * HD * sizeof(float), st)) return rc;
  p.dbq = parts[0]; p.dbk = parts[1]; p.dbv = parts[2];
  launch_kernel(attention_bwd_kernel, dim3(n_seq * heads), dim3(bwd_warps * 32), smem, st, p);
  UNIVL_CHECK_LAUNCH("attention_bwd");
  if (dbq != nullptr)
    for (int w = 0; w < 3; ++w)
      if (int rc = partials_reduce(parts[w], n_seq, 1, (long long)heads * HD, outs[w], (long long)heads * HD, st))
        return rc;
  return UNIVL_OK;
}
