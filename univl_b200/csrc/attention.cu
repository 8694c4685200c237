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
#include "attention_common.cuh"

namespace univl {

constexpr int ATT_FWD_WARPS = 8;   // upper bounds; the launch uses one warp per 16-row task up to these
constexpr int ATT_BWD_WARPS = 12;

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
// ADDR: the row addressing of Q/K/V (attention_common.cuh Addr).  Under the varlen addressings each CTA takes its own
// sequence's Sq / Sk (the launch is sized for the longest) and writes output / lse at VarlenSrc's rows.
template <int NKB, int ADDR>
__global__ void __launch_bounds__(ATT_FWD_WARPS * 32)  // (capping S=96 at 112 registers for 3 CTAs/SM measured 6% slower)
attention_fwd_kernel(const AttnParams p_in, const PairSrc pb, const VarlenSrc vl) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = resolve_rng(p_in);
  if (!seq_shape<ADDR>(p, vl, blockIdx.x / p.heads)) return;
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sQ = reinterpret_cast<bf16*>(smem_att);
  bf16* sK = sQ + Sq16 * LDS;
  bf16* sV = sK + Sk16 * LDS;
  float* madd = reinterpret_cast<float*>(sV + Sk16 * LDS);

  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2;

  load_rows<ADDR, OP_Q>(sQ, p, pb, vl, seq, h, 0, p.Sq, Sq16);
  load_rows<ADDR, OP_K>(sK, p, pb, vl, seq, h, 0, p.Sk, Sk16);
  load_rows<ADDR, OP_V>(sV, p, pb, vl, seq, h, 0, p.Sk, Sk16);
  build_key_mask(madd, p, seq, Sk16);
  cp_async_wait_all();
  __syncthreads();

  for (int q0 = warp * 16; q0 < Sq16; q0 += (int)(blockDim.x >> 5) * 16) {
    uint32_t qa[4][4];
    load_a_frags(sQ, q0, lane, qa);
    const int i0 = q0 + g, i1 = q0 + g + 8;
    float o[8][4];
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    if constexpr (NKB > 0) {
      const int nkb = Sk16 >> 4;
      float s[NKB][2][4];
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) mma_a_yT(qa, sK, kb * 16, lane, s[kb]);
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) {
          scale_mask(p, madd, kb * 16, i0, i1, lane, s[kb]);
          row_max(s[kb], m0, m1);
        }
      m0 = quad_max(m0);
      m1 = quad_max(m1);
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb)
        if (kb < nkb) {
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              s[kb][nb][e] = __expf(s[kb][nb][e] - m0);
              s[kb][nb][2 + e] = __expf(s[kb][nb][2 + e] - m1);
              l0 += s[kb][nb][e];
              l1 += s[kb][nb][2 + e];
            }
        }
      l0 = quad_sum(l0);
      l1 = quad_sum(l1);
      const float r0 = 1.0f / l0, r1 = 1.0f / l1;
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
                p0 = dropout(p, philox_u16(rnd, e | (nb << 2)), p0);
                p1 = dropout(p, philox_u16(rnd, e | 2 | (nb << 2)), p1);
              }
              s[kb][nb][e] = p0;
              s[kb][nb][2 + e] = p1;
            }
          uint32_t pa[4];
          pack_a(s[kb], pa);
          mma_p_z(pa, sV, kb * 16, lane, o);
        }
    } else {
      // pass 1: row max and sum of exponentials
      for (int j0 = 0; j0 < Sk16; j0 += 16) {
        float s[2][4];
        mma_a_yT(qa, sK, j0, lane, s);
        scale_mask(p, madd, j0, i0, i1, lane, s);
        float cm0 = -INFINITY, cm1 = -INFINITY;
        row_max(s, cm0, cm1);
        const float n0 = fmaxf(m0, quad_max(cm0)), n1 = fmaxf(m1, quad_max(cm1));
        float e0 = 0.f, e1 = 0.f;
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            e0 += __expf(s[nb][e] - n0);
            e1 += __expf(s[nb][2 + e] - n1);
          }
        l0 = l0 * __expf(m0 - n0) + quad_sum(e0);
        l1 = l1 * __expf(m1 - n1) + quad_sum(e1);
        m0 = n0;
        m1 = n1;
      }
      const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
      // pass 2: normalised probabilities -> P V
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
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = j0 + nb * 8 + 2 * (lane & 3) + e;
            const float2 a = mask_add(p, madd[j], i0, j, madd[j], i1, j);
            float p0 = __expf(s[nb][e] * p.scale + a.x - m0) * inv0;
            float p1 = __expf(s[nb][2 + e] * p.scale + a.y - m1) * inv1;
            if (p.drop_on) {
              p0 = dropout(p, philox_u16(rnd, e | (nb << 2)), p0);
              p1 = dropout(p, philox_u16(rnd, e | 2 | (nb << 2)), p1);
            }
            s[nb][e] = p0;
            s[nb][2 + e] = p1;
          }
        uint32_t pa[4];
        pack_a(s, pa);
        mma_p_z(pa, sV, j0, lane, o);
      }
    }
    store_fwd_rows<ADDR>(p, vl, seq, h, q0, lane, o, m0, l0, m1, l1);
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

template <bool SHARE>
__device__ __forceinline__ void bwd_dq_task(const AttnParams& p, const BwdSmem& sm, int task, int lane, int seq, int h,
                                            long long bh, int Sq16, int Sk16) {
  // ---------------- dQ for 16 query rows ----------------
  const int q0 = task * 16;
  const int g = lane >> 2, t = lane & 3;
  uint32_t qa[4][4], da[4][4];
  load_a_frags(sm.sQ, q0, lane, qa);
  load_a_frags(sm.sdO, q0, lane, da);
  const int i0 = q0 + g, i1 = q0 + g + 8;
  const float lse0 = sm.sLse[i0], lse1 = sm.sLse[i1], D0 = sm.sD[i0], D1 = sm.sD[i1];
  float acc[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nb][e] = 0.f;
  for (int j0 = 0; j0 < Sk16; j0 += 16) {
    float s[2][4], dp[2][4];
    mma_a_yT(qa, sm.sK, j0, lane, s);
    mma_a_yT(da, sm.sV, j0, lane, dp);
    uint4 rnd = make_uint4(0, 0, 0, 0);
    uint32_t rw[4] = {0, 0, 0, 0};
    if (p.drop_on) {
      if (p.rng_rowmajor) tile_rng_rowmajor(p, bh, q0, j0 >> 4, lane, rw);
      else rnd = tile_rng(p, bh, q0 >> 4, j0 >> 4, Sq16 >> 4, Sk16 >> 4, lane);
    }
    scale_mask(p, sm.madd, j0, i0, i1, lane, s);
#pragma unroll
    for (int nb = 0; nb < 2; ++nb) {
      const int jb = j0 + nb * 8 + 2 * t;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t u0 = p.rng_rowmajor ? (e ? rw[nb] >> 16 : rw[nb] & 0xFFFFu) : philox_u16(rnd, e | (nb << 2));
        const uint32_t u1 = p.rng_rowmajor ? (e ? rw[2 + nb] >> 16 : rw[2 + nb] & 0xFFFFu)
                                           : philox_u16(rnd, e | 2 | (nb << 2));
        // dP is consumed: its registers take the dropped probabilities
        bwd_pair(p, s[nb][e], s[nb][2 + e], dp[nb][e], dp[nb][2 + e], lse0, lse1, D0, D1, u0, u1);
      }
      if (SHARE) {
        *reinterpret_cast<uint32_t*>(sm.sP + i0 * sm.ldp + jb) = pack_bf16x2(dp[nb][0], dp[nb][1]);
        *reinterpret_cast<uint32_t*>(sm.sP + i1 * sm.ldp + jb) = pack_bf16x2(dp[nb][2], dp[nb][3]);
        *reinterpret_cast<uint32_t*>(sm.sdS + i0 * sm.ldp + jb) = pack_bf16x2(s[nb][0], s[nb][1]);
        *reinterpret_cast<uint32_t*>(sm.sdS + i1 * sm.ldp + jb) = pack_bf16x2(s[nb][2], s[nb][3]);
      }
    }
    uint32_t pa[4];
    pack_a(s, pa);
    mma_p_z(pa, sm.sK, j0, lane, acc);
  }
  if (sm.csum != nullptr) tile_colsum(acc, sm.csum + task * 64, lane);
  store_rows(p.dq + h * HD, p.lddq, (long long)seq * p.Sq, q0, p.Sq, lane, acc);
}

// the key-major tasks' epilogue: bias-gradient column sums and the dK / dV rows of this task's 16 keys
__device__ __forceinline__ void store_dkdv(const AttnParams& p, const BwdSmem& sm, int task, int lane, int seq, int h,
                                           const float (&dk)[8][4], const float (&dv)[8][4]) {
  if (sm.csum != nullptr) {
    tile_colsum(dk, sm.csum + (sm.nQ + task) * 64, lane);
    tile_colsum(dv, sm.csum + (sm.nQ + sm.nK + task) * 64, lane);
  }
  store_rows(p.dk + h * HD, p.lddk, (long long)seq * p.Sk, task * 16, p.Sk, lane, dk);
  store_rows(p.dv + h * HD, p.lddv, (long long)seq * p.Sk, task * 16, p.Sk, lane, dv);
}

// key-major pass that recomputes the transposed score / dP tiles (any S <= 256)
__device__ __forceinline__ void bwd_dkdv_task_recompute(const AttnParams& p, const BwdSmem& sm, int task, int lane,
                                                        int seq, int h, long long bh, int Sq16, int Sk16) {
  // ---------------- dK, dV for 16 key rows (transposed tiles) ----------------
  const int k0 = task * 16;
  const int g = lane >> 2;
  uint32_t ka[4][4], va[4][4];
  load_a_frags(sm.sK, k0, lane, ka);
  load_a_frags(sm.sV, k0, lane, va);
  const float ma0 = sm.madd[k0 + g], ma1 = sm.madd[k0 + g + 8];
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  for (int q0 = 0; q0 < Sq16; q0 += 16)
    dkdv_tile(p, ka, va, ma0, ma1, k0, sm.sQ, sm.sdO, sm.sLse, sm.sD, q0, q0, bh, Sq16 >> 4, Sk16 >> 4, lane, dk, dv);
  store_dkdv(p, sm, task, lane, seq, h, dk, dv);
}

// key-major pass on the tiles the query-major pass left in shared memory: dV = P_drop^T dO, dK = dS^T Q.  The A
// operand of both products is a transposed 16 x 16 block of a [query][key] matrix = ldmatrix.trans.
__device__ __forceinline__ void bwd_dkdv_task_shared(const AttnParams& p, const BwdSmem& sm, int task, int lane, int seq,
                                                     int h, int Sq16) {
  const int k0 = task * 16;
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
  store_dkdv(p, sm, task, lane, seq, h, dk, dv);
}

// ------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(ATT_BWD_WARPS * 32)
attention_bwd_kernel(const AttnParams p_in) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = resolve_rng(p_in);
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

  load_rows<ADDR_DENSE, OP_Q>(sQ, p, {}, {}, seq, h, 0, p.Sq, Sq16);
  load_rows<ADDR_DENSE, OP_DO>(sdO, p, {}, {}, seq, h, 0, p.Sq, Sq16);
  load_rows<ADDR_DENSE, OP_K>(sK, p, {}, {}, seq, h, 0, p.Sk, Sk16);
  load_rows<ADDR_DENSE, OP_V>(sV, p, {}, {}, seq, h, 0, p.Sk, Sk16);
  build_key_mask(madd, p, seq, Sk16);
  cp_async_wait_all();
  __syncthreads();
  stage_d_lse(p, sdO, seq, h, bh, 0, p.Sq, Sq16, sD, sLse, nullptr);
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

int attention_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl, cudaStream_t stream) {
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  const size_t smem = (size_t)(Sq16 + 2 * Sk16) * LDS * 2 + (size_t)Sk16 * 4;
  const int nkb = Sk16 / 16;
  const FwdKernel kern = with_addr(addr, [nkb](auto addr_c) -> FwdKernel {
    constexpr int ADDR = decltype(addr_c)::value;
    return nkb <= 3 ? attention_fwd_kernel<3, ADDR>
           : nkb <= 6 ? attention_fwd_kernel<6, ADDR>
           : nkb <= 8 ? attention_fwd_kernel<8, ADDR> : attention_fwd_kernel<0, ADDR>;
  });
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "attention_fwd smem attribute: %s", cudaGetErrorString(e));
  // warps per CTA: one per 16-row task up to 3, else two tasks per warp — smaller CTAs, more of them resident per SM, so
  // the load phase of one overlaps the math of the others (S = 96: 3-warp CTAs measured +0.8% on the whole step)
  const int fwd_tasks = Sq16 / 16;
  int fwd_warps = fwd_tasks <= 3 ? fwd_tasks : (fwd_tasks + 1) / 2;
  if (fwd_warps > ATT_FWD_WARPS) fwd_warps = ATT_FWD_WARPS;
  launch_kernel(kern, dim3(p.n_seq * p.heads), dim3(fwd_warps * 32), smem, stream, p, pb, vl);
  UNIVL_CHECK_LAUNCH("attention_fwd");
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
                           causal, scale, p_drop, rng_state, stream_id, 256))
    return rc;
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_fwd: bad output");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  return attention_fwd_launch(p, ADDR_DENSE, PairSrc{}, VarlenSrc{}, (cudaStream_t)stream);
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
                           causal, scale, p_drop, rng_state, stream_id, 256))
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
