// univl_b200 — key-tiled multi-head attention core for sequences of up to 1024 tokens, forward and backward.
//
// Same semantics as attention.cu (read its header): scores = Q K^T * scale, THEN + additive mask (-10000 for masked
// keys, -10000 once for (padded OR future) keys under `causal`, -inf only for the padding past Sk inside the last
// 16-key block); P = softmax; P = dropout(P); ctx = P V.  attention.cu keeps the whole K/V of one (sequence, head) in
// shared memory and so stops at 256 tokens; this kernel streams 64-row K/V tiles through a cp.async double buffer, so
// its shared memory is fixed apart from the 4-byte-per-key mask row (4 KB at 1024 keys).
//
// Forward: one CTA per (sequence, head, 64-query block), one warp per 16 query rows; an online row max and sum live
// in registers (flash-style), and the row log-sum-exp goes to lse[n_seq, heads, Sq] exactly as attention.cu writes it.
// Every key tile is visited: no tile is skipped for being masked, because a row whose keys are all masked attends to
// all of them with its raw scores, and a causal row whose keys are all padded attends to its future keys.
//
// Backward recomputes P from Q, K and the saved lse, with no floating-point atomics:
//   - dq kernel: one CTA per (sequence, head, 64-query block) streams K/V tiles; it also writes D_i = dO_i . O_i for
//     the dk/dv kernel;
//   - dk/dv kernel: one CTA per (sequence, head, 64-key block) streams Q/dO tiles in query order.
// The optional projection-bias gradients are written as one partial row per (sequence, block) and added in that order
// by partials_reduce, so every launch gives the same bits.
//
// Dropout uses attention.cu's tile_rng layout with nQb = Sq16 / 16 and nKb = Sk16 / 16 on the same mma fragments, so
// the dropout mask is a function of (sequence, head, query, key) alone and matches attention.cu's at any length both take.
#include "attention_common.cuh"

namespace univl {

constexpr int LONG_MAX_S = 1024;  // the longest position table of the model (the cross encoder's)
constexpr int LONG_HEADS = 12;
constexpr int LB = 64;            // query rows (forward, dq) or key rows (dk/dv) of one CTA: 4 warps x 16 rows
constexpr int LT = 64;            // rows of one streamed K/V (forward, dq) or Q/dO (dk/dv) tile
constexpr int LONG_WARPS = LB / 16;

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// this CTA's partial bias-gradient row: the sum of its warps' column-sum slots in warp order
__device__ __forceinline__ void write_partial_row(const float* slots, int nwarps, float* dst) {
  for (int col = threadIdx.x; col < HD; col += blockDim.x) {
    float v = 0.f;
    for (int w = 0; w < nwarps; ++w) v += slots[w * HD + col];
    dst[col] = v;
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward (ADDR: the row addressing of Q/K/V, attention_common.cuh Addr; under the pair addressings a key tile
// may straddle the boundary between the two sources.  Under the varlen addressings each CTA takes its own sequence's
// Sq / Sk, the query blocks past its Sq exit at once, and output / lse go to VarlenSrc's rows.)
// ------------------------------------------------------------------------------------------------------------
template <int ADDR>
__global__ void __launch_bounds__(LONG_WARPS * 32)
attention_long_fwd_kernel(const AttnParams p_in, const PairSrc pb, const VarlenSrc vl) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = resolve_rng(p_in);
  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int qbase = blockIdx.y * LB;
  // under the varlen addressings a CTA may have no query rows; the whole CTA leaves before any barrier
  if (!seq_shape<ADDR>(p, vl, seq) || qbase >= p.Sq) return;
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sQ = reinterpret_cast<bf16*>(smem_att);                 // [LB][LDS]
  bf16* sKV = sQ + LB * LDS;                                    // stage s: K at s * 2 * LT rows, V after it
  float* madd = reinterpret_cast<float*>(sKV + 4 * LT * LDS);  // [Sk16]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2;
  const int qrows = min(LB, p.Sq - qbase), qrows16 = min(LB, Sq16 - qbase);
  const int nT = (Sk16 + LT - 1) / LT;

  auto load_kv = [&](int tile, int stage) {
    const int k0 = tile * LT;
    bf16* sK = sKV + stage * 2 * LT * LDS;
    load_rows<ADDR, OP_K>(sK, p, pb, vl, seq, h, k0, min(LT, p.Sk - k0), LT);
    load_rows<ADDR, OP_V>(sK + LT * LDS, p, pb, vl, seq, h, k0, min(LT, p.Sk - k0), LT);
  };
  load_rows<ADDR, OP_Q>(sQ, p, pb, vl, seq, h, qbase, qrows, qrows16);
  build_key_mask(madd, p, seq, Sk16);
  load_kv(0, 0);
  cp_async_commit();

  const int q0 = qbase + warp * 16;  // this warp's first query row
  const bool active = warp * 16 < qrows16;
  const int i0 = q0 + g, i1 = i0 + 8;
  uint32_t qa[4][4];
  float o[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nb][e] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // l: this lane's share of the row sums

  for (int tile = 0; tile < nT; ++tile) {
    if (tile + 1 < nT) {
      load_kv(tile + 1, (tile + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (tile == 0) load_a_frags(sQ, warp * 16, lane, qa);
      const bf16* sK = sKV + (tile & 1) * 2 * LT * LDS;
      const bf16* sV = sK + LT * LDS;
      const int k0 = tile * LT;
      const int nkb = min(LT, Sk16 - k0) >> 4;
      float s[LT / 16][2][4];
#pragma unroll
      for (int kb = 0; kb < LT / 16; ++kb)
        if (kb < nkb) mma_a_yT(qa, sK, kb * 16, lane, s[kb]);
      float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
      for (int kb = 0; kb < LT / 16; ++kb)
        if (kb < nkb) {
          scale_mask(p, madd, k0 + kb * 16, i0, i1, lane, s[kb]);
          row_max(s[kb], cm0, cm1);
        }
      // every processed 16-key block holds a real key, so the running max is finite after the first tile
      const float n0 = fmaxf(m0, quad_max(cm0)), n1 = fmaxf(m1, quad_max(cm1));
      const float c0 = __expf(m0 - n0), c1 = __expf(m1 - n1);
      m0 = n0;
      m1 = n1;
      l0 *= c0;
      l1 *= c1;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        o[nb][0] *= c0;
        o[nb][1] *= c0;
        o[nb][2] *= c1;
        o[nb][3] *= c1;
      }
#pragma unroll
      for (int kb = 0; kb < LT / 16; ++kb)
        if (kb < nkb) {
          uint4 rnd = make_uint4(0, 0, 0, 0);
          if (p.drop_on) rnd = tile_rng(p, bh, q0 >> 4, (k0 >> 4) + kb, Sq16 >> 4, Sk16 >> 4, lane);
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float p0 = __expf(s[kb][nb][e] - m0), p1 = __expf(s[kb][nb][2 + e] - m1);
              l0 += p0;
              l1 += p1;
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
    }
    __syncthreads();  // the next iteration refills this stage
  }
  if (!active) return;
  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  const float r0 = 1.0f / l0, r1 = 1.0f / l1;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    o[nb][0] *= r0;
    o[nb][1] *= r0;
    o[nb][2] *= r1;
    o[nb][3] *= r1;
  }
  store_fwd_rows<ADDR>(p, vl, seq, h, q0, lane, o, m0, l0, m1, l1);
}

// ------------------------------------------------------------------------------------------------------------
// backward, query-major: dQ = dS K for one 64-query block; writes D_i = dO_i . O_i for the key-major kernel
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LONG_WARPS * 32)
attention_long_bwd_dq_kernel(const AttnParams p_in, float* __restrict__ Dg, float* __restrict__ part_q) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = resolve_rng(p_in);
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sQ = reinterpret_cast<bf16*>(smem_att);                 // [LB][LDS]
  bf16* sdO = sQ + LB * LDS;                                    // [LB][LDS]
  bf16* sKV = sdO + LB * LDS;                                   // 2 stages of K, V [LT][LDS]
  float* madd = reinterpret_cast<float*>(sKV + 4 * LT * LDS);  // [Sk16]
  float* sLse = madd + Sk16;                                    // [LB]
  float* sD = sLse + LB;                                        // [LB]
  float* csum = sD + LB;                                        // [LONG_WARPS][64]

  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int qbase = blockIdx.y * LB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2;
  const int qrows = min(LB, p.Sq - qbase), qrows16 = min(LB, Sq16 - qbase);
  const int nT = (Sk16 + LT - 1) / LT;

  auto load_kv = [&](int tile, int stage) {
    const int k0 = tile * LT;
    bf16* sK = sKV + stage * 2 * LT * LDS;
    load_rows<ADDR_DENSE, OP_K>(sK, p, {}, {}, seq, h, k0, min(LT, p.Sk - k0), LT);
    load_rows<ADDR_DENSE, OP_V>(sK + LT * LDS, p, {}, {}, seq, h, k0, min(LT, p.Sk - k0), LT);
  };
  load_rows<ADDR_DENSE, OP_Q>(sQ, p, {}, {}, seq, h, qbase, qrows, qrows16);
  load_rows<ADDR_DENSE, OP_DO>(sdO, p, {}, {}, seq, h, qbase, qrows, qrows16);
  cp_async_commit();
  load_kv(0, 0);
  cp_async_commit();
  build_key_mask(madd, p, seq, Sk16);
  cp_async_wait<1>();
  __syncthreads();
  stage_d_lse(p, sdO, seq, h, bh, qbase, qrows, qrows16, sD, sLse, Dg);

  const int q0 = qbase + warp * 16;
  const bool active = warp * 16 < qrows16;
  const int i0 = q0 + g, i1 = i0 + 8;
  uint32_t qa[4][4], da[4][4];
  float acc[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nb][e] = 0.f;
  float lse0 = 0.f, lse1 = 0.f, D0 = 0.f, D1 = 0.f;

  for (int tile = 0; tile < nT; ++tile) {
    if (tile + 1 < nT) {
      load_kv(tile + 1, (tile + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (tile == 0) {
        load_a_frags(sQ, warp * 16, lane, qa);
        load_a_frags(sdO, warp * 16, lane, da);
        lse0 = sLse[warp * 16 + g];
        lse1 = sLse[warp * 16 + g + 8];
        D0 = sD[warp * 16 + g];
        D1 = sD[warp * 16 + g + 8];
      }
      const bf16* sK = sKV + (tile & 1) * 2 * LT * LDS;
      const bf16* sV = sK + LT * LDS;
      const int k0 = tile * LT;
      const int nkb = min(LT, Sk16 - k0) >> 4;
      for (int kb = 0; kb < nkb; ++kb) {
        float s[2][4], dp[2][4];
        mma_a_yT(qa, sK, kb * 16, lane, s);
        mma_a_yT(da, sV, kb * 16, lane, dp);
        uint4 rnd = make_uint4(0, 0, 0, 0);
        if (p.drop_on) rnd = tile_rng(p, bh, q0 >> 4, (k0 >> 4) + kb, Sq16 >> 4, Sk16 >> 4, lane);
        scale_mask(p, madd, k0 + kb * 16, i0, i1, lane, s);
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            bwd_pair(p, s[nb][e], s[nb][2 + e], dp[nb][e], dp[nb][2 + e], lse0, lse1, D0, D1,
                     philox_u16(rnd, e | (nb << 2)), philox_u16(rnd, e | 2 | (nb << 2)));
        uint32_t pa[4];
        pack_a(s, pa);
        mma_p_z(pa, sK, kb * 16, lane, acc);
      }
    }
    __syncthreads();  // the next iteration refills this stage
  }
  const int nw = (int)(blockDim.x >> 5);
  if (active) {
    if (part_q != nullptr) tile_colsum(acc, csum + warp * HD, lane);
    store_rows(p.dq + h * HD, p.lddq, (long long)seq * p.Sq + qbase, warp * 16, qrows, lane, acc);
  }
  if (part_q != nullptr) {
    __syncthreads();
    write_partial_row(csum, min(nw, qrows16 >> 4),
                      part_q + (((long long)seq * gridDim.y + blockIdx.y) * p.heads + h) * HD);
  }
}

// ------------------------------------------------------------------------------------------------------------
// backward, key-major: dV = P_drop^T dO and dK = dS^T Q for one 64-key block, query tiles in ascending order
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LONG_WARPS * 32)
attention_long_bwd_dkdv_kernel(const AttnParams p_in, const float* __restrict__ Dg, float* __restrict__ part_k,
                               float* __restrict__ part_v) {
  pdl_trigger();
  pdl_wait();
  AttnParams p = resolve_rng(p_in);
  extern __shared__ __align__(16) uint8_t smem_att[];
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  bf16* sK = reinterpret_cast<bf16*>(smem_att);                 // [LB][LDS]
  bf16* sV = sK + LB * LDS;                                     // [LB][LDS]
  bf16* sQdO = sV + LB * LDS;                                   // 2 stages of Q, dO [LT][LDS]
  float* sLD = reinterpret_cast<float*>(sQdO + 4 * LT * LDS);  // 2 stages of lse [LT], D [LT]
  float* madd = sLD + 4 * LT;                                   // [Sk16]
  float* csum = madd + Sk16;                                    // dk slots [LONG_WARPS][64], then dv slots

  const int seq = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  const long long bh = blockIdx.x;
  const int kbase = blockIdx.y * LB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2;
  const int krows = min(LB, p.Sk - kbase), krows16 = min(LB, Sk16 - kbase);
  const int nT = (Sq16 + LT - 1) / LT;

  auto load_qdo = [&](int tile, int stage) {
    const int q0 = tile * LT;
    const int rows = min(LT, p.Sq - q0);
    bf16* sQ = sQdO + stage * 2 * LT * LDS;
    load_rows<ADDR_DENSE, OP_Q>(sQ, p, {}, {}, seq, h, q0, rows, LT);
    load_rows<ADDR_DENSE, OP_DO>(sQ + LT * LDS, p, {}, {}, seq, h, q0, rows, LT);
    float* ld = sLD + stage * 2 * LT;
    for (int r = threadIdx.x; r < LT; r += blockDim.x) {
      ld[r] = r < rows ? p.lse[bh * p.Sq + q0 + r] : INFINITY;  // +inf: P = 0 on the padding rows
      ld[LT + r] = r < rows ? Dg[bh * p.Sq + q0 + r] : 0.f;
    }
  };
  load_rows<ADDR_DENSE, OP_K>(sK, p, {}, {}, seq, h, kbase, krows, krows16);
  load_rows<ADDR_DENSE, OP_V>(sV, p, {}, {}, seq, h, kbase, krows, krows16);
  build_key_mask(madd, p, seq, Sk16);
  load_qdo(0, 0);
  cp_async_commit();

  const int k0 = kbase + warp * 16;  // this warp's first key row
  const bool active = warp * 16 < krows16;
  uint32_t ka[4][4], va[4][4];
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int nb = 0; nb < 8; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  float ma0 = 0.f, ma1 = 0.f;

  for (int tile = 0; tile < nT; ++tile) {
    if (tile + 1 < nT) {
      load_qdo(tile + 1, (tile + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      if (tile == 0) {
        load_a_frags(sK, warp * 16, lane, ka);
        load_a_frags(sV, warp * 16, lane, va);
        ma0 = madd[k0 + g];
        ma1 = madd[k0 + g + 8];
      }
      const bf16* sQ = sQdO + (tile & 1) * 2 * LT * LDS;
      const bf16* sdO = sQ + LT * LDS;
      const float* sLse = sLD + (tile & 1) * 2 * LT;
      const float* sD = sLse + LT;
      const int q0t = tile * LT;
      const int nqb = min(LT, Sq16 - q0t) >> 4;
      for (int qb = 0; qb < nqb; ++qb)
        dkdv_tile(p, ka, va, ma0, ma1, k0, sQ, sdO, sLse, sD, qb * 16, q0t + qb * 16, bh, Sq16 >> 4, Sk16 >> 4, lane,
                  dk, dv);
    }
    __syncthreads();  // the next iteration refills this stage
  }
  const int nw = (int)(blockDim.x >> 5);
  if (active) {
    if (part_k != nullptr) {
      tile_colsum(dk, csum + warp * HD, lane);
      tile_colsum(dv, csum + (LONG_WARPS + warp) * HD, lane);
    }
    store_rows(p.dk + h * HD, p.lddk, (long long)seq * p.Sk + kbase, warp * 16, krows, lane, dk);
    store_rows(p.dv + h * HD, p.lddv, (long long)seq * p.Sk + kbase, warp * 16, krows, lane, dv);
  }
  if (part_k != nullptr) {
    __syncthreads();
    const long long row = (((long long)seq * gridDim.y + blockIdx.y) * p.heads + h) * HD;
    write_partial_row(csum, min(nw, krows16 >> 4), part_k + row);
    write_partial_row(csum + LONG_WARPS * HD, min(nw, krows16 >> 4), part_v + row);
  }
}

int attention_long_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl,
                              cudaStream_t stream) {
  const int Sq16 = (p.Sq + 15) & ~15, Sk16 = (p.Sk + 15) & ~15;
  const size_t smem = (size_t)(LB + 4 * LT) * LDS * 2 + (size_t)Sk16 * 4;
  const FwdKernel kern =
      with_addr(addr, [](auto addr_c) -> FwdKernel { return attention_long_fwd_kernel<decltype(addr_c)::value>; });
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "attention_long_fwd smem attribute: %s", cudaGetErrorString(e));
  const int warps = Sq16 / 16 < LONG_WARPS ? Sq16 / 16 : LONG_WARPS;
  launch_kernel(kern, dim3(p.n_seq * p.heads, (Sq16 + LB - 1) / LB), dim3(warps * 32), smem, stream, p, pb, vl);
  UNIVL_CHECK_LAUNCH("attention_long_fwd");
  return UNIVL_OK;
}

}  // namespace univl

using namespace univl;

// As univl_attention_fwd, for 0 < Sq, Sk <= 1024 and 12 heads.
extern "C" int univl_attention_long_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                        long long ldv, void* o, long long ldo, float* lse, const long long* mask_a,
                                        const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs, int n_seq,
                                        int heads, int Sq, int Sk, int causal, float scale, float p_drop,
                                        const unsigned long long* rng_state, unsigned long long stream_id, void* stream) {
  AttnParams p = {};
  if (int rc = fill_common(p, q, ldq, k, ldk, v, ldv, mask_a, mask_b, Wa, Fb, Nb, all_pairs, n_seq, heads, Sq, Sk,
                           causal, scale, p_drop, rng_state, stream_id, LONG_MAX_S))
    return rc;
  UNIVL_CHECK_ARG(heads == LONG_HEADS, "attention_long_fwd: heads must be %d (got %d)", LONG_HEADS, heads);
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_long_fwd: bad output");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  return attention_long_fwd_launch(p, ADDR_DENSE, PairSrc{}, VarlenSrc{}, (cudaStream_t)stream);
}

// As univl_attention_bwd, for 0 < Sq, Sk <= 1024, 12 heads and rng_layout 0 (the forward was univl_attention_long_fwd
// or univl_attention_fwd).
extern "C" int univl_attention_long_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                        long long ldv, const void* o, long long ldo, const float* lse, const void* d_o,
                                        long long lddo, void* dq, long long lddq, void* dk, long long lddk, void* dv,
                                        long long lddv, const long long* mask_a, const long long* mask_b, int Wa, int Fb,
                                        int Nb, int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal,
                                        float scale, float p_drop, const unsigned long long* rng_state,
                                        unsigned long long stream_id, int rng_layout, float* dbq, float* dbk, float* dbv,
                                        void* stream) {
  AttnParams p = {};
  if (int rc = fill_common(p, q, ldq, k, ldk, v, ldv, mask_a, mask_b, Wa, Fb, Nb, all_pairs, n_seq, heads, Sq, Sk,
                           causal, scale, p_drop, rng_state, stream_id, LONG_MAX_S))
    return rc;
  UNIVL_CHECK_ARG(heads == LONG_HEADS, "attention_long_bwd: heads must be %d (got %d)", LONG_HEADS, heads);
  UNIVL_CHECK_ARG(o && lse && d_o && dq && dk && dv, "attention_long_bwd: null pointer");
  UNIVL_CHECK_ARG((ldo % 8) == 0 && (lddo % 8) == 0 && (lddq % 2) == 0 && (lddk % 2) == 0 && (lddv % 2) == 0,
                  "attention_long_bwd: bad strides");
  UNIVL_CHECK_ARG(rng_layout == 0, "attention_long_bwd: rng_layout must be 0 (got %d): the row-major layout is only "
                  "drawn by the fused forward, which runs at S <= 128", rng_layout);
  UNIVL_CHECK_ARG((dbq == nullptr) == (dbk == nullptr) && (dbq == nullptr) == (dbv == nullptr),
                  "attention_long_bwd: bias-gradient pointers must be all set or all null");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)const_cast<void*>(o); p.ldo = ldo; p.lse = const_cast<float*>(lse);
  p.d_o = (const bf16*)d_o; p.lddo = lddo;
  p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  const int Sq16 = (Sq + 15) & ~15, Sk16 = (Sk + 15) & ~15;
  const int nQB = (Sq16 + LB - 1) / LB, nKB = (Sk16 + LB - 1) / LB;
  const size_t smem_dq = (size_t)(2 * LB + 4 * LT) * LDS * 2 + (size_t)(Sk16 + 2 * LB + LONG_WARPS * HD) * 4;
  const size_t smem_dkdv = (size_t)(2 * LB + 4 * LT) * LDS * 2 + (size_t)(4 * LT + Sk16 + 2 * LONG_WARPS * HD) * 4;
  cudaError_t e = cudaFuncSetAttribute(attention_long_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem_dq);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(attention_long_bwd_dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem_dkdv);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "attention_long_bwd smem attribute: %s", cudaGetErrorString(e));
  cudaStream_t st = (cudaStream_t)stream;
  const long long row = (long long)heads * HD;
  float* Dg = nullptr;
  if (int rc = scratch_alloc((void**)&Dg, (size_t)n_seq * heads * Sq * sizeof(float), st)) return rc;
  // bias gradients: one partial row per (sequence, block), summed in that order after the kernels
  float* outs[3] = {dbq, dbk, dbv};
  float* parts[3] = {nullptr, nullptr, nullptr};
  const int nparts[3] = {n_seq * nQB, n_seq * nKB, n_seq * nKB};
  if (dbq != nullptr)
    for (int w = 0; w < 3; ++w)
      if (int rc = scratch_alloc((void**)&parts[w], (size_t)nparts[w] * row * sizeof(float), st)) return rc;
  const int qwarps = Sq16 / 16 < LONG_WARPS ? Sq16 / 16 : LONG_WARPS;
  const int kwarps = Sk16 / 16 < LONG_WARPS ? Sk16 / 16 : LONG_WARPS;
  launch_kernel(attention_long_bwd_dq_kernel, dim3(n_seq * heads, nQB), dim3(qwarps * 32), smem_dq, st, p, Dg,
                parts[0]);
  UNIVL_CHECK_LAUNCH("attention_long_bwd (dq)");
  launch_kernel(attention_long_bwd_dkdv_kernel, dim3(n_seq * heads, nKB), dim3(kwarps * 32), smem_dkdv, st, p,
                (const float*)Dg, parts[1], parts[2]);
  UNIVL_CHECK_LAUNCH("attention_long_bwd (dk/dv)");
  cudaFreeAsync(Dg, st);
  if (dbq != nullptr)
    for (int w = 0; w < 3; ++w)
      if (int rc = partials_reduce(parts[w], nparts[w], 1, row, outs[w], row, st)) return rc;
  return UNIVL_OK;
}
