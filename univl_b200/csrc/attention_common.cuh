// univl_b200 — device helpers shared by the two mma.sync attention cores: attention.cu (S <= 256, whole K/V of one
// (sequence, head) in shared memory) and attention_long.cu (key-tiled, S <= 1024).  Both kernels use the same fragment
// layouts, the same key-mask row and the same dropout counter layout (tile_rng), so a (sequence, head, query, key)
// element draws the same dropout bit in either kernel.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace univl {

constexpr int HD = 64;        // head dim
constexpr int LDS = 72;       // smem row stride in elements (144 B: conflict-free ldmatrix)

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

// The pair forward's second source (univl_attention_pair_fwd): its q/k/v projections, read for sequence rows >= Wa.  A
// kernel argument of its own, so AttnParams and the kernels that do not read it keep their layout.
struct PairSrc {
  const bf16 *q, *k, *v;
  long long ldq, ldk, ldv;
};

// Row addressing of the forward kernels' Q/K/V tiles, a compile-time variant:
//   ADDR_DENSE          sequence s is rows [s * S, (s + 1) * S) of q/k/v (univl_attention_fwd)
//   ADDR_PAIR           all-pairs concat(a_i, b_j) of two sources (univl_attention_pair_fwd)
//   ADDR_VARLEN_PAIR    varlen sequences whose rows are picked from two sources by index lists (VarlenSrc)
//   ADDR_VARLEN_PACKED  varlen sequences stored back to back (VarlenSrc)
//   ADDR_PAIR_LIST      listed pairs concat(a_i, b_j), (i, j) = (VarlenSrc idx_a[s], idx_b[s]), rows as ADDR_PAIR
//                       (univl_attention_pair_list_fwd)
enum Addr : int { ADDR_DENSE = 0, ADDR_PAIR = 1, ADDR_VARLEN_PAIR = 2, ADDR_VARLEN_PACKED = 3, ADDR_PAIR_LIST = 4 };

// The varlen forward's sequences (univl_attention_varlen_fwd, univl_gather_rows_varlen).  Sequence p has
// Sk_p = cu[p + 1] - cu[p] rows, every one of them a real key (no mask).  Pair addressing (idx_a != null): row r < len_a[p]
// is row idx_a[start_a[p] + r] of source a, row r >= len_a[p] is row idx_b[start_b[p] + r - len_a[p]] of source b.
// Packed addressing: row r is row cu[p] + r of source a.  q_first: one query per sequence, its row 0 (under packed
// addressing the query rows are instead row p of q), and output row p; otherwise all Sk_p rows query, output at cu[p].
struct VarlenSrc {
  const int* cu;  // [n_seq + 1]
  const int *idx_a, *idx_b, *start_a, *start_b, *len_a;
  int q_first;
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

// column 0 of row r of varlen sequence p (VarlenSrc); a / b point at column 0 of each source
__device__ __forceinline__ const bf16* varlen_row(const VarlenSrc& vl, const bf16* a, long long lda, const bf16* b,
                                                  long long ldb, int p, int r) {
  if (vl.idx_a == nullptr) return a + (long long)(vl.cu[p] + r) * lda;
  const int la = vl.len_a[p];
  return r < la ? a + (long long)vl.idx_a[vl.start_a[p] + r] * lda : b + (long long)vl.idx_b[vl.start_b[p] + r - la] * ldb;
}

// ---- row addressing: what a kernel needs to know of its sequence, for any Addr ------------------------------------
// The kernels call these with their ADDR and never branch on it themselves.  The backward kernels use ADDR_DENSE.
enum Operand : int { OP_Q, OP_K, OP_V, OP_DO };

template <int ADDR>
constexpr bool addr_varlen = ADDR == ADDR_VARLEN_PAIR || ADDR == ADDR_VARLEN_PACKED;

// This CTA's sequence shape: under the varlen addressings its own Sk / Sq into p (the launch is sized for the longest).
// False for an empty sequence.
template <int ADDR>
__device__ __forceinline__ bool seq_shape(AttnParams& p, const VarlenSrc& vl, int seq) {
  if constexpr (addr_varlen<ADDR>) {
    p.Sk = vl.cu[seq + 1] - vl.cu[seq];
    p.Sq = vl.q_first ? 1 : p.Sk;
    return p.Sk > 0;
  }
  return true;
}

// rows [r0, r0 + rows) of operand OP of sequence `seq`, head h, into smem [rows16][LDS], zero-filling rows >= rows.
//   ADDR_DENSE: row s is row seq * S + s of the operand (S = Sq for Q / dO, Sk for K / V).
//   ADDR_PAIR, ADDR_PAIR_LIST: the sequence is concat(text i, video j), (i, j) the all-pairs pairing of seq or the listed
//     pair (vl.idx_a[seq], vl.idx_b[seq]); row s is row i * Wa + s of the first source (s < Wa), else row
//     j * Fb + s - Wa of the second (pb).
//   ADDR_VARLEN_*: row s is varlen_row's, except packed token-0 queries (q_first), which are row seq of q.
template <int ADDR, int OP>
__device__ __forceinline__ void load_rows(bf16* dst, const AttnParams& p, const PairSrc& pb, const VarlenSrc& vl, int seq,
                                          int h, int r0, int rows, int rows16) {
  const bf16* a = OP == OP_Q ? p.q : OP == OP_K ? p.k : OP == OP_V ? p.v : p.d_o;
  const long long lda = OP == OP_Q ? p.ldq : OP == OP_K ? p.ldk : OP == OP_V ? p.ldv : p.lddo;
  const bf16* b = OP == OP_Q ? pb.q : OP == OP_K ? pb.k : pb.v;
  const long long ldb = OP == OP_Q ? pb.ldq : OP == OP_K ? pb.ldk : pb.ldv;
  auto load = [&](auto row) {  // row(r): column h * HD of tile row r
    for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
      const int r = idx >> 3, c = idx & 7;
      bf16* d = dst + r * LDS + c * 8;
      if (r < rows) cp_async16(d, row(r) + c * 8);
      else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
    }
  };
  auto contiguous = [&](const bf16* src) { load([&](int r) { return src + (long long)r * lda; }); };
  if constexpr (ADDR == ADDR_PAIR || ADDR == ADDR_PAIR_LIST) {
    long long i, j;
    if constexpr (ADDR == ADDR_PAIR_LIST) {
      i = vl.idx_a[seq];
      j = vl.idx_b[seq];
    } else {
      pair_sources(seq, 1, p.n_seq, p.Nb, i, j);
    }
    const bf16* ra = a + i * p.Wa * lda + h * HD;
    const bf16* rb = b + j * p.Fb * ldb + h * HD;
    load([&](int r) {
      const int s = r0 + r;
      return s < p.Wa ? ra + (long long)s * lda : rb + (long long)(s - p.Wa) * ldb;
    });
  } else if constexpr (addr_varlen<ADDR>) {
    if (OP == OP_Q && vl.q_first && vl.idx_a == nullptr) contiguous(a + (long long)seq * lda + h * HD);
    else load([&](int r) { return varlen_row(vl, a, lda, b, ldb, seq, r0 + r) + h * HD; });
  } else {
    const int S = OP == OP_Q || OP == OP_DO ? p.Sq : p.Sk;
    contiguous(a + ((long long)seq * S + r0) * lda + h * HD);
  }
}

// output row of query 0 of sequence `seq`.  Looked up where the output is stored rather than kept live through the kernel.
template <int ADDR>
__device__ __forceinline__ long long out_row0(const AttnParams& p, const VarlenSrc& vl, int seq) {
  if constexpr (addr_varlen<ADDR>) return vl.q_first ? seq : vl.cu[seq];
  else return (long long)seq * p.Sq;
}

// lse index of query i of (sequence, head) bh, whose output row is ob + i: lse [n_seq, heads, Sq], or [rows, heads]
// under the varlen addressings
template <int ADDR>
__device__ __forceinline__ long long lse_index(const AttnParams& p, long long ob, long long bh, int h, int i) {
  if constexpr (addr_varlen<ADDR>) return (ob + i) * p.heads + h;
  else return bh * p.Sq + i;
}

// additive key mask for this sequence into smem: 0 / -10000 for real keys, -inf for padding beyond Sk
__device__ __forceinline__ void build_key_mask(float* madd, const AttnParams& p, int seq, int Sk16) {
  long long i, j;
  pair_sources(seq, p.all_pairs, p.n_seq, p.Nb, i, j);
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

// the kernel's parameters with the device RNG state {seed, epoch} resolved into seed / stream (graph-replayable)
__device__ __forceinline__ AttnParams resolve_rng(const AttnParams& p_in) {
  AttnParams p = p_in;
  if (p.drop_on && p.rng != nullptr) {
    p.seed = p.rng[0];
    p.stream += p.rng[1] << 20;
  }
  return p;
}

// additive masks of two (query i, key j) elements: the key's padding mask ma, or -10000 once for a future key of a
// causal row.  One causal test for the pair: a test per element costs the short forward kernels up to 7 registers.
__device__ __forceinline__ float2 mask_add(const AttnParams& p, float ma0, int i0, int j0, float ma1, int i1, int j1) {
  float a0 = ma0, a1 = ma1;
  if (p.causal) {
    if (j0 > i0 && a0 == 0.f) a0 = -10000.f;
    if (j1 > i1 && a1 == 0.f) a1 = -10000.f;
  }
  return make_float2(a0, a1);
}

// s = s * scale + mask over a query-major 16 x 16 tile: keys j0.., this lane's query rows i0 and i1 = i0 + 8
__device__ __forceinline__ void scale_mask(const AttnParams& p, const float* madd, int j0, int i0, int i1, int lane,
                                           float (&s)[2][4]) {
  const int t = lane & 3;
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = j0 + nb * 8 + 2 * t + e;
      const float2 a = mask_add(p, madd[j], i0, j, madd[j], i1, j);
      s[nb][e] = s[nb][e] * p.scale + a.x;
      s[nb][2 + e] = s[nb][2 + e] * p.scale + a.y;
    }
}

// this lane's share of the maxima of its two query rows of a 16 x 16 tile, into m0 / m1
__device__ __forceinline__ void row_max(const float (&s)[2][4], float& m0, float& m1) {
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      m0 = fmaxf(m0, s[nb][e]);
      m1 = fmaxf(m1, s[nb][2 + e]);
    }
}

// a row's max / sum over the four lanes of a quad, which hold its 16 x 16 tile columns
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// dropout of one element with 16-bit random u: kept and scaled by 1 / (1 - p_drop), or 0
__device__ __forceinline__ float dropout(const AttnParams& p, uint32_t u, float x) {
  return u < p.drop_threshold ? x * p.drop_scale : 0.f;
}

// a 16 x 16 fp32 accumulator tile as the bf16 A fragment of the next mma
__device__ __forceinline__ void pack_a(const float (&c)[2][4], uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(c[0][0], c[0][1]);
  a[1] = pack_bf16x2(c[0][2], c[0][3]);
  a[2] = pack_bf16x2(c[1][0], c[1][1]);
  a[3] = pack_bf16x2(c[1][2], c[1][3]);
}

// store a warp's 16 x 64 accumulator (fragment rows r0 + g and r0 + g + 8) as bf16 into col0[(row0 + r) * ld + col] for
// rows r < `rows`
__device__ __forceinline__ void store_rows(bf16* col0, long long ld, long long row0, int r0, int rows, int lane,
                                           const float (&acc)[8][4]) {
  const int g = lane >> 2, t = lane & 3;
  const int i0 = r0 + g, i1 = i0 + 8;
  bf16* row_0 = col0 + (row0 + i0) * ld;
  bf16* row_1 = col0 + (row0 + i1) * ld;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    if (i0 < rows) *reinterpret_cast<uint32_t*>(row_0 + nb * 8 + 2 * t) = pack_bf16x2(acc[nb][0], acc[nb][1]);
    if (i1 < rows) *reinterpret_cast<uint32_t*>(row_1 + nb * 8 + 2 * t) = pack_bf16x2(acc[nb][2], acc[nb][3]);
  }
}

// The forward's epilogue for one warp's 16 query rows q0..: the context rows (heads merged: column h * 64 + d) and the
// row log-sum-exp m + log(l)
template <int ADDR>
__device__ __forceinline__ void store_fwd_rows(const AttnParams& p, const VarlenSrc& vl, int seq, int h, int q0, int lane,
                                               const float (&o)[8][4], float m0, float l0, float m1, float l1) {
  const long long ob = out_row0<ADDR>(p, vl, seq);
  store_rows(p.o + h * HD, p.ldo, ob, q0, p.Sq, lane, o);
  const int i0 = q0 + (lane >> 2), i1 = i0 + 8;
  if ((lane & 3) == 0 && p.lse != nullptr) {
    if (i0 < p.Sq) p.lse[lse_index<ADDR>(p, ob, blockIdx.x, h, i0)] = m0 + __logf(l0);
    if (i1 < p.Sq) p.lse[lse_index<ADDR>(p, ob, blockIdx.x, h, i1)] = m1 + __logf(l1);
  }
}

// Backward staging of query rows [qbase, qbase + rows16) of (sequence seq, head h) = bh, rows >= rows being padding:
// sD[r] = D = dO . O (8 lanes per row, 8 dims each) and sLse[r] = lse (+inf on padding -> P = 0); D also to Dg if set.
__device__ __forceinline__ void stage_d_lse(const AttnParams& p, const bf16* sdO, int seq, int h, long long bh,
                                            int qbase, int rows, int rows16, float* sD, float* sLse, float* Dg) {
  for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    float part = 0.f;
    if (r < rows) {
      const uint4 uo =
          *reinterpret_cast<const uint4*>(p.o + ((long long)seq * p.Sq + qbase + r) * p.ldo + h * HD + c * 8);
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
      sLse[r] = r < rows ? p.lse[bh * p.Sq + qbase + r] : INFINITY;
      if (Dg != nullptr && r < rows) Dg[bh * p.Sq + qbase + r] = part;
    }
  }
}

// Two backward elements from their masked scores s0 / s1 (scale and mask applied), in place: P = exp(s - lse)
// recomputed, dP (dp) dropped with the 16-bit randoms u; s becomes dS = P * (dP_drop - D) * scale, dp becomes P_drop.
__device__ __forceinline__ void bwd_pair(const AttnParams& p, float& s0, float& s1, float& dp0, float& dp1, float lse0,
                                         float lse1, float D0, float D1, uint32_t u0, uint32_t u1) {
  const float p0 = __expf(s0 - lse0), p1 = __expf(s1 - lse1);
  float g0 = dp0, g1 = dp1, pk0 = p0, pk1 = p1;
  if (p.drop_on) {
    g0 = dropout(p, u0, g0);
    g1 = dropout(p, u1, g1);
    pk0 = dropout(p, u0, p0);
    pk1 = dropout(p, u1, p1);
  }
  s0 = p0 * (g0 - D0) * p.scale;
  s1 = p1 * (g1 - D1) * p.scale;
  dp0 = pk0;
  dp1 = pk1;
}

// One 16 x 16 step of the key-major dK / dV pass.  This warp's 16 keys k0.. (ka / va: their K / V A-fragments, ma0 /
// ma1: the key mask of rows k0 + g and k0 + g + 8) meet the 16 queries q0.., which are rows qr.. of sQ, sdO, sLse and
// sD.  Recomputes the transposed score and dP tiles, then dV += P_drop^T dO and dK += dS^T Q.
__device__ __forceinline__ void dkdv_tile(const AttnParams& p, const uint32_t (&ka)[4][4], const uint32_t (&va)[4][4],
                                          float ma0, float ma1, int k0, const bf16* sQ, const bf16* sdO,
                                          const float* sLse, const float* sD, int qr, int q0, long long bh, int nQb,
                                          int nKb, int lane, float (&dk)[8][4], float (&dv)[8][4]) {
  const int g = lane >> 2, t = lane & 3;
  const int j0r = k0 + g, j1r = j0r + 8;
  float st[2][4], dpt[2][4];
  mma_a_yT(ka, sQ, qr, lane, st);    // S^T tile: rows = keys, cols = queries
  mma_a_yT(va, sdO, qr, lane, dpt);  // dP^T tile
  uint4 rnd[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
  if (p.drop_on) {
    rnd[0] = tile_rng(p, bh, q0 >> 4, k0 >> 4, nQb, nKb, ((2 * t) << 2) | (g >> 1));
    rnd[1] = tile_rng(p, bh, q0 >> 4, k0 >> 4, nQb, nKb, ((2 * t + 1) << 2) | (g >> 1));
  }
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = nb * 8 + 2 * t + e, i = q0 + c;
      const float lse = sLse[qr + c], D = sD[qr + c];
      const float2 a = mask_add(p, ma0, i, j0r, ma1, i, j1r);
      st[nb][e] = st[nb][e] * p.scale + a.x;
      st[nb][2 + e] = st[nb][2 + e] * p.scale + a.y;
      // element (query i, key j): word (j & 1) | ((i >> 3) & 1) << 1 | ((j >> 3) & 1) << 2 ; j = g (+8)
      bwd_pair(p, st[nb][e], st[nb][2 + e], dpt[nb][e], dpt[nb][2 + e], lse, lse, D, D,
               philox_u16(rnd[e], (g & 1) | (nb << 1)), philox_u16(rnd[e], (g & 1) | (nb << 1) | 4));
    }
  uint32_t pa[4], sa[4];
  pack_a(dpt, pa);
  pack_a(st, sa);
  mma_p_z(pa, sdO, qr, lane, dv);
  mma_p_z(sa, sQ, qr, lane, dk);
}

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

// argument checks and the parameter fields both entry pairs share; max_s is the entry's sequence-length limit
static inline int fill_common(AttnParams& p, const void* q, long long ldq, const void* k, long long ldk, const void* v,
                              long long ldv, const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb,
                              int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal, float scale,
                              float p_drop, const unsigned long long* rng_state, unsigned long long stream_id,
                              int max_s) {
  UNIVL_CHECK_ARG(q && k && v, "attention: null q/k/v");
  UNIVL_CHECK_ARG(n_seq >= 0 && heads > 0 && Sq > 0 && Sk > 0 && Sq <= max_s && Sk <= max_s,
                  "attention: unsupported shape n_seq=%d heads=%d Sq=%d Sk=%d (S <= %d)", n_seq, heads, Sq, Sk, max_s);
  UNIVL_CHECK_ARG((ldq % 8) == 0 && (ldk % 8) == 0 && (ldv % 8) == 0, "attention: row strides must be multiples of 8");
  UNIVL_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0,
                  "attention: q/k/v must be 16-byte aligned");
  UNIVL_CHECK_ARG(mask_a == nullptr || Wa + Fb == Sk, "attention: mask parts (%d + %d) must cover Sk=%d", Wa, Fb, Sk);
  UNIVL_CHECK_ARG(!(Fb > 0 && mask_a != nullptr && mask_b == nullptr), "attention: missing second mask part");
  UNIVL_CHECK_ARG(!all_pairs || Nb > 0, "attention: all_pairs needs Nb > 0");
  UNIVL_CHECK_ARG(all_pairs >= 0 && (all_pairs <= 1 || (Nb % all_pairs == 0 && n_seq % Nb == 0)),
                  "attention: %d pairing groups need Nb=%d divisible by them and n_seq=%d divisible by Nb", all_pairs,
                  Nb, n_seq);
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

// the second source of the pair addressings (PairSrc): set, 16-byte aligned, row strides multiples of 8
static inline int fill_pair_src(PairSrc& pb, const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                long long ldv, const char* what) {
  UNIVL_CHECK_ARG(q && k && v, "%s: null second-source q/k/v", what);
  UNIVL_CHECK_ARG((ldq % 8) == 0 && (ldk % 8) == 0 && (ldv % 8) == 0,
                  "%s: second-source row strides must be multiples of 8", what);
  UNIVL_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0,
                  "%s: second-source q/k/v must be 16-byte aligned", what);
  pb = PairSrc{(const bf16*)q, (const bf16*)k, (const bf16*)v, ldq, ldk, ldv};
  return UNIVL_OK;
}

using FwdKernel = void (*)(const AttnParams, const PairSrc, const VarlenSrc);

// f(std::integral_constant<int, ADDR>{}) for the runtime addressing addr: how a launch picks its kernel instance
template <class F>
static inline FwdKernel with_addr(Addr addr, F f) {
  switch (addr) {
    case ADDR_PAIR: return f(std::integral_constant<int, ADDR_PAIR>{});
    case ADDR_PAIR_LIST: return f(std::integral_constant<int, ADDR_PAIR_LIST>{});
    case ADDR_VARLEN_PAIR: return f(std::integral_constant<int, ADDR_VARLEN_PAIR>{});
    case ADDR_VARLEN_PACKED: return f(std::integral_constant<int, ADDR_VARLEN_PACKED>{});
    default: return f(std::integral_constant<int, ADDR_DENSE>{});
  }
}

// Launch the forward kernels for a filled AttnParams (o, lse and the shape set, n_seq > 0).  addr: the row addressing
// (Addr); pb is the second source of ADDR_PAIR and ADDR_VARLEN_PAIR, vl the sequences of the varlen addressings, each
// ignored otherwise.  Under the varlen addressings p.Sq / p.Sk are the longest sequence's, which size the launch, and
// the output / lse rows are VarlenSrc's (lse[row * heads + h]).
// attention.cu: Sq, Sk <= 256; attention_long.cu: Sq, Sk <= 1024 and 12 heads.
int attention_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl, cudaStream_t stream);
int attention_long_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl,
                              cudaStream_t stream);

// the forward for Sk <= 1024 keys and 12 heads: attention.cu's kernels up to 256 keys, attention_long.cu's beyond
static inline int attention_fwd_any_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl,
                                           cudaStream_t stream) {
  if (p.Sk <= 256) return attention_fwd_launch(p, addr, pb, vl, stream);
  return attention_long_fwd_launch(p, addr, pb, vl, stream);
}

}  // namespace univl
