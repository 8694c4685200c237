// univl_b200 — device helpers shared by the two mma.sync attention cores: attention.cu (S <= 256, whole K/V of one
// (sequence, head) in shared memory) and attention_long.cu (key-tiled, S <= 1024).  Both kernels use the same fragment
// layouts, the same key-mask row and the same dropout counter layout (tile_rng), so a (sequence, head, query, key)
// element draws the same dropout bit in either kernel.
#pragma once

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
//   ADDR_PAIR           all-pairs concat(a_i, b_j) of two sources (load_pair_tile, univl_attention_pair_fwd)
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

// copy `rows` x 64 bf16 (head slice) into smem [rows16][LDS], zero-filling rows >= rows
__device__ __forceinline__ void load_head_tile(bf16* dst, const bf16* src, long long ld, int rows, int rows16) {
  for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    bf16* d = dst + r * LDS + c * 8;
    if (r < rows) cp_async16(d, src + (long long)r * ld + c * 8);
    else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
  }
}

// load_head_tile for the pair forward: rows [r0, r0 + rows) of sequence `seq` = concat(text i, video j) (all-pairs
// pairing under ADDR_PAIR, the pair list vl.idx_a / vl.idx_b under ADDR_PAIR_LIST), whose row s is row i * Wa + s of
// the first source a (s < Wa) or row j * Fb + s - Wa of the second source b.  a / b point at column 0 of the q, k or v
// projections of each source.
template <int ADDR>
__device__ __forceinline__ void load_pair_tile(bf16* dst, const bf16* a, long long lda, const bf16* b, long long ldb,
                                               const AttnParams& p, const VarlenSrc& vl, int seq, int h, int r0,
                                               int rows, int rows16) {
  long long i, j;
  if constexpr (ADDR == ADDR_PAIR_LIST) {
    i = vl.idx_a[seq];
    j = vl.idx_b[seq];
  } else {
    pair_sources(seq, 1, p.n_seq, p.Nb, i, j);
  }
  const bf16* ra = a + i * p.Wa * lda + h * HD;
  const bf16* rb = b + j * p.Fb * ldb + h * HD;
  for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    const int s = r0 + r;
    bf16* d = dst + r * LDS + c * 8;
    if (r < rows) cp_async16(d, (s < p.Wa ? ra + (long long)s * lda : rb + (long long)(s - p.Wa) * ldb) + c * 8);
    else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
  }
}

// column 0 of row r of varlen sequence p (VarlenSrc); a / b point at column 0 of each source
__device__ __forceinline__ const bf16* varlen_row(const VarlenSrc& vl, const bf16* a, long long lda, const bf16* b,
                                                  long long ldb, int p, int r) {
  if (vl.idx_a == nullptr) return a + (long long)(vl.cu[p] + r) * lda;
  const int la = vl.len_a[p];
  return r < la ? a + (long long)vl.idx_a[vl.start_a[p] + r] * lda : b + (long long)vl.idx_b[vl.start_b[p] + r - la] * ldb;
}

// load_head_tile for the varlen forward: rows [r0, r0 + rows) of varlen sequence `seq`, zero-filling rows >= rows
__device__ __forceinline__ void load_varlen_tile(bf16* dst, const bf16* a, long long lda, const bf16* b, long long ldb,
                                                 const VarlenSrc& vl, int seq, int h, int r0, int rows, int rows16) {
  for (int idx = threadIdx.x; idx < rows16 * 8; idx += blockDim.x) {
    const int r = idx >> 3, c = idx & 7;
    bf16* d = dst + r * LDS + c * 8;
    if (r < rows) cp_async16(d, varlen_row(vl, a, lda, b, ldb, seq, r0 + r) + h * HD + c * 8);
    else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
  }
}

// the query rows [r0, r0 + rows) of varlen sequence `seq`: as its keys, except packed token-0 queries (row seq of q)
__device__ __forceinline__ void load_varlen_q(bf16* dst, const bf16* a, long long lda, const bf16* b, long long ldb,
                                              const VarlenSrc& vl, int seq, int h, int r0, int rows, int rows16) {
  if (vl.q_first && vl.idx_a == nullptr) load_head_tile(dst, a + (long long)seq * lda + h * HD, lda, rows, rows16);
  else load_varlen_tile(dst, a, lda, b, ldb, vl, seq, h, r0, rows, rows16);
}

// this CTA's varlen sequence `seq` into p's Sk / Sq
__device__ __forceinline__ void varlen_shape(AttnParams& p, const VarlenSrc& vl, int seq) {
  p.Sk = vl.cu[seq + 1] - vl.cu[seq];
  p.Sq = vl.q_first ? 1 : p.Sk;
}

// output row of query 0 of varlen sequence `seq` (its lse rows: row * heads + h).  Looked up where the output is stored
// rather than kept live through the kernel.
__device__ __forceinline__ long long varlen_out_row(const VarlenSrc& vl, int seq) {
  return vl.q_first ? seq : vl.cu[seq];
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

// Launch the forward kernels for a filled AttnParams (o, lse and the shape set, n_seq > 0).  addr: the row addressing
// (Addr); pb is the second source of ADDR_PAIR and ADDR_VARLEN_PAIR, vl the sequences of the varlen addressings, each
// ignored otherwise.  Under the varlen addressings p.Sq / p.Sk are the longest sequence's, which size the launch, and
// the output / lse rows are VarlenSrc's (lse[row * heads + h]).
// attention.cu: Sq, Sk <= 256; attention_long.cu: Sq, Sk <= 1024 and 12 heads.
int attention_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl, cudaStream_t stream);
int attention_long_fwd_launch(const AttnParams& p, Addr addr, const PairSrc& pb, const VarlenSrc& vl,
                              cudaStream_t stream);

}  // namespace univl
