// univl_b200 — fused QKV-projection + multi-head self-attention on wgmma / TMA (sm_90a), forward and backward.
//
// Reference op sequence replaced (modules/module_bert.py:171-197 = module_visual.py:155-181 = module_cross.py:162-188;
// decoder self-attention module_decoder.py:220-247 with the causal mask of :385-396):
//     q,k,v = x Wq^T + bq, x Wk^T + bk, x Wv^T + bv ;  scores = q k^T / 8 + mask ;  P = dropout(softmax(scores)) ;
//     ctx = P v, heads merged.
// ONE kernel: the [T,2304] q/k/v tensor and the [B,12,S,S] scores never exist in HBM (q/k/v are optionally ALSO
// written out for the backward pass in training).
//
// Work item = (row block, head).  A row block is G = floor(128 / S) whole sequences = RB = G*S <= 128 consecutive
// token rows (S = 48 -> 96 rows, S = 96 -> 96, S = 128 -> 128); a CTA walks a contiguous range of items, heads
// fastest, so its x rows stay in L2 for the 12 heads.  RB is a template parameter (80, 96, 112 or 128), so every
// product below has its exact width.  Warp roles (384 threads): warpgroup 0 is the TMA producer, warpgroups 1 and 2
// each own 64 query rows of the block.  Per item:
//   1. projection   acc[64, 192] = x[64 rows, 768] . Wqkv_h[192, 768]^T   12 k-blocks x 4 wgmma m64n192k16 per
//                   warpgroup; x and the three 64-row weight slices arrive by TMA into a 4-stage mbarrier ring
//   2. drain        registers (+bias) -> bf16 -> Q, K, V shared-memory tiles in the 128B-swizzled operand layout (one
//                   physical layout serves Q as K-major A, K as K-major B, V as MN-major B)
//   3. S = Q K^T    4 wgmma (m64, N = RB, k16) into registers
//   4. softmax      in registers, one quad of lanes per query row: scale + additive mask (-10000 padding / causal,
//                   block-diagonal across the packed sequences), exact max / sum, Philox dropout, log-sum-exp -> HBM
//   5. O = P V      P stays in registers as the A operand (RB / 16 wgmma m64n64k16), O -> merged-head context rows.
#include <stdlib.h>

#include "common.cuh"
#include "tmap.cuh"
#include "wgmma.cuh"

namespace univl {

constexpr int FA_THREADS = 384;                 // TMA producer warpgroup + two consumer warpgroups
constexpr int FA_STAGES = 4;
constexpr int FA_KB = 12;                       // 768 / 64 k-blocks
constexpr int FA_X_BYTES = 128 * 64 * 2;        // 16 KB: x rows of one k-block
constexpr int FA_W_BYTES = 192 * 64 * 2;        // 24 KB: q/k/v weight rows of one head, one k-block
constexpr int FA_STAGE_BYTES = FA_X_BYTES + FA_W_BYTES;
constexpr int FA_TILE_BYTES = 128 * 128;        // one [128 rows][64 bf16] operand tile
constexpr int FA_OFF_Q = FA_STAGES * FA_STAGE_BYTES;
constexpr int FA_OFF_K = FA_OFF_Q + FA_TILE_BYTES;
constexpr int FA_OFF_V = FA_OFF_K + FA_TILE_BYTES;
constexpr int FA_OFF_MADD = FA_OFF_V + FA_TILE_BYTES;         // 128 floats
constexpr int FA_OFF_BAR = FA_OFF_MADD + 512;                 // full[FA_STAGES] empty[FA_STAGES]
constexpr int FA_SMEM_BYTES = FA_OFF_BAR + 2 * FA_STAGES * 8 + 1024;
static_assert(FA_SMEM_BYTES <= 227 * 1024, "shared memory per block");

struct FusedAttnParams {
  int T, S, G, RB, n_seq, heads, n_blocks;
  const float* bias;          // [3 * heads * 64]
  bf16* o;
  long long ldo;
  float* lse;                 // [n_seq, heads, S]
  const long long* mask_a;
  const long long* mask_b;
  int Wa, Fb, Nb, all_pairs, causal;
  float scale;
  int drop_on;
  uint32_t drop_threshold;
  float drop_scale;
  const unsigned long long* rng;
  uint64_t stream;
  int store_qkv;
  int x_box_rows;   // rows of the x TMA box: RB when RB % 32 == 0 (see the launcher), else 128
};

// items [begin, end) of this CTA: contiguous ranges, the first (total % grid) CTAs take one more
__device__ __forceinline__ void fa_item_range(int total, int& begin, int& end) {
  const int per = total / (int)gridDim.x, rem = total % (int)gridDim.x;
  const int b = (int)blockIdx.x;
  begin = b * per + min(b, rem);
  end = begin + per + (b < rem ? 1 : 0);
}

// additive key mask of row block rb (log2 domain) for key column `kcol` of the block: 0 / -10000; shared by the heads
__device__ __forceinline__ float fa_key_mask(const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb,
                                             int all_pairs, int S, int G, int n_seq, int NK, int rb, int kcol) {
  if (kcol >= NK) return 0.f;
  const int g = kcol / S, kpos = kcol - g * S;
  const long long seq = (long long)rb * G + g;
  long long mv = 1;
  if (mask_a != nullptr && seq < n_seq) {
    const long long mi = all_pairs ? seq / Nb : seq, mj = all_pairs ? seq % Nb : seq;
    if (kpos < Wa) mv = mask_a[mi * Wa + kpos];
    else if (mask_b != nullptr) mv = mask_b[mj * Fb + (kpos - Wa)];
  }
  return mv != 0 ? 0.f : -10000.0f * 1.44269504088896340736f;
}

// Dropout keep bits of one query row, NK keys.  Layout (row-major, matched by univl_attention_bwd rng_layout 1): element
// (bh, query, key) is 16-bit word (key & 7) of Philox(seed, stream, (bh * S + query) * (S / 8) + key / 8).  In the wgmma
// fragment the four lanes of a quad share a row and lane q holds keys 8 j + 2 q + {0, 1}, i.e. 32-bit word q of group
// j's Philox output: each lane computes every fourth group and a 4 x 4 transpose over the quad hands out the words, so
// one Philox call still decides 8 elements.  Bit 2 j + e of keep[j / 16] = key 8 j + 2 q + e kept.
template <int NK>
__device__ __forceinline__ void fa_keep_bits(uint64_t seed, uint64_t stream, uint64_t base, int c0_groups,
                                             uint32_t thr, int quad, uint32_t (&keep)[(NK / 8 + 15) / 16]) {
#pragma unroll
  for (int i = 0; i < (NK / 8 + 15) / 16; ++i) keep[i] = 0;
#pragma unroll
  for (int j4 = 0; j4 < (NK / 8 + 3) / 4; ++j4) {
    const int mine = 4 * j4 + quad;  // group this lane draws
    const uint4 r = philox4x32(seed, stream, base + (uint64_t)(int64_t)(mine - c0_groups));
    const uint32_t wv[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int src = quad ^ k;
      const uint32_t send = wv[src];  // word `src` is what lane (quad ^ k) needs
      const uint32_t got = k == 0 ? send : __shfl_xor_sync(0xffffffffu, send, k);
      const int gj = 4 * j4 + src;    // group whose word quad lane `quad` received
      if (gj < NK / 8) {
        const uint32_t bits = ((got & 0xFFFFu) < thr ? 1u : 0u) | ((got >> 16) < thr ? 2u : 0u);
        keep[gj >> 4] |= bits << (2 * (gj & 15));
      }
    }
  }
}

template <int NK>
__global__ void __launch_bounds__(FA_THREADS, 1)
fused_qkv_attention_fwd_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                               const __grid_constant__ CUtensorMap tmap_qkv, const FusedAttnParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + FA_OFF_BAR);
  uint64_t* empty_bar = full_bar + FA_STAGES;
  float* madd = reinterpret_cast<float*>(smem + FA_OFF_MADD);

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    if (p.store_qkv) tma_prefetch_desc(&tmap_qkv);
    for (int s = 0; s < FA_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  int item_begin, item_end;
  fa_item_range(p.n_blocks * p.heads, item_begin, item_end);

  if (wg == 0) {
    // ------------------------------------------ TMA producer ------------------------------------------
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int w = item_begin; w < item_end; ++w) {
        const int rb = w / p.heads, h = w - rb * p.heads;
        const int r0 = rb * p.RB;
        for (int kb = 0; kb < FA_KB; ++kb, ++it) {
          const int s = it % FA_STAGES;
          const uint32_t ph = (it / FA_STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sx = smem + s * FA_STAGE_BYTES;
          uint8_t* sw = sx + FA_X_BYTES;
          // the x box holds only the RB rows that carry queries / keys (tile rows RB..127 feed only rows nobody reads)
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(p.x_box_rows * 128 + FA_W_BYTES));
          tma_load_2d(sx, &tmap_x, &full_bar[s], kb * 64, r0);  // rows >= T arrive as zeros
#pragma unroll
          for (int m = 0; m < 3; ++m)  // q / k / v weight rows of head h: rows m*H + h*64 of Wqkv[3H, 768]
            tma_load_2d(sw + m * 8192, &tmap_w, &full_bar[s], kb * 64, m * p.heads * 64 + h * 64);
        }
      }
    }
    return;
  }

  // ------------------------------------------ consumer warpgroups ------------------------------------------
  regs_alloc<232>();
  const int c = wg - 1;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31, quad = lane & 3;
  const int r_lo = c * 64 + warp * 16 + (lane >> 2);  // tile rows r_lo and r_lo + 8 of the fragments
  const uint64_t seed = (p.drop_on && p.rng != nullptr) ? p.rng[0] : 0ull;   // device-side {seed, epoch}
  const uint64_t stream = p.stream + ((p.drop_on && p.rng != nullptr) ? (p.rng[1] << 20) : 0ull);
  const float sl2 = p.scale * 1.44269504088896340736f;
  const float neg_big = -10000.0f * 1.44269504088896340736f;
  const uint32_t sQ = smem_u32(smem + FA_OFF_Q), sK = smem_u32(smem + FA_OFF_K), sV = smem_u32(smem + FA_OFF_V);
  int cur_rb = -1;
  uint32_t it = 0;
  for (int w = item_begin; w < item_end; ++w) {
    const int rb = w / p.heads, h = w - rb * p.heads;

    // ---- 1. projection ----
    float acc[96];
#pragma unroll
    for (int e = 0; e < 96; ++e) acc[e] = 0.f;
    int prev_s = -1;
    for (int kb = 0; kb < FA_KB; ++kb, ++it) {
      const int s = it % FA_STAGES;
      const uint32_t ph = (it / FA_STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint32_t sx = smem_u32(smem + s * FA_STAGE_BYTES) + c * (64 * 128);
      const uint32_t sw = smem_u32(smem + s * FA_STAGE_BYTES) + FA_X_BYTES;
      wgmma_fence();
      fence_regs(acc);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        WgmmaSS<192>::mma<0, 0>(acc, make_smem_desc_sw128(sx + 32 * k, 16, 1024),
                                make_smem_desc_sw128(sw + 32 * k, 16, 1024), (kb > 0 || k > 0) ? 1 : 0);
      wgmma_commit();
      fence_regs(acc);
      wgmma_wait<1>();
      if (prev_s >= 0 && t == 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (t == 0) mbar_arrive(&empty_bar[prev_s]);

    // ---- 2. Q / K / V tiles (and the key mask when the row block changes) ----
    if (p.store_qkv && t == 0) bulk_wait_read<0>();  // the previous item's q/k/v stores have read the tiles
    named_bar(1, 256);  // both warpgroups are done with the previous item's tiles and mask
    if (rb != cur_rb && c == 0)
      madd[t] = fa_key_mask(p.mask_a, p.mask_b, p.Wa, p.Fb, p.Nb, p.all_pairs, p.S, p.G, p.n_seq, NK, rb, t);
    cur_rb = rb;
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      const float* bias = p.bias + m * p.heads * 64 + h * 64;
      uint8_t* tile = smem + FA_OFF_Q + m * FA_TILE_BYTES;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * quad));
        const float* a = acc + 4 * (8 * m + j);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = r_lo + 8 * hr;
          *reinterpret_cast<uint32_t*>(tile + r * 128 + ((j ^ (r & 7)) << 4) + quad * 4) =
              pack_bf16x2(a[2 * hr] + bb.x, a[2 * hr + 1] + bb.y);
        }
      }
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core and the bulk-copy engine
    named_bar(2, 256);
    if (p.store_qkv && t == 0) {
      // this warpgroup's 64 rows, in 32-row boxes that start inside the block (a box may spill past RB into the next
      // block's rows: with x_box_rows = 128 those are that block's true values)
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
          const int rr = c * 64 + hb * 32;
          if (rr < p.RB)
            tma_store_2d(&tmap_qkv, smem + FA_OFF_Q + m * FA_TILE_BYTES + rr * 128, m * p.heads * 64 + h * 64,
                         rb * p.RB + rr);
        }
      bulk_commit();
    }

    // ---- 3. S = Q K^T ----
    float sa[NK / 2];
#pragma unroll
    for (int e = 0; e < NK / 2; ++e) sa[e] = 0.f;
    wgmma_fence();
    fence_regs(sa);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      WgmmaSS<NK>::template mma<0, 0>(sa, make_smem_desc_sw128(sQ + c * (64 * 128) + 32 * k, 16, 1024),
                                      make_smem_desc_sw128(sK + 32 * k, 16, 1024), k > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sa);

    // ---- 4. softmax of rows r_lo (hr = 0) and r_lo + 8 (hr = 1) ----
    uint32_t pa[NK / 16][4];  // P as the register A operand of O = P V
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r_lo + 8 * hr;
      const int g = row / p.S, c0 = g * p.S, qpos = row - c0;
      const long long seq = (long long)rb * p.G + g;
      const bool valid = row < p.RB && seq < p.n_seq;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < NK / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = 8 * j + 2 * quad + e;
          const bool own = valid && key >= c0 && key < c0 + p.S;
          float a = madd[key];
          if (p.causal && (key - c0) > qpos && a == 0.f) a = neg_big;
          const float v = own ? fmaf(sa[4 * j + 2 * hr + e], sl2, a) : -INFINITY;
          sa[4 * j + 2 * hr + e] = v;
          mx = fmaxf(mx, v);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mref = valid ? mx : 0.f;  // rows without a query: keep the arithmetic finite
      float l = 0.f;
#pragma unroll
      for (int j = 0; j < NK / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = ex2_approx(sa[4 * j + 2 * hr + e] - mref);  // exp2(-inf) = 0 outside the own sequence
          sa[4 * j + 2 * hr + e] = v;
          l += v;
        }
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = valid ? (p.drop_on ? p.drop_scale : 1.0f) / l : 0.f;
      const long long bh = seq * p.heads + h;
      uint32_t keep[(NK / 8 + 15) / 16];
      if (p.drop_on) {
        const uint64_t base = ((uint64_t)bh * p.S + qpos) * (uint64_t)(p.S >> 3);
        fa_keep_bits<NK>(seed, stream, base, c0 >> 3, p.drop_threshold, quad, keep);
      }
#pragma unroll
      for (int j = 0; j < NK / 8; ++j) {
        float pr0 = sa[4 * j + 2 * hr] * inv, pr1 = sa[4 * j + 2 * hr + 1] * inv;
        if (p.drop_on) {
          const uint32_t kb2 = keep[j >> 4] >> (2 * (j & 15));
          if (!(kb2 & 1u)) pr0 = 0.f;
          if (!(kb2 & 2u)) pr1 = 0.f;
        }
        // A fragment of k-slice j / 2: {row, k 0-7}, {row + 8, k 0-7}, {row, k 8-15}, {row + 8, k 8-15}
        pa[j >> 1][(j & 1) * 2 + hr] = pack_bf16x2(pr0, pr1);
      }
      if (quad == 0 && valid && p.lse != nullptr)
        p.lse[bh * p.S + qpos] = (mx + __log2f(l)) * 0.69314718055994530942f;
    }

    // ---- 5. O = P V, merged-head context rows ----
    float oa[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) oa[e] = 0.f;
    wgmma_fence();
    fence_regs(oa);
#pragma unroll
    for (int kk = 0; kk < NK / 16; ++kk)  // contraction over keys: V [keys][64] is the MN-major B operand
      WgmmaRS<64>::mma<1>(oa, pa[kk], make_smem_desc_sw128(sV + kk * 2048, FA_TILE_BYTES, 1024), kk > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(oa);
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r_lo + 8 * hr;
      const long long tok = (long long)rb * p.RB + row;
      if (row < p.RB && tok < p.T) {
        bf16* orow = p.o + tok * p.ldo + h * 64 + 2 * quad;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(orow + 8 * j) = pack_bf16x2(oa[4 * j + 2 * hr], oa[4 * j + 2 * hr + 1]);
      }
    }
  }
  if (p.store_qkv && t == 0) bulk_wait_read<0>();
}

}  // namespace univl

using namespace univl;

// 1 if univl_fused_qkv_attention_supported supports this shape (else the caller uses the unfused QKV GEMM + attention core)
extern "C" int univl_fused_qkv_attention_supported(int n_seq, int heads, int S, int H) {
  return (n_seq > 0 && heads == 12 && H == 768 && S >= 16 && S <= 128 && (S % 16) == 0) ? 1 : 0;
}

// the kernel instantiation for the row-block width RB = floor(128 / S) * S
template <template <int> class K, typename Fn>
static int fa_dispatch(int RB, Fn&& fn) {
  switch (RB) {
    case 80: return fn(K<80>::kernel);
    case 96: return fn(K<96>::kernel);
    case 112: return fn(K<112>::kernel);
    case 128: return fn(K<128>::kernel);
  }
  return set_error(UNIVL_ERR_ARG, "fused_attention: row block %d", RB);
}
template <int NK>
struct FaFwdKernel {
  static constexpr auto kernel = fused_qkv_attention_fwd_kernel<NK>;
};

// ctx[T, H] = MHA(x[T, H]) with q/k/v = x Wqkv^T + bias computed in the same kernel (T = n_seq * S, H = heads * 64 = 768).
// wqkv: bf16 [3H, H] (rows: query | key | value weights), bias fp32 [3H].  qkv_out (nullable): bf16 [T, 3H] copy of the
// projected q | k | v for the backward pass.  Mask / dropout arguments as univl_attention_fwd, except the dropout
// layout, which is row-major (see fa_keep_bits) and matched by univl_attention_bwd(..., rng_layout = 1).
extern "C" int univl_fused_qkv_attention_fwd(const void* x, long long ldx, const void* wqkv, long long ldw,
                                             const float* bias, void* qkv_out, long long ld_qkv, void* o,
                                             long long ldo, float* lse, const long long* mask_a,
                                             const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs, int n_seq,
                                             int heads, int S, int causal, float scale, float p_drop,
                                             const unsigned long long* rng_state, unsigned long long stream_id,
                                             void* stream) {
  const int H = heads * 64;
  UNIVL_CHECK_ARG(x && wqkv && bias && o, "fused_attention: null pointer");
  UNIVL_CHECK_ARG(univl_fused_qkv_attention_supported(n_seq, heads, S, H),
                  "fused_attention: unsupported shape n_seq=%d heads=%d S=%d (12 heads, S %% 16 == 0, 16 <= S <= 128)",
                  n_seq, heads, S);
  UNIVL_CHECK_ARG((ldx % 8) == 0 && (ldw % 8) == 0 && (ldo % 8) == 0 && ((uintptr_t)x & 15) == 0 &&
                      ((uintptr_t)wqkv & 15) == 0 && ((uintptr_t)o & 15) == 0 && ((uintptr_t)bias & 15) == 0,
                  "fused_attention: operands must be 16-byte aligned with row strides that are multiples of 8");
  UNIVL_CHECK_ARG(mask_a == nullptr || Wa + Fb == S, "fused_attention: mask parts (%d + %d) must cover S=%d", Wa, Fb, S);
  UNIVL_CHECK_ARG(!(Fb > 0 && mask_a != nullptr && mask_b == nullptr), "fused_attention: missing second mask part");
  UNIVL_CHECK_ARG(!all_pairs || Nb > 0, "fused_attention: all_pairs needs Nb > 0");
  UNIVL_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, "fused_attention: bad dropout probability");
  UNIVL_CHECK_ARG(p_drop == 0.f || rng_state != nullptr, "fused_attention: dropout needs rng_state");
  UNIVL_CHECK_ARG(qkv_out == nullptr || ((ld_qkv % 8) == 0 && ((uintptr_t)qkv_out & 15) == 0),
                  "fused_attention: qkv_out must be 16-byte aligned");
  FusedAttnParams p = {};
  p.T = n_seq * S; p.S = S; p.G = 128 / S; p.RB = p.G * S; p.n_seq = n_seq; p.heads = heads;
  p.n_blocks = (n_seq + p.G - 1) / p.G;
  p.bias = bias; p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  p.mask_a = mask_a; p.mask_b = mask_b; p.Wa = Wa; p.Fb = Fb; p.Nb = Nb > 0 ? Nb : 1; p.all_pairs = all_pairs;
  p.causal = causal; p.scale = scale;
  p.drop_on = p_drop > 0.f;
  p.drop_threshold = dropout_threshold16(p_drop);
  p.drop_scale = p_drop > 0.f ? 1.0f / (1.0f - p_drop) : 1.0f;
  p.rng = rng_state; p.stream = stream_id;
  p.store_qkv = qkv_out != nullptr;
  CUtensorMap tx, tw, tq;
  int rc;
  // x box = the RB rows of the block when the q/k/v copies go out in whole 32-row boxes; otherwise all 128 tile rows, so
  // that the rows a partial box spills into the next block are that block's true values
  p.x_box_rows = (p.RB % 32 == 0) ? p.RB : 128;
  if ((rc = make_tmap(&tx, x, p.T, H, ldx, p.x_box_rows))) return rc;   // box {64 k, x_box_rows}
  if ((rc = make_tmap(&tw, wqkv, 3 * H, H, ldw, 64))) return rc;        // box {64 k, 64 weight rows}
  if (qkv_out != nullptr) {
    if ((rc = make_tmap_epi(&tq, qkv_out, false, p.T, 3 * H, ld_qkv))) return rc;  // box {64 cols, 32 rows}
  } else {
    tq = tx;
  }
  const int sms = usable_sms();
  const long long items = (long long)p.n_blocks * heads;
  const int grid = (int)(items < sms ? items : sms);
  return fa_dispatch<FaFwdKernel>(p.RB, [&](auto kern) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM_BYTES);
    if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "fused_attention smem attribute: %s", cudaGetErrorString(e));
    e = launch_kernel(kern, dim3(grid), dim3(FA_THREADS), (size_t)FA_SMEM_BYTES, (cudaStream_t)stream, tx, tw, tq, p);
    if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "fused_attention launch: %s", cudaGetErrorString(e));
    UNIVL_CHECK_LAUNCH("fused_qkv_attention_fwd");
    return UNIVL_OK;
  });
}

// =====================================================================================================================
// Backward of the attention core (same row-block x head decomposition, same masks and dropout layout as the forward
// above).  Inputs: the saved q | k | v [T, 3H], the context O and its gradient dO [T, H], the log-sum-exp.  Per item,
// with warpgroup c of the two consumer warpgroups owning query rows (and, for dK / dV, key rows) [64 c, 64 c + 64):
//     S  = Q K^T,  dP = dO V^T                         (wgmma into registers)
//     P  = exp(S * scale + mask - lse);  P~ = dropout(P);  dS = P o (dropout'(dP) - D) * scale,  D_i = sum_d dO_id O_id
//     dQ = dS K   (dS from registers, K MN-major)
//     dV = P~^T dO, dK = dS^T Q   (P~ and dS through shared memory as MN-major A operands; contraction over queries)
//     -> bf16 rows of dq | dk | dv [T, 3H], and the projection-bias gradients (column sums): shuffles, then one
//        partial row per (row block, warp) that partials_reduce adds in order.
// The Q, K, V, dO, O tiles arrive by TMA straight in the 128B-swizzled layout every product reads, double-buffered, so
// the next item's operands load while this one computes.
// =====================================================================================================================
namespace univl {

constexpr int FB_IN_BYTES = 5 * FA_TILE_BYTES;              // Q, K, V, dO, O tiles of one item
constexpr int FB_OFF_P = 2 * FB_IN_BYTES;                   // P~ tile (two 64-key atoms)
constexpr int FB_OFF_DS = FB_OFF_P + 2 * FA_TILE_BYTES;     // dS tile
constexpr int FB_OFF_MADD = FB_OFF_DS + 2 * FA_TILE_BYTES;
constexpr int FB_OFF_BAR = FB_OFF_MADD + 512;               // in_full[2] in_empty[2]
constexpr int FB_SMEM_BYTES = FB_OFF_BAR + 4 * 8 + 1024;
static_assert(FB_SMEM_BYTES <= 227 * 1024, "shared memory per block");

struct FusedAttnBwdParams {
  int T, S, G, RB, n_seq, heads, n_blocks;
  const float* lse;
  bf16* dqkv;
  long long ld_dqkv;
  float* dbias;               // partial rows [n_blocks * 8][3 * heads * 64], or null
  const long long* mask_a;
  const long long* mask_b;
  int Wa, Fb, Nb, all_pairs, causal;
  float scale;
  int drop_on;
  uint32_t drop_threshold;
  float drop_scale;
  const unsigned long long* rng;
  uint64_t stream;
};

// rows r_lo, r_lo + 8 of a 64-column gradient fragment -> bf16 rows of dqkv, and this warp's column sums into its
// partial row of dbias (row rb * 8 + warpgroup * 4 + warp; summed in row order after the kernel)
__device__ __forceinline__ void fb_drain(const FusedAttnBwdParams& p, const float (&v)[32], int rb, int r_lo, int quad,
                                         int lane, int col0, int part_row) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = r_lo + 8 * hr;
    const long long tok = (long long)rb * p.RB + row;
    if (row < p.RB && tok < p.T) {
      bf16* dst = p.dqkv + tok * p.ld_dqkv + col0 + 2 * quad;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(v[4 * j + 2 * hr], v[4 * j + 2 * hr + 1]);
    }
  }
  if (p.dbias == nullptr) return;
  const bool ok0 = r_lo < p.RB && (long long)rb * p.RB + r_lo < p.T;
  const bool ok1 = r_lo + 8 < p.RB && (long long)rb * p.RB + r_lo + 8 < p.T;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float s = (ok0 ? v[4 * j + e] : 0.f) + (ok1 ? v[4 * j + 2 + e] : 0.f);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (lane < 4) p.dbias[(long long)part_row * 3 * p.heads * 64 + col0 + 8 * j + 2 * quad + e] = s;
    }
  }
}

template <int NK>
__global__ void __launch_bounds__(FA_THREADS, 1)
fused_attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                           const __grid_constant__ CUtensorMap tmap_o, const FusedAttnBwdParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* in_full = reinterpret_cast<uint64_t*>(smem + FB_OFF_BAR);   // [2] TMA -> consumers
  uint64_t* in_empty = in_full + 2;                                      // [2] consumers -> TMA
  float* madd = reinterpret_cast<float*>(smem + FB_OFF_MADD);

  const int wg = threadIdx.x >> 7;
  const int H = p.heads * 64;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_o);
    for (int b = 0; b < 2; ++b) {
      mbar_init(&in_full[b], 1);
      mbar_init(&in_empty[b], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  int item_begin, item_end;
  fa_item_range(p.n_blocks * p.heads, item_begin, item_end);
  const int n_items = item_end - item_begin;

  if (wg == 0) {
    // ------------------------------------------ TMA producer ------------------------------------------
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      for (int j = 0; j < n_items; ++j) {
        const int b = j & 1;
        const int w = item_begin + j;
        const int rb = w / p.heads, h = w - rb * p.heads;
        const int r0 = rb * p.RB;
        mbar_wait(&in_empty[b], (((uint32_t)j >> 1) & 1) ^ 1);
        uint8_t* dst = smem + b * FB_IN_BYTES;
        mbar_arrive_expect_tx(&in_full[b], FB_IN_BYTES);
#pragma unroll
        for (int m = 0; m < 3; ++m) tma_load_2d(dst + m * FA_TILE_BYTES, &tmap_qkv, &in_full[b], m * H + h * 64, r0);
        tma_load_2d(dst + 3 * FA_TILE_BYTES, &tmap_do, &in_full[b], h * 64, r0);
        tma_load_2d(dst + 4 * FA_TILE_BYTES, &tmap_o, &in_full[b], h * 64, r0);
      }
    }
    return;
  }

  // ------------------------------------------ consumer warpgroups ------------------------------------------
  regs_alloc<232>();
  const int c = wg - 1;
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31, quad = lane & 3;
  const int r_lo = c * 64 + warp * 16 + (lane >> 2);
  const uint64_t seed = (p.drop_on && p.rng != nullptr) ? p.rng[0] : 0ull;
  const uint64_t stream = p.stream + ((p.drop_on && p.rng != nullptr) ? (p.rng[1] << 20) : 0ull);
  const float sl2 = p.scale * 1.44269504088896340736f;
  const float neg_big = -10000.0f * 1.44269504088896340736f;
  const float ds_scale = p.drop_on ? p.drop_scale : 1.0f;
  const uint32_t sP = smem_u32(smem + FB_OFF_P), sdS = smem_u32(smem + FB_OFF_DS);
  int cur_rb = -1;
  for (int j = 0; j < n_items; ++j) {
    const int w = item_begin + j;
    const int rb = w / p.heads, h = w - rb * p.heads;
    const int b = j & 1;
    uint8_t* in = smem + b * FB_IN_BYTES;
    const uint32_t sQ = smem_u32(in), sK = sQ + FA_TILE_BYTES, sV = sQ + 2 * FA_TILE_BYTES,
                   sdO = sQ + 3 * FA_TILE_BYTES;

    named_bar(1, 256);  // both warpgroups are done with the previous item's P~ / dS tiles and mask
    if (rb != cur_rb) {
      if (c == 0)
        madd[t] = fa_key_mask(p.mask_a, p.mask_b, p.Wa, p.Fb, p.Nb, p.all_pairs, p.S, p.G, p.n_seq, NK, rb, t);
      named_bar(2, 256);
      cur_rb = rb;
    }
    mbar_wait(&in_full[b], ((uint32_t)j >> 1) & 1);

    // ---- S = Q K^T, dP = dO V^T for this warpgroup's 64 query rows ----
    float sa[NK / 2], dpa[NK / 2];
#pragma unroll
    for (int e = 0; e < NK / 2; ++e) sa[e] = dpa[e] = 0.f;
    wgmma_fence();
    fence_regs(sa);
    fence_regs(dpa);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      WgmmaSS<NK>::template mma<0, 0>(sa, make_smem_desc_sw128(sQ + c * (64 * 128) + 32 * k, 16, 1024),
                                      make_smem_desc_sw128(sK + 32 * k, 16, 1024), k > 0 ? 1 : 0);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      WgmmaSS<NK>::template mma<0, 0>(dpa, make_smem_desc_sw128(sdO + c * (64 * 128) + 32 * k, 16, 1024),
                                      make_smem_desc_sw128(sV + 32 * k, 16, 1024), k > 0 ? 1 : 0);
    wgmma_commit();

    // D_i = <dO_i, O_i> over the 64 dims of this head (each quad lane: 16 of them), while the products run
    float D[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r_lo + 8 * hr;
      const uint8_t* drow = in + 3 * FA_TILE_BYTES + row * 128;
      const uint8_t* orow = drow + FA_TILE_BYTES;
      float d = 0.f;
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        const int off = ((2 * quad + cc) ^ (row & 7)) << 4;
        const uint4 ud = *reinterpret_cast<const uint4*>(drow + off), uo = *reinterpret_cast<const uint4*>(orow + off);
        const uint32_t wo[4] = {uo.x, uo.y, uo.z, uo.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 a = unpack_bf16x2(wo[e]), bb = unpack_bf16x2(wd[e]);
          d = fmaf(a.x, bb.x, d);
          d = fmaf(a.y, bb.y, d);
        }
      }
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      D[hr] = d;
    }
    wgmma_wait<0>();
    fence_regs(sa);
    fence_regs(dpa);

    // ---- P~, dS: to registers (dS as the A operand of dQ) and to the shared-memory tiles (dK, dV) ----
    uint32_t dsa[NK / 16][4];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r_lo + 8 * hr;
      const int g = row / p.S, c0 = g * p.S, qpos = row - c0;
      const long long seq = (long long)rb * p.G + g;
      const bool valid = row < p.RB && seq < p.n_seq;
      const long long bh = seq * p.heads + h;
      const float lse2 = valid ? p.lse[bh * p.S + qpos] * 1.44269504088896340736f : 0.f;
      uint32_t keep[(NK / 8 + 15) / 16];
      if (p.drop_on) {
        const uint64_t base = ((uint64_t)bh * p.S + qpos) * (uint64_t)(p.S >> 3);
        fa_keep_bits<NK>(seed, stream, base, c0 >> 3, p.drop_threshold, quad, keep);
      }
      uint8_t* prow = smem + FB_OFF_P + row * 128;
      uint8_t* srow = smem + FB_OFF_DS + row * 128;
#pragma unroll
      for (int jj = 0; jj < NK / 8; ++jj) {
        float pd[2], dsv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = 8 * jj + 2 * quad + e;
          const bool own = valid && key >= c0 && key < c0 + p.S;
          float a = madd[key];
          if (p.causal && (key - c0) > qpos && a == 0.f) a = neg_big;
          const float pr = ex2_approx(fmaf(sa[4 * jj + 2 * hr + e], sl2, a) - lse2);
          const bool kp = !p.drop_on || ((keep[jj >> 4] >> (2 * (jj & 15) + e)) & 1u);
          const float gdrop = kp ? dpa[4 * jj + 2 * hr + e] * ds_scale : 0.f;
          pd[e] = own && kp ? pr * ds_scale : 0.f;
          dsv[e] = own ? pr * (gdrop - D[hr]) * p.scale : 0.f;
        }
        const uint32_t pu = pack_bf16x2(pd[0], pd[1]), su = pack_bf16x2(dsv[0], dsv[1]);
        dsa[jj >> 1][(jj & 1) * 2 + hr] = su;
        const int off = (jj >> 3) * FA_TILE_BYTES + (((jj & 7) ^ (row & 7)) << 4) + quad * 4;
        *reinterpret_cast<uint32_t*>(prow + off) = pu;
        *reinterpret_cast<uint32_t*>(srow + off) = su;
      }
    }

    // ---- dQ = dS K (contraction over keys; K [keys][64] is the MN-major B operand) ----
    float dqa[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) dqa[e] = 0.f;
    wgmma_fence();
    fence_regs(dqa);
#pragma unroll
    for (int kk = 0; kk < NK / 16; ++kk)
      WgmmaRS<64>::mma<1>(dqa, dsa[kk], make_smem_desc_sw128(sK + kk * 2048, FA_TILE_BYTES, 1024), kk > 0 ? 1 : 0);
    wgmma_commit();

    fence_proxy_async_smem();  // P~ / dS tile writes -> visible to the tensor core
    named_bar(3, 256);         // both warpgroups' query rows are in the tiles

    // ---- dV = P~^T dO, dK = dS^T Q for key rows [64 c, 64 c + 64): contraction over the RB query rows ----
    float dva[32], dka[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) dva[e] = dka[e] = 0.f;
    wgmma_fence();
    fence_regs(dva);
    fence_regs(dka);
#pragma unroll
    for (int kk = 0; kk < NK / 16; ++kk) {
      WgmmaSS<64>::mma<1, 1>(dva, make_smem_desc_sw128(sP + c * FA_TILE_BYTES + kk * 2048, FA_TILE_BYTES, 1024),
                             make_smem_desc_sw128(sdO + kk * 2048, FA_TILE_BYTES, 1024), kk > 0 ? 1 : 0);
      WgmmaSS<64>::mma<1, 1>(dka, make_smem_desc_sw128(sdS + c * FA_TILE_BYTES + kk * 2048, FA_TILE_BYTES, 1024),
                             make_smem_desc_sw128(sQ + kk * 2048, FA_TILE_BYTES, 1024), kk > 0 ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dqa);
    fence_regs(dva);
    fence_regs(dka);
    if (t == 0) mbar_arrive(&in_empty[b]);  // this warpgroup no longer reads the item's input tiles

    const int part_row = rb * 8 + c * 4 + warp;
    fb_drain(p, dqa, rb, r_lo, quad, lane, h * 64, part_row);
    fb_drain(p, dka, rb, r_lo, quad, lane, H + h * 64, part_row);
    fb_drain(p, dva, rb, r_lo, quad, lane, 2 * H + h * 64, part_row);
  }
}

template <int NK>
struct FaBwdKernel {
  static constexpr auto kernel = fused_attention_bwd_kernel<NK>;
};

}  // namespace univl

// dq | dk | dv [T, 3H] (bf16) = backward of the attention core for the shapes univl_fused_qkv_attention_supported
// accepts, from the saved q | k | v [T, 3H], the context o, its gradient d_o and the log-sum-exp.  dbias (nullable, fp32
// [3H]) accumulates the column sums (projection-bias gradients).  Dropout masks: the row-major layout of the fused forward.
extern "C" int univl_fused_attention_bwd(const void* qkv, long long ld_qkv, const void* o, long long ldo,
                                         const float* lse, const void* d_o, long long lddo, void* dqkv,
                                         long long ld_dqkv, float* dbias, const long long* mask_a,
                                         const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs, int n_seq,
                                         int heads, int S, int causal, float scale, float p_drop,
                                         const unsigned long long* rng_state, unsigned long long stream_id,
                                         void* stream) {
  const int H = heads * 64;
  UNIVL_CHECK_ARG(qkv && o && lse && d_o && dqkv, "fused_attention_bwd: null pointer");
  UNIVL_CHECK_ARG(univl_fused_qkv_attention_supported(n_seq, heads, S, H),
                  "fused_attention_bwd: unsupported shape n_seq=%d heads=%d S=%d", n_seq, heads, S);
  UNIVL_CHECK_ARG((ld_qkv % 8) == 0 && (ldo % 8) == 0 && (lddo % 8) == 0 && (ld_dqkv % 8) == 0 &&
                      ((uintptr_t)qkv & 15) == 0 && ((uintptr_t)o & 15) == 0 && ((uintptr_t)d_o & 15) == 0 &&
                      ((uintptr_t)dqkv & 15) == 0,
                  "fused_attention_bwd: operands must be 16-byte aligned with row strides that are multiples of 8");
  UNIVL_CHECK_ARG(mask_a == nullptr || Wa + Fb == S, "fused_attention_bwd: mask parts must cover S");
  UNIVL_CHECK_ARG(!(Fb > 0 && mask_a != nullptr && mask_b == nullptr), "fused_attention_bwd: missing second mask part");
  UNIVL_CHECK_ARG(!all_pairs || Nb > 0, "fused_attention_bwd: all_pairs needs Nb > 0");
  UNIVL_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f && (p_drop == 0.f || rng_state != nullptr),
                  "fused_attention_bwd: bad dropout arguments");
  FusedAttnBwdParams p = {};
  p.T = n_seq * S; p.S = S; p.G = 128 / S; p.RB = p.G * S; p.n_seq = n_seq; p.heads = heads;
  p.n_blocks = (n_seq + p.G - 1) / p.G;
  p.lse = lse;
  p.dqkv = (bf16*)dqkv; p.ld_dqkv = ld_dqkv;
  p.mask_a = mask_a; p.mask_b = mask_b; p.Wa = Wa; p.Fb = Fb; p.Nb = Nb > 0 ? Nb : 1; p.all_pairs = all_pairs;
  p.causal = causal; p.scale = scale;
  p.drop_on = p_drop > 0.f;
  p.drop_threshold = dropout_threshold16(p_drop);
  p.drop_scale = p_drop > 0.f ? 1.0f / (1.0f - p_drop) : 1.0f;
  p.rng = rng_state; p.stream = stream_id;
  CUtensorMap tq, td, to;
  int rc;
  if ((rc = make_tmap(&tq, qkv, p.T, 3 * H, ld_qkv, 128))) return rc;   // box {64 cols, 128 rows}
  if ((rc = make_tmap(&td, d_o, p.T, H, lddo, 128))) return rc;
  if ((rc = make_tmap(&to, o, p.T, H, ldo, 128))) return rc;
  const int sms = usable_sms();
  const long long items = (long long)p.n_blocks * heads;
  const int grid = (int)(items < sms ? items : sms);
  const int n_parts = p.n_blocks * 8;
  if (dbias != nullptr)
    if ((rc = scratch_alloc((void**)&p.dbias, (size_t)n_parts * 3 * H * sizeof(float), (cudaStream_t)stream))) return rc;
  rc = fa_dispatch<FaBwdKernel>(p.RB, [&](auto kern) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM_BYTES);
    if (e != cudaSuccess)
      return set_error(UNIVL_ERR_CUDA, "fused_attention_bwd smem attribute: %s", cudaGetErrorString(e));
    e = launch_kernel(kern, dim3(grid), dim3(FA_THREADS), (size_t)FB_SMEM_BYTES, (cudaStream_t)stream, tq, td, to, p);
    if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "fused_attention_bwd launch: %s", cudaGetErrorString(e));
    UNIVL_CHECK_LAUNCH("fused_attention_bwd");
    return UNIVL_OK;
  });
  if (rc != UNIVL_OK || dbias == nullptr) return rc;
  return partials_reduce(p.dbias, n_parts, 1, 3 * H, dbias, 3 * H, (cudaStream_t)stream);
}
