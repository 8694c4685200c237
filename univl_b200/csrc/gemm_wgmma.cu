// univl_b200 — persistent, warp-specialised wgmma / TMA GEMM for sm_90a.
//
//   D[M,N] = epilogue( sum_k A(m,k) * B(n,k) )          bf16 operands, fp32 accumulation in registers
//
// One kernel template serves the three GEMMs of every nn.Linear on the UniVL hot path
// (reference: modules/module_bert.py:172-174,208,234,247 and the autograd mirror):
//   forward  Y  = X  W^T   A = X  [T,K]  K-major     B = W [N,K]  K-major
//   dgrad    dX = dY W     A = dY [T,N]  K-major     B = W [N,K]  MN-major (contraction over N)
//   wgrad    dW = dY^T X   A = dY [T,N]  MN-major    B = X [T,K]  MN-major (contraction over T)
// so neither weights nor activations are ever transposed in HBM: the operand "major" is the transpose bit of the wgmma
// instruction and a different TMA box shape.
//
// Structure: the producer / consumer ring of pipeline.cuh on 128 x BLOCK_N output tiles, optional split-K.  The
// consumer warpgroups issue wgmma on each stage and run the fused epilogue straight from their accumulator registers,
// in one of two schedules chosen by the tile width:
//     BLOCK_N = 256       cooperative: both warpgroups work on every tile, each on 64 of its 128 rows
//                         (m64 x 256 x k16 per k16 step); the tensor cores idle while the two run the epilogue.
//     BLOCK_N = 64 / 128  ping-pong: each warpgroup owns whole tiles, the two alternating the CTA's tiles, and issues
//                         two m64 x BLOCK_N x k16 wgmma per k16 step (rows 0-63 and 64-127).  A pair of named barriers
//                         hands the tensor cores from one warpgroup's mainloop to the other's in tile order, so one
//                         warpgroup's epilogue runs while the other's MMAs do.  (256 accumulator floats per warpgroup
//                         would not fit in registers, so the 256-wide tile stays cooperative.)
// grid = min(#work items, #SMs); each CTA walks work items round-robin in the order decode_work() defines, and the
// producer's ring runs continuously across tiles, so the next tile's operands load while the epilogue runs.  Both
// schedules give every output element the same chain of k16 wgmmas in the same k order and the same epilogue, so the
// tile width does not change a bit of the result.
// Split-K (fp32 weight gradients, EPI_ATOMIC_F32, K >= SPLIT_MIN_K or a forced split_k): a work item is a (tile,
// split) pair.  Its epilogue stores alpha * acc into a scratch slot of its own, and the last of a tile's items to
// arrive (per warp, counted on a zeroed counter) adds every split's slot in split order and then into the output —
// in the owning warpgroup's epilogue, so under the ping-pong schedule it overlaps the other warpgroup's MMAs
// (splitk_fixup).  No item waits for another.  Below SPLIT_MIN_K the automatic plan's splits are instead summed in
// registers by one unsplit 64-wide work item per tile (GemmParams::kb_seg): the same segments, the same order, the
// same bits.
#include "common.cuh"
#include "fp8.cuh"
#include "pipeline.cuh"
#include "tmap.cuh"

#include <climits>
#include <stdio.h>
#include <type_traits>

namespace univl {

enum GemmEpilogue : int {
  EPI_BIAS_BF16 = 0,      // out(bf16) = alpha*acc + bias
  EPI_BIAS_GELU_BF16 = 1, // aux_out(bf16) = acc + bias ; out(bf16) = gelu_erf(acc + bias)
  EPI_GELU_BWD_BF16 = 2,  // out(bf16) = acc * gelu_erf'(aux_in)
  EPI_ADD_BF16 = 3,       // out(bf16) = alpha*acc + aux_in
  EPI_BIAS_F32 = 4,       // out(f32)  = alpha*acc + bias
  EPI_ATOMIC_F32 = 5,     // out(f32) += alpha*acc      (gradient accumulation; split-K partials summed in split order)
};

struct GemmParams {
  int M, N, Kc;
  int k_blocks_per_split;
  int epilogue;
  float alpha;
  void* out;
  long long ldo;
  const float* bias;
  const bf16* aux_in;
  long long ld_aux_in;
  bf16* aux_out;
  long long ld_aux_out;
  int vec2;  // 1 = every epilogue operand takes 2-element vector accesses (aligned base, even leading dimension)
  int vec8;  // 1 = the bf16 outputs (out, aux_out) take 16-byte stores of 8 columns (16-byte aligned base, ld % 8 == 0)
  // EPI_ATOMIC_F32 with splits > 1 (else null): the split-K fix-up's slots, [tiles][splits][2 halves][64 x BLOCK_N]
  // floats in accumulator-fragment order, and its arrival counters, [tiles][2 halves][4 warps], zero at launch
  float* slots;
  unsigned* arrived;
  int splits;
  // EPI_ATOMIC_F32 on the 64-wide tile: a work item of more k-blocks than this sums its k range in segments of
  // kb_seg k-blocks, t = 0, t += alpha * segment in k order, then out += t — the bits of a split-K plan with kb_seg
  // k-blocks per split, without its scratch memory
  int kb_seg;
};

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int PLAN_SMS = 132;  // H100 SXM: the tile-width / split-K plan is a pure function of the problem
// below it, an automatic split-K plan runs unsplit with in-register k-segment sums (see plan_gemm)
constexpr int SPLIT_MIN_K = 4096;

template <int BLOCK_N, int STAGES>
struct GemmSmem {
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFFSET + 2 * STAGES * 8;  // full[STAGES], empty[STAGES]
  static constexpr int DYN_BYTES = TOTAL + 1024;             // slack for manual 1024 B alignment
  static_assert(DYN_BYTES <= 227 * 1024, "shared memory per block");
};

struct WorkItem {
  int m0, n0, kb_begin, num_kb;
};
// Rasterisation: without split-K the n-tile index runs fastest, so the CTAs in flight at any moment cover a band of a
// few m-tiles across ALL n-tiles — every A tile (activations, streamed from HBM) is fetched from DRAM once and reused
// from L2 by the other n-tiles, while the whole B operand (weights) stays L2-resident.
// With split-K (weight gradients) the tiles of one split run together so they share that split's token slab.
__device__ __forceinline__ WorkItem decode_work(int w, int m_tiles, int n_tiles, int total_kb, int kb_per, int bn) {
  const int tiles = m_tiles * n_tiles;
  const int split = w / tiles;
  const int rem = w - split * tiles;
  int m_blk, n_blk;
  if (kb_per >= total_kb) {
    m_blk = rem / n_tiles;
    n_blk = rem - m_blk * n_tiles;
  } else {
    n_blk = rem / m_tiles;
    m_blk = rem - n_blk * m_tiles;
  }
  WorkItem it;
  it.m0 = m_blk * BLOCK_M;
  it.n0 = n_blk * bn;
  it.kb_begin = split * kb_per;
  it.num_kb = min(total_kb, it.kb_begin + kb_per) - it.kb_begin;
  return it;
}

// fused epilogue of the accumulator values of columns (col, col + 1) of one row; col is even.  alpha: the scale of
// the accumulator values (p.alpha, or 1 for the split-K sums, which carry it already)
__device__ __forceinline__ void epi_pair(const GemmParams& p, float alpha, int row, int col, float v0, float v1) {
  if (row >= p.M || col >= p.N) return;
  const bool two = col + 1 < p.N;
  const bool vec = two && p.vec2;
  const int epi = p.epilogue;
  v0 *= alpha;
  v1 *= alpha;
  if (p.bias != nullptr && (epi == EPI_BIAS_BF16 || epi == EPI_BIAS_GELU_BF16 || epi == EPI_BIAS_F32)) {
    v0 += __ldg(p.bias + col);
    if (two) v1 += __ldg(p.bias + col + 1);
  }
  if (epi == EPI_ATOMIC_F32 || epi == EPI_BIAS_F32) {
    float* o = reinterpret_cast<float*>(p.out) + (long long)row * p.ldo + col;
    if (epi == EPI_ATOMIC_F32) {  // this thread is the element's only writer in the launch (split-K: the last arriver's)
      if (vec) {
        float2 a = *reinterpret_cast<float2*>(o);
        *reinterpret_cast<float2*>(o) = make_float2(a.x + v0, a.y + v1);
      } else {
        o[0] += v0;
        if (two) o[1] += v1;
      }
    } else {
      if (vec) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
      else {
        o[0] = v0;
        if (two) o[1] = v1;
      }
    }
    return;
  }
  if (epi == EPI_GELU_BWD_BF16 || epi == EPI_ADD_BF16) {
    const bf16* a = p.aux_in + (long long)row * p.ld_aux_in + col;
    float x0, x1 = 0.f;
    if (vec) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a));
      x0 = f.x;
      x1 = f.y;
    } else {
      x0 = __bfloat162float(a[0]);
      if (two) x1 = __bfloat162float(a[1]);
    }
    if (epi == EPI_GELU_BWD_BF16) {
      v0 *= gelu_erf_grad(x0);
      v1 *= gelu_erf_grad(x1);
    } else {
      v0 += x0;
      v1 += x1;
    }
  }
  if (epi == EPI_BIAS_GELU_BF16) {
    bf16* ao = p.aux_out + (long long)row * p.ld_aux_out + col;
    if (vec) *reinterpret_cast<uint32_t*>(ao) = pack_bf16x2(v0, v1);
    else {
      ao[0] = __float2bfloat16(v0);
      if (two) ao[1] = __float2bfloat16(v1);
    }
    v0 = gelu_erf(v0);
    v1 = gelu_erf(v1);
  }
  bf16* o = reinterpret_cast<bf16*>(p.out) + (long long)row * p.ldo + col;
  if (vec) *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(v0, v1);
  else {
    o[0] = __float2bfloat16(v0);
    if (two) o[1] = __float2bfloat16(v1);
  }
}

// 8-column groups per chunk of the unchecked epilogue: 16 aux_in words or 16 bias floats per chunk, two chunks in
// flight; every instance compiles without spills under regs_alloc<232> (check with -Xptxas -v when changing it)
constexpr int EPI_CHUNK = 8;

// 4 x 4 transpose of 32-bit words across the four lanes of a quad (q = lane % 4): on entry w[k] is this lane's word of
// 8-column group k (columns 2 q, 2 q + 1 of the group); on return the four words of group q, word k from lane k, which
// is the group's 8 columns in order.  Two butterfly stages; the whole warp must call it.
__device__ __forceinline__ uint4 quad_transpose(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, int q) {
  const bool odd = q & 1;
  uint32_t r0 = __shfl_xor_sync(0xffffffffu, odd ? w0 : w1, 1);
  uint32_t r1 = __shfl_xor_sync(0xffffffffu, odd ? w2 : w3, 1);
  if (odd) {
    w0 = r0;
    w2 = r1;
  } else {
    w1 = r0;
    w3 = r1;
  }
  const bool hi = q & 2;
  r0 = __shfl_xor_sync(0xffffffffu, hi ? w0 : w2, 2);
  r1 = __shfl_xor_sync(0xffffffffu, hi ? w1 : w3, 2);
  if (hi) {
    w0 = r0;
    w1 = r1;
  } else {
    w2 = r0;
    w3 = r1;
  }
  return make_uint4(w0, w1, w2, w3);
}

// Unchecked epilogue of a work item whose 128 x BLOCK_N tile lies wholly inside M x N, with p.vec2 set: no bounds
// checks, every access a 2-element vector.  The epilogue is a template argument,
// so the fragment walk is straight-line code.  It runs in chunks of EPI_CHUNK 8-column groups.  Each chunk's global
// loads (bias, aux_in, the accumulated output) are issued together, and before the previous chunk's arithmetic, so
// their latencies overlap each other and that arithmetic instead of adding up.  Loading ahead of the previous chunk's
// stores is safe for the exact in-place use epi_pair allows (aux_in == out, same leading dimension): a chunk's loads
// never touch the elements of an earlier chunk, and within a chunk every element's load is consumed by the arithmetic
// before its result is stored (by the same thread, or with WIDE by a lane of the same quad after the shuffles).
// It computes exactly what epi_pair computes: the same fp32 operations in the same order, with __fmul_rn / __fadd_rn
// so that alpha * acc and the add after it stay two roundings and are not contracted to an FFMA.
// BIAS: p.bias is set (bias epilogues).  alpha: as in epi_pair.
// WIDE (p.vec8, bf16 outputs): the four lanes of a quad, which hold 2 columns each of the same 8-column groups,
// exchange their packed results (quad_transpose) so that each lane stores one group whole, 16 bytes.  A warp's store
// then covers 64 contiguous bytes (two full 32-byte sectors) of each of its 8 rows, with a quarter of the store
// instructions, where the 4-byte stores cover 16 bytes (half a sector) of each row.
template <int EPI, bool BIAS, int BLOCK_N, bool WIDE = false>
__device__ __forceinline__ void epi_tile(const GemmParams& p, float alpha, int row, int col0,
                                         const float (&acc)[BLOCK_N / 2]) {
  constexpr int GROUPS = BLOCK_N / 8;
  // WIDE holds a quad's results for the shuffles: half-size chunks keep the 256-wide tile free of spills
  constexpr int CHUNK = WIDE ? 4 : (GROUPS < EPI_CHUNK ? GROUPS : EPI_CHUNK);
  static_assert(CHUNK % 4 == 0, "a chunk holds whole quads of 8-column groups");
  constexpr bool AUX = EPI == EPI_GELU_BWD_BF16 || EPI == EPI_ADD_BF16;
  constexpr bool OUT_F32 = EPI == EPI_BIAS_F32 || EPI == EPI_ATOMIC_F32;
  static_assert(!(WIDE && OUT_F32), "16-byte stores are for the bf16 outputs");
  constexpr bool ACCUM = EPI == EPI_ATOMIC_F32;  // out += alpha * acc
  const int q = threadIdx.x & 3;
  const float* bias = p.bias + col0;
  const bf16* ax = p.aux_in + (long long)row * p.ld_aux_in + col0;
  const long long ax8 = 8 * p.ld_aux_in;
  bf16* ao = p.aux_out + (long long)row * p.ld_aux_out + col0;
  const long long ao8 = 8 * p.ld_aux_out;
  const long long o8 = 8 * p.ldo;
  float* of = reinterpret_cast<float*>(p.out) + (long long)row * p.ldo + col0;
  bf16* ob = reinterpret_cast<bf16*>(p.out) + (long long)row * p.ldo + col0;
  // two load buffers, alternating between chunks
  float b[2][CHUNK][2];
  uint32_t x[2][CHUNK][2];
  float2 a[2][CHUNK][2];
  auto load = [&](int j0, int s) {
#pragma unroll
    for (int j = 0; j < CHUNK; ++j) {
      const int c = (j0 + j) * 8;
      if constexpr (BIAS) {
        b[s][j][0] = __ldg(bias + c);
        b[s][j][1] = __ldg(bias + c + 1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // rows row, row + 8
        if constexpr (AUX) x[s][j][h] = *reinterpret_cast<const uint32_t*>(ax + h * ax8 + c);
        if constexpr (ACCUM) a[s][j][h] = *reinterpret_cast<const float2*>(of + h * o8 + c);
      }
    }
  };
  load(0, 0);
#pragma unroll
  for (int j0 = 0; j0 < GROUPS; j0 += CHUNK) {
    const int s = (j0 / CHUNK) & 1;
    if (j0 + CHUNK < GROUPS) load(j0 + CHUNK, s ^ 1);
#pragma unroll
    for (int jq = 0; jq < CHUNK; jq += 4) {  // one quad of 8-column groups
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // rows row, row + 8
        uint32_t wo[4], wa[4];       // WIDE: packed out / aux_out words of the quad's groups in this row
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = jq + jj;
          const int c = (j0 + j) * 8;
          float v0 = __fmul_rn(acc[4 * (j0 + j) + 2 * h], alpha);
          float v1 = __fmul_rn(acc[4 * (j0 + j) + 2 * h + 1], alpha);
          if constexpr (BIAS) {
            v0 = __fadd_rn(v0, b[s][j][0]);
            v1 = __fadd_rn(v1, b[s][j][1]);
          }
          if constexpr (AUX) {
            const float2 f = unpack_bf16x2(x[s][j][h]);
            if constexpr (EPI == EPI_GELU_BWD_BF16) {
              v0 = __fmul_rn(v0, gelu_erf_grad(f.x));
              v1 = __fmul_rn(v1, gelu_erf_grad(f.y));
            } else {
              v0 = __fadd_rn(v0, f.x);
              v1 = __fadd_rn(v1, f.y);
            }
          }
          if constexpr (OUT_F32) {
            if constexpr (ACCUM) {
              v0 = __fadd_rn(a[s][j][h].x, v0);
              v1 = __fadd_rn(a[s][j][h].y, v1);
            }
            *reinterpret_cast<float2*>(of + h * o8 + c) = make_float2(v0, v1);
          } else {
            if constexpr (EPI == EPI_BIAS_GELU_BF16) {
              const uint32_t w = pack_bf16x2(v0, v1);
              if constexpr (WIDE) wa[jj] = w;
              else *reinterpret_cast<uint32_t*>(ao + h * ao8 + c) = w;
              v0 = gelu_erf(v0);
              v1 = gelu_erf(v1);
            }
            const uint32_t w = pack_bf16x2(v0, v1);
            if constexpr (WIDE) wo[jj] = w;
            else *reinterpret_cast<uint32_t*>(ob + h * o8 + c) = w;
          }
        }
        if constexpr (WIDE) {
          // this lane stores group j0 + jq + q whole: 8 (j0 + jq) + 6 q columns from col0 = 2 q
          const int c = (j0 + jq) * 8 + 6 * q;
          if constexpr (EPI == EPI_BIAS_GELU_BF16)
            *reinterpret_cast<uint4*>(ao + h * ao8 + c) = quad_transpose(wa[0], wa[1], wa[2], wa[3], q);
          *reinterpret_cast<uint4*>(ob + h * o8 + c) = quad_transpose(wo[0], wo[1], wo[2], wo[3], q);
        }
      }
    }
  }
}

// fused epilogue of one warpgroup's 64 x BLOCK_N accumulator block.  accumulator fragment: warp w holds rows
// 16 w + lane / 4 (+ 8); register 4 j + {0, 1} (+ {2, 3} for row + 8) are columns 8 j + 2 (lane % 4) + {0, 1}.
// The epilogue is chosen once per work item (inside: its whole tile lies in the output): tiles wholly inside the
// output take the unchecked epi_tile, edge tiles and launches without 2-element vector access the checked per-pair
// epi_pair.
template <int BLOCK_N>
__device__ __forceinline__ void epilogue_block(const GemmParams& p, bool inside, float alpha, int n0, int row,
                                               int col0, const float (&acc)[BLOCK_N / 2]) {
  if (inside) {
    const bool bias = p.bias != nullptr;
    const bool wide = p.vec8;
    switch (p.epilogue) {
      case EPI_BIAS_BF16:
        if (wide) {
          if (bias) epi_tile<EPI_BIAS_BF16, true, BLOCK_N, true>(p, alpha, row, col0, acc);
          else epi_tile<EPI_BIAS_BF16, false, BLOCK_N, true>(p, alpha, row, col0, acc);
        } else {
          if (bias) epi_tile<EPI_BIAS_BF16, true, BLOCK_N>(p, alpha, row, col0, acc);
          else epi_tile<EPI_BIAS_BF16, false, BLOCK_N>(p, alpha, row, col0, acc);
        }
        break;
      case EPI_BIAS_GELU_BF16:
        if (wide) {
          if (bias) epi_tile<EPI_BIAS_GELU_BF16, true, BLOCK_N, true>(p, alpha, row, col0, acc);
          else epi_tile<EPI_BIAS_GELU_BF16, false, BLOCK_N, true>(p, alpha, row, col0, acc);
        } else {
          if (bias) epi_tile<EPI_BIAS_GELU_BF16, true, BLOCK_N>(p, alpha, row, col0, acc);
          else epi_tile<EPI_BIAS_GELU_BF16, false, BLOCK_N>(p, alpha, row, col0, acc);
        }
        break;
      case EPI_GELU_BWD_BF16:
        if (wide) epi_tile<EPI_GELU_BWD_BF16, false, BLOCK_N, true>(p, alpha, row, col0, acc);
        else epi_tile<EPI_GELU_BWD_BF16, false, BLOCK_N>(p, alpha, row, col0, acc);
        break;
      case EPI_ADD_BF16:
        if (wide) epi_tile<EPI_ADD_BF16, false, BLOCK_N, true>(p, alpha, row, col0, acc);
        else epi_tile<EPI_ADD_BF16, false, BLOCK_N>(p, alpha, row, col0, acc);
        break;
      case EPI_BIAS_F32:
        if (bias) epi_tile<EPI_BIAS_F32, true, BLOCK_N>(p, alpha, row, col0, acc);
        else epi_tile<EPI_BIAS_F32, false, BLOCK_N>(p, alpha, row, col0, acc);
        break;
      default:
        epi_tile<EPI_ATOMIC_F32, false, BLOCK_N>(p, alpha, row, col0, acc);
    }
  } else {
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      if (n0 + j * 8 >= p.N) break;  // warp-uniform
      epi_pair(p, alpha, row, col0 + j * 8, acc[4 * j], acc[4 * j + 1]);
      epi_pair(p, alpha, row + 8, col0 + j * 8, acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
}

__device__ __forceinline__ bool tile_inside(const GemmParams& p, const WorkItem& wi, int bn) {
  return p.vec2 && wi.m0 + BLOCK_M <= p.M && wi.n0 + bn <= p.N;
}

// In-kernel split-K fix-up of one warp's share (16 rows x BLOCK_N) of a tile half (rows 64 half .. 64 half + 63).
// The work item stores alpha * acc into its slot, in fragment order (float4 j of warpgroup thread t at j * 128 + t,
// so every thread later reads back exactly the values it wrote, 16 bytes at a time), and publishes it: a release
// fence by every lane, then one acq_rel add on the warp's counter.  The item whose add brings the counter to
// p.splits is the last arriver: it returns true with acc = t, where t = 0, t += alpha * acc_s for s = 0 .. splits - 1
// in split order (its own split from its registers, the others from their slots) — the order partials_reduce adds
// rows in, so the sum does not depend on which item arrives last.  Every other item returns false and is done.  No
// warp ever waits for another, so the kernel cannot deadlock however few of its CTAs are resident.
template <int BLOCK_N>
__device__ __forceinline__ bool splitk_fixup(const GemmParams& p, int tile, int half, int split, float alpha,
                                             float (&acc)[BLOCK_N / 2]) {
  constexpr int V = BLOCK_N / 8;  // float4 per thread
  // float4 loads in flight per slot: 8 spills the 256-wide tile's 128 accumulator registers (check with -Xptxas -v)
  constexpr int CHUNK = BLOCK_N == 256 ? 4 : 8;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const long long slot = 64LL * BLOCK_N;  // floats per (tile, split, half)
  float4* base = reinterpret_cast<float4*>(p.slots + ((long long)tile * p.splits * 2 + half) * slot) + t;
  float4* mine = base + split * (2 * slot / 4);
#pragma unroll
  for (int j = 0; j < V; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[4 * j + e] = __fmul_rn(acc[4 * j + e], alpha);
    __stcg(mine + j * 128, make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]));
  }
  fence_acq_rel_gpu();
  __syncwarp();
  unsigned before = 0;
  if (lane == 0) before = atom_add_acq_rel_gpu(p.arrived + (tile * 2 + half) * 4 + (t >> 5), 1u);
  before = __shfl_sync(0xffffffffu, before, 0);
  if (before != (unsigned)p.splits - 1) return false;
  fence_acq_rel_gpu();
#pragma unroll
  for (int j0 = 0; j0 < V; j0 += CHUNK) {
    float4 s4[CHUNK];
#pragma unroll
    for (int j = 0; j < CHUNK; ++j) s4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < p.splits; ++s) {
      float4 v[CHUNK];
      if (s == split) {
#pragma unroll
        for (int j = 0; j < CHUNK; ++j) {
          const int a = 4 * (j0 + j);
          v[j] = make_float4(acc[a], acc[a + 1], acc[a + 2], acc[a + 3]);
        }
      } else {
        const float4* src = base + s * (2 * slot / 4);
#pragma unroll
        for (int j = 0; j < CHUNK; ++j) v[j] = __ldcg(src + (j0 + j) * 128);
      }
#pragma unroll
      for (int j = 0; j < CHUNK; ++j) {
        s4[j].x = __fadd_rn(s4[j].x, v[j].x);
        s4[j].y = __fadd_rn(s4[j].y, v[j].y);
        s4[j].z = __fadd_rn(s4[j].z, v[j].z);
        s4[j].w = __fadd_rn(s4[j].w, v[j].w);
      }
    }
#pragma unroll
    for (int j = 0; j < CHUNK; ++j) {
      const int a = 4 * (j0 + j);
      acc[a] = s4[j].x;
      acc[a + 1] = s4[j].y;
      acc[a + 2] = s4[j].z;
      acc[a + 3] = s4[j].w;
    }
  }
  return true;
}

// the split-K fix-up (when p.slots is set) and then the epilogue of one tile half; a split-K item that is not its
// tile's last arriver has no epilogue.  alpha: the scale of acc (1 for in-register k-segment sums, which carry it)
template <int BLOCK_N>
__device__ __forceinline__ void finish_block(const GemmParams& p, const WorkItem& wi, int n_tiles, int kb_per,
                                             bool inside, float alpha, int half, int row, int col0,
                                             float (&acc)[BLOCK_N / 2]) {
  if (p.slots != nullptr) {
    const int tile = (wi.m0 / BLOCK_M) * n_tiles + wi.n0 / BLOCK_N;
    if (!splitk_fixup<BLOCK_N>(p, tile, half, wi.kb_begin / kb_per, alpha, acc)) return;
    alpha = 1.f;  // t carries it
  }
  epilogue_block<BLOCK_N>(p, inside, alpha, wi.n0, row, col0, acc);
}

// named barriers of the ping-pong hand-off: consumer warpgroup c waits on TURN_BAR + c for its turn at the MMAs
constexpr int TURN_BAR = 1;

// TMA producer (one thread): streams the k-blocks of the CTA's work items, in order, into the STAGES-deep ring.
// ELEM: operand bytes per element (2 = bf16, 1 = e4m3).  A k-block is 128 bytes of K whatever the type (64 bf16 or
// 128 e4m3), so the stage bytes, the 128B swizzle and the box shapes are the same for both; only the k coordinate
// of a block differs.
template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN, int ELEM = 2>
__device__ __forceinline__ void produce_ring(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, uint8_t* smem,
                                             const Ring<STAGES>& ring, int num_work, int m_tiles, int n_tiles,
                                             int total_kb, int kb_per) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  uint32_t it = 0;
  for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
    const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, kb_per, BLOCK_N);
    for (int i = 0; i < wi.num_kb; ++i, ++it) {
      const int s = ring.acquire(it, L::STAGE_BYTES);
      uint64_t* bar = &ring.full[s];
      uint8_t* sa = smem + s * L::STAGE_BYTES;
      uint8_t* sb = sa + L::A_BYTES;
      const int k_elem = (wi.kb_begin + i) * (128 / ELEM);
      if (!A_MN) {
        tma_load_2d(sa, tmap_a, bar, k_elem, wi.m0);  // box {128 B of k, 128 rows}
      } else {
#pragma unroll
        for (int c = 0; c < BLOCK_M / 64; ++c)  // box {64 m, 64 k-rows}
          tma_load_2d(sa + c * (BLOCK_K * 128), tmap_a, bar, wi.m0 + c * 64, k_elem);
      }
      if (!B_MN) {
        tma_load_2d(sb, tmap_b, bar, k_elem, wi.n0);  // box {128 B of k, BLOCK_N rows}
      } else {
#pragma unroll
        for (int c = 0; c < BLOCK_N / 64; ++c)
          tma_load_2d(sb + c * (BLOCK_K * 128), tmap_b, bar, wi.n0 + c * 64, k_elem);
      }
    }
  }
}

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(PIPELINE_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const GemmParams p, const int num_work) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  constexpr bool PING = BLOCK_N <= 128;  // ping-pong schedule (else cooperative), see the top of this file
  // in-register k-segment sums (p.kb_seg): the 64-wide tile has the registers for a second accumulator set
  constexpr bool FOLD = BLOCK_N == 64;
  Ring<STAGES> ring;
  uint8_t* smem = kernel_prologue(ring, L::BAR_OFFSET, PING ? 1 : 2, &tmap_a, &tmap_b);  // consumers per stage

  const int wg = threadIdx.x >> 7;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int total_kb = (p.Kc + BLOCK_K - 1) / BLOCK_K;
  const int kb_per = p.k_blocks_per_split;

  if (wg == 0) {
    if (producer_regs())
      produce_ring<BLOCK_N, STAGES, A_MN, B_MN>(&tmap_a, &tmap_b, smem, ring, num_work, m_tiles, n_tiles, total_kb,
                                                kb_per);
  } else if constexpr (!PING) {
    // ------------------------------ cooperative consumers ------------------------------
    consumer_regs();
    const int c = wg - 1;  // rows [64 c, 64 c + 64) of every tile
    const int t = threadIdx.x & 127;
    const int warp = t >> 5, lane = t & 31;
    uint32_t it = 0;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
      const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, kb_per, BLOCK_N);
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int e = 0; e < BLOCK_N / 2; ++e) acc[e] = 0.f;
      const int last = mma_kblocks<BLOCK_N, A_MN, B_MN, L::STAGE_BYTES, L::A_BYTES>(ring, smem, c * (64 * 128), acc,
                                                                                     0, wi.num_kb, it, t == 0);
      mma_drain(ring, last, acc, t == 0);
      const int row = wi.m0 + c * 64 + warp * 16 + (lane >> 2);
      const int col0 = wi.n0 + 2 * (lane & 3);
      finish_block<BLOCK_N>(p, wi, n_tiles, kb_per, tile_inside(p, wi, BLOCK_N), p.alpha, c, row, col0, acc);
    }
  } else {
    // ------------------------------ ping-pong consumers ------------------------------
    // Warpgroup c owns the CTA's items j = c, c + 2, c + 4, ...: all 128 rows of each.  Its mainloop of item j starts
    // only once the other warpgroup has issued its last MMA of item j - 1 (TURN_BAR + c), and it hands over the same
    // way when it has issued its own, so the two mainloops take turns in item order and each warpgroup's epilogue runs
    // under the other's MMAs.  The hand-off is also what keeps the two warpgroups' ring waits in order (Ring::wait):
    // every k-block before item j has passed its wait when item j starts.
    consumer_regs();
    const int c = wg - 1;
    const int t = threadIdx.x & 127;
    const int warp = t >> 5, lane = t & 31;
    uint32_t it = 0;  // ring position: advances over the other warpgroup's k-blocks as well as this one's
    int j = 0;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x, ++j) {
      const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, kb_per, BLOCK_N);
      if ((j & 1) != c) {  // the other warpgroup's item (num_kb differs between items under split-K)
        it += wi.num_kb;
        continue;
      }
      float acc[2][BLOCK_N / 2];  // rows 0-63 and 64-127 of the tile
#pragma unroll
      for (int e = 0; e < BLOCK_N / 2; ++e) acc[0][e] = acc[1][e] = 0.f;
      // k-segments (see GemmParams::kb_seg): the MMAs restart from zero at each segment, and sum += alpha * acc
      // after it, in k order
      const bool fold = FOLD && p.kb_seg < wi.num_kb;
      const int seg = fold ? p.kb_seg : wi.num_kb;
      float sum[2][FOLD ? BLOCK_N / 2 : 1];
      if constexpr (FOLD) {
#pragma unroll
        for (int e = 0; e < BLOCK_N / 2; ++e) sum[0][e] = sum[1][e] = 0.f;
      }
      if (j > 0) named_bar(TURN_BAR + c, 256);
      for (int i0 = 0; i0 < wi.num_kb; i0 += seg) {
        const int i1 = min(wi.num_kb, i0 + seg);
        const int last =
            mma_kblocks<BLOCK_N, 2, A_MN, B_MN, L::STAGE_BYTES, L::A_BYTES>(ring, smem, 0, acc, i0, i1, it, t == 0);
        if (i1 == wi.num_kb && w + (int)gridDim.x < num_work)
          named_bar_arrive(TURN_BAR + (c ^ 1), 256);  // the next item's turn
        mma_drain(ring, last, acc, t == 0);
        if constexpr (FOLD) {
          if (fold) {
#pragma unroll
            for (int e = 0; e < BLOCK_N / 2; ++e) {
              sum[0][e] = __fadd_rn(sum[0][e], __fmul_rn(acc[0][e], p.alpha));
              sum[1][e] = __fadd_rn(sum[1][e], __fmul_rn(acc[1][e], p.alpha));
            }
          }
        }
      }
      float alpha = p.alpha;
      if constexpr (FOLD) {
        if (fold) {
#pragma unroll
          for (int e = 0; e < BLOCK_N / 2; ++e) {
            acc[0][e] = sum[0][e];
            acc[1][e] = sum[1][e];
          }
          alpha = 1.f;  // the sums carry it
        }
      }
      const bool inside = tile_inside(p, wi, BLOCK_N);
      const int row = wi.m0 + warp * 16 + (lane >> 2);
      const int col0 = wi.n0 + 2 * (lane & 3);
      finish_block<BLOCK_N>(p, wi, n_tiles, kb_per, inside, alpha, 0, row, col0, acc[0]);
      finish_block<BLOCK_N>(p, wi, n_tiles, kb_per, inside, alpha, 1, row + 64, col0, acc[1]);
    }
  }
}

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int splits,
                       cudaStream_t stream) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  auto kern = gemm_wgmma_kernel<BLOCK_N, STAGES, A_MN, B_MN>;
  const char* name = "univl_gemm_bf16";
  if (int rc = persistent_prepare(kern, L::DYN_BYTES, name)) return rc;
  const long long work =
      (long long)((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N) * (long long)splits;
  return persistent_launch(kern, name, work, L::DYN_BYTES, stream, ta, tb, p, (int)work);
}

template <int BLOCK_N, int STAGES>
static int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          int splits, cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch_gemm<BLOCK_N, STAGES, false, false>(ta, tb, p, splits, stream);
  if (!a_mn && b_mn) return launch_gemm<BLOCK_N, STAGES, false, true>(ta, tb, p, splits, stream);
  if (a_mn && b_mn) return launch_gemm<BLOCK_N, STAGES, true, true>(ta, tb, p, splits, stream);
  return launch_gemm<BLOCK_N, STAGES, true, false>(ta, tb, p, splits, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// FP8 (e4m3 x e4m3) GEMM with fine-grained scaling, forward only:
//   D[M,N] = epilogue( sum_kb  sa[kb, m] * sb[n / 128, kb] * sum_{k in block kb} A(m,k) B(n,k) )
// A [M,K] e4m3 with one scale per (row, 128-column block), sa laid out [K/128, M]; B [N,K] e4m3 with one scale per
// 128 x 128 block, sb [N/128, K/128].  Both K-major (8-bit wgmma takes no other layout).
// The producer, ring, work decoding and descriptors are the bf16 kernel's: a k-block is 128 e4m3 = 128 bytes, one
// stage holds the same bytes with the same swizzle, and a k32 step advances the descriptors by the same 32 bytes.
// The consumers run the cooperative schedule on 128 x 128 tiles (each warpgroup 64 rows).  Every k-block is one
// scaling block: its four k32 wgmmas accumulate into a temporary, which is then promoted into the fp32 accumulator
// with one FMA by sa * sb (a product of two powers of two, exact).  So the tensor cores' in-instruction accumulation,
// whose precision is not specified for 8-bit inputs, only ever sums 128 products.  The accumulator and two
// temporaries (3 x 64 floats per thread) fit in registers without spills, which the 256-wide tile (3 x 128) would not.
// Epilogues: FP8_EPI_BIAS_BF16  out(bf16) = acc + bias (the bf16 kernel's unchecked / checked epilogue code)
//            FP8_EPI_GELU_E4M3  out(e4m3), out_scale = gelu_erf(acc + bias) quantized per (row, 128-column block), the
//                               scale found from the accumulator fragment with two quad shuffles
enum Fp8Epilogue : int { FP8_EPI_BIAS_BF16 = 0, FP8_EPI_GELU_E4M3 = 1 };

struct Fp8Params {
  const float* a_scale;  // [K/128, M]
  const float* b_scale;  // [N/128, K/128]
  uint8_t* out_q;        // FP8_EPI_GELU_E4M3: e4m3 [M, ldo]
  float* out_scale;      // FP8_EPI_GELU_E4M3: [N/128, M]
};

constexpr int FP8_BLOCK_N = 128;
constexpr int FP8_STAGES = 6;

template <int EPI, bool PAIRS>
__global__ void __launch_bounds__(PIPELINE_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmParams p, const Fp8Params f, const int num_work) {
  using L = GemmSmem<FP8_BLOCK_N, FP8_STAGES>;
  Ring<FP8_STAGES> ring;
  uint8_t* smem = kernel_prologue(ring, L::BAR_OFFSET, 2, &tmap_a, &tmap_b);

  const int wg = threadIdx.x >> 7;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = p.N / FP8_BLOCK_N;
  const int total_kb = p.Kc / 128;

  if (wg == 0) {
    if (producer_regs())
      produce_ring<FP8_BLOCK_N, FP8_STAGES, false, false, 1>(&tmap_a, &tmap_b, smem, ring, num_work, m_tiles, n_tiles,
                                                              total_kb, total_kb);
    return;
  }
  consumer_regs();
  const int c = wg - 1;  // rows [64 c, 64 c + 64) of every tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31;
  const int M = p.M;
  uint32_t it = 0;
  for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
    const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, total_kb, FP8_BLOCK_N);
    const int row = wi.m0 + c * 64 + warp * 16 + (lane >> 2);  // and row + 8
    const bool in0 = row < M, in1 = row + 8 < M;
    const float* sa = f.a_scale + row;
    const float* sb = f.b_scale + (long long)(wi.n0 / FP8_BLOCK_N) * total_kb;
    float acc[FP8_BLOCK_N / 2];
#pragma unroll
    for (int e = 0; e < FP8_BLOCK_N / 2; ++e) acc[e] = 0.f;
    // Block kb's four wgmmas go into a temporary (issue), which is then added into acc with the block's scales
    // (promote, after waiting until at most `newer` younger wgmma groups are in flight).  With an even number of
    // blocks (PAIRS) two temporaries alternate, so that the MMAs of block kb + 1 run while block kb is promoted; the
    // wgmmas and waits sit in straight-line code and a loop, never under a data-dependent branch, which would make
    // ptxas serialize them.  An odd number of blocks takes one temporary and waits for each block's MMAs.
    auto issue = [&](float (&tmp)[FP8_BLOCK_N / 2], int kb) {
      const int s = ring.wait(it + kb);
      const uint32_t a_s = smem_u32(smem + s * L::STAGE_BYTES) + c * (64 * 128);
      const uint32_t b_s = smem_u32(smem + s * L::STAGE_BYTES) + L::A_BYTES;
      wgmma_fence();
      fence_regs(tmp);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        WgmmaSSE4M3N128::mma(tmp, make_smem_desc_sw128(a_s + k * 32, 16, 1024),
                             make_smem_desc_sw128(b_s + k * 32, 16, 1024), k > 0 ? 1 : 0);
      wgmma_commit();
      fence_regs(tmp);
    };
    auto promote = [&](auto newer, float (&tmp)[FP8_BLOCK_N / 2], int kb) {
      // the block's scales, loaded before the wait so their latency hides under it
      const float bs = __ldg(sb + kb);
      const float s0 = in0 ? __ldg(sa + (long long)kb * M) : 0.f;
      const float s1 = in1 ? __ldg(sa + (long long)kb * M + 8) : 0.f;
      wgmma_wait<decltype(newer)::value>();
      fence_regs(tmp);
      if (t == 0) ring.release(ring.stage(it + kb));
      const float f0 = s0 * bs, f1 = s1 * bs;
#pragma unroll
      for (int j = 0; j < FP8_BLOCK_N / 8; ++j) {
        acc[4 * j] = __fmaf_rn(tmp[4 * j], f0, acc[4 * j]);
        acc[4 * j + 1] = __fmaf_rn(tmp[4 * j + 1], f0, acc[4 * j + 1]);
        acc[4 * j + 2] = __fmaf_rn(tmp[4 * j + 2], f1, acc[4 * j + 2]);
        acc[4 * j + 3] = __fmaf_rn(tmp[4 * j + 3], f1, acc[4 * j + 3]);
      }
    };
    using One = std::integral_constant<int, 1>;
    using None = std::integral_constant<int, 0>;
    float ta[FP8_BLOCK_N / 2];
    if constexpr (PAIRS) {
      float tb[FP8_BLOCK_N / 2];
      issue(ta, 0);
      issue(tb, 1);
      int kb = 0;
      for (; kb + 2 < total_kb; kb += 2) {
        promote(One(), ta, kb);
        issue(ta, kb + 2);
        promote(One(), tb, kb + 1);
        issue(tb, kb + 3);
      }
      promote(One(), ta, kb);
      promote(None(), tb, kb + 1);
    } else {
      for (int kb = 0; kb < total_kb; ++kb) {
        issue(ta, kb);
        promote(None(), ta, kb);
      }
    }
    it += total_kb;
    const int col0 = wi.n0 + 2 * (lane & 3);
    if constexpr (EPI == FP8_EPI_BIAS_BF16) {
      if (tile_inside(p, wi, FP8_BLOCK_N)) {
        if (p.vec8) epi_tile<EPI_BIAS_BF16, true, FP8_BLOCK_N, true>(p, p.alpha, row, col0, acc);
        else epi_tile<EPI_BIAS_BF16, true, FP8_BLOCK_N>(p, p.alpha, row, col0, acc);
      } else {
#pragma unroll
        for (int j = 0; j < FP8_BLOCK_N / 8; ++j) {
          epi_pair(p, p.alpha, row, col0 + j * 8, acc[4 * j], acc[4 * j + 1]);
          epi_pair(p, p.alpha, row + 8, col0 + j * 8, acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
    } else {
      // the tile's 128 columns are one scaling block: a row's amax is the max over its quad's fragments
      const float* bias = p.bias + col0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // rows row, row + 8
        float amax = 0.f;
#pragma unroll
        for (int j = 0; j < FP8_BLOCK_N / 8; ++j) {
          const float v0 = gelu_erf(__fadd_rn(acc[4 * j + 2 * h], __ldg(bias + 8 * j)));
          const float v1 = gelu_erf(__fadd_rn(acc[4 * j + 2 * h + 1], __ldg(bias + 8 * j + 1)));
          acc[4 * j + 2 * h] = v0;
          acc[4 * j + 2 * h + 1] = v1;
          amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
        }
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        const float sc = e4m3_scale(amax);
        const float inv = e4m3_inv_scale(sc);
        const int r = row + 8 * h;
        if (r < M) {
          uint8_t* q = f.out_q + (long long)r * p.ldo + col0;
#pragma unroll
          for (int j = 0; j < FP8_BLOCK_N / 8; ++j)
            *reinterpret_cast<uint16_t*>(q + 8 * j) =
                e4m3x2(__fmul_rn(acc[4 * j + 2 * h], inv), __fmul_rn(acc[4 * j + 2 * h + 1], inv));
          if ((lane & 3) == 0) f.out_scale[(long long)(wi.n0 / FP8_BLOCK_N) * M + r] = sc;
        }
      }
    }
  }
}

template <int EPI, bool PAIRS>
static int launch_gemm_fp8(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, const Fp8Params& f,
                           cudaStream_t stream) {
  using L = GemmSmem<FP8_BLOCK_N, FP8_STAGES>;
  auto kern = gemm_fp8_kernel<EPI, PAIRS>;
  const char* name = "univl_gemm_fp8";
  if (int rc = persistent_prepare(kern, L::DYN_BYTES, name)) return rc;
  const long long work = (long long)((p.M + BLOCK_M - 1) / BLOCK_M) * (p.N / FP8_BLOCK_N);
  return persistent_launch(kern, name, work, L::DYN_BYTES, stream, ta, tb, p, f, (int)work);
}

// ------------------------------------------------------------------------------------------------------------------
// Vocabulary cross-entropy without logits in HBM (the MLM and caption heads):
//   logit[r, c] = sum_k x(r,k) W(c,k) + bias[c],  loss = mean over groups of the mean over scored rows of
//   logsumexp(logit[r, :V]) - logit[r, labels[r]]
// The mainloop is the bf16 kernel's cooperative one on 128 x 128 tiles (both operands K-major), so every logit has the
// bits EPI_BIAS_F32 gives it: the same k16 wgmma chain and the same fp32 bias add.  A work item is one 128-row tile x
// a chunk of VX_CHUNK consecutive 128-column tiles; the CTA walks the chunk's tiles in column order.
//   forward  (MODE = VX_FWD): each thread keeps, per row of its fragment, a running max m and sum s of exp(logit - m)
//            over the columns it holds, updated tile by tile; at the end of the item the four lanes of a quad fold
//            their (m, s) with two xor shuffles (symmetric, so every lane gets the same bits) and lane 0 writes the
//            row's (m, s, label logit) for the chunk.  vocab_xent_rows_kernel folds the chunks in chunk order.
//            Without labels every row is scored (the beam search's lse pass) and no label logit is taken.
//   backward (MODE = VX_BWD):  dl[r, c] = (exp(logit - lse[r]) - [c == label]) * g(r) as bf16, the arithmetic of
//            xent_bwd_kernel; columns [V, ld_d) and rows with label -1 get 0.
//   beam     (MODE = VX_BEAM): key = (logit - lse[r]) + score[r] for every column c < V (Beam.advance's word_prob +
//            scores); each thread keeps its row's VX_BEAM_MAX best (key, c) in registers, in the order key descending
//            then c ascending; at the end of the item the four lanes of a quad merge their lists with shuffles and
//            lane 0 writes the row's list for the chunk.  vocab_beam_merge_kernel takes an instance's top n_beam from
//            its live rows' lists.
// The chunking is a pure function of (T, V) (vx_plan), never of the SMs in use, so the bits do not depend on the
// grid, reserved SMs or which CTA runs an item.
constexpr int VX_BLOCK_N = 128;
constexpr int VX_STAGES = 6;
constexpr int VX_FWD = 0, VX_BWD = 1, VX_BEAM = 2;
constexpr int VX_BEAM_MAX = 8;  // candidates a beam work item keeps per row: the largest n_beam

// (k1, i1) comes before (k2, i2) in the beam order: key descending, then index ascending (a total order on distinct
// indices, so every selection by it is exact)
__device__ __forceinline__ bool vb_before(float k1, int i1, float k2, int i2) {
  return k1 > k2 || (k1 == k2 && i1 < i2);
}

// insert (key, idx) into the sorted list (k, ix) if it beats the last entry; the list stays sorted by vb_before
__device__ __forceinline__ void vb_insert(float (&k)[VX_BEAM_MAX], int (&ix)[VX_BEAM_MAX], float key, int idx) {
  if (!vb_before(key, idx, k[VX_BEAM_MAX - 1], ix[VX_BEAM_MAX - 1])) return;
  k[VX_BEAM_MAX - 1] = key;
  ix[VX_BEAM_MAX - 1] = idx;
#pragma unroll
  for (int i = VX_BEAM_MAX - 1; i > 0; --i) {
    if (vb_before(k[i], ix[i], k[i - 1], ix[i - 1])) {
      const float tk = k[i]; k[i] = k[i - 1]; k[i - 1] = tk;
      const int ti = ix[i]; ix[i] = ix[i - 1]; ix[i - 1] = ti;
    }
  }
}

struct VocabXentParams {
  int T, V, Kc;
  int m_tiles, n_tiles, chunks, chunk_tiles;
  const float* bias;        // nullable
  const long long* labels;  // [T], -1 = not scored
  float4* part;             // forward: [T, chunks] (m, s, label logit, 0)
  // backward and beam
  const float* lse;
  // beam
  const float* score;  // [T]
  int2* cand;          // [T, chunks, VX_BEAM_MAX] (key bits, column); unfilled entries (-inf, INT_MAX)
  const float* count;   // [groups]
  const float* gscale;  // nullable: 1
  int rows_per_group, groups;
  bf16* dl;
  long long ld_d;
};

template <int MODE>
__global__ void __launch_bounds__(PIPELINE_THREADS, 1)
vocab_xent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const VocabXentParams p, const int num_work) {
  using L = GemmSmem<VX_BLOCK_N, VX_STAGES>;
  Ring<VX_STAGES> ring;
  uint8_t* smem = kernel_prologue(ring, L::BAR_OFFSET, 2, &tmap_a, &tmap_b);
  const int wg = threadIdx.x >> 7;
  const int total_kb = (p.Kc + BLOCK_K - 1) / BLOCK_K;

  // work item w: chunk w / m_tiles, m-tile w % m_tiles — the CTAs in flight share a few chunks of W through L2
  if (wg == 0) {
    if (!producer_regs()) return;
    uint32_t it = 0;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
      const int chunk = w / p.m_tiles;
      const int m0 = (w - chunk * p.m_tiles) * BLOCK_M;
      const int nt1 = min(p.n_tiles, (chunk + 1) * p.chunk_tiles);
      for (int nt = chunk * p.chunk_tiles; nt < nt1; ++nt) {
        for (int kb = 0; kb < total_kb; ++kb, ++it) {
          const int s = ring.acquire(it, L::STAGE_BYTES);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          tma_load_2d(sa, &tmap_a, &ring.full[s], kb * BLOCK_K, m0);
          tma_load_2d(sa + L::A_BYTES, &tmap_b, &ring.full[s], kb * BLOCK_K, nt * VX_BLOCK_N);
        }
      }
    }
    return;
  }
  consumer_regs();
  const int c = wg - 1;  // rows [64 c, 64 c + 64) of every tile
  const int t = threadIdx.x & 127;
  const int warp = t >> 5, lane = t & 31, q = lane & 3;
  uint32_t it = 0;
  for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
    const int chunk = w / p.m_tiles;
    const int row = (w - chunk * p.m_tiles) * BLOCK_M + c * 64 + warp * 16 + (lane >> 2);  // and row + 8
    long long lab[2];
    float m[2], s[2], xt[2], lse[2], g[2], sc[2];
    float bk[2][VX_BEAM_MAX];
    int bi[2][VX_BEAM_MAX];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      lab[h] = (r < p.T && p.labels != nullptr) ? __ldg(p.labels + r) : -1;
      m[h] = -INFINITY;
      s[h] = 0.f;
      xt[h] = 0.f;
      if constexpr (MODE == VX_BEAM) {
        lse[h] = r < p.T ? __ldg(p.lse + r) : 0.f;
        sc[h] = r < p.T ? __ldg(p.score + r) : 0.f;
#pragma unroll
        for (int i = 0; i < VX_BEAM_MAX; ++i) {
          bk[h][i] = -INFINITY;
          bi[h][i] = INT_MAX;
        }
      }
      if constexpr (MODE == VX_BWD) {
        lse[h] = 0.f;
        g[h] = 0.f;
        if (lab[h] != -1) {
          lse[h] = __ldg(p.lse + r);
          // (gscale / G) / count: xent_bwd_kernel's scale, in its order
          g[h] = ((p.gscale ? __ldg(p.gscale) : 1.f) / (float)p.groups) / __ldg(p.count + r / p.rows_per_group);
        }
      }
    }
    const int nt1 = min(p.n_tiles, (chunk + 1) * p.chunk_tiles);
    for (int nt = chunk * p.chunk_tiles; nt < nt1; ++nt) {
      float acc[VX_BLOCK_N / 2];
#pragma unroll
      for (int e = 0; e < VX_BLOCK_N / 2; ++e) acc[e] = 0.f;
      const int last = mma_kblocks<VX_BLOCK_N, false, false, L::STAGE_BYTES, L::A_BYTES>(ring, smem, c * (64 * 128),
                                                                                          acc, 0, total_kb, it, t == 0);
      mma_drain(ring, last, acc, t == 0);

      const int col0 = nt * VX_BLOCK_N + 2 * q;
      // the logits of this thread's columns (bias added as EPI_BIAS_F32 adds it); columns >= V are never read
#pragma unroll
      for (int j = 0; j < VX_BLOCK_N / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + 8 * j + e;
          const float b = (p.bias != nullptr && col < p.V) ? __ldg(p.bias + col) : 0.f;
          acc[4 * j + e] = __fadd_rn(acc[4 * j + e], b);
          acc[4 * j + 2 + e] = __fadd_rn(acc[4 * j + 2 + e], b);
        }
      }
      if constexpr (MODE == VX_FWD) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float tm = -INFINITY;
#pragma unroll
          for (int j = 0; j < VX_BLOCK_N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (col0 + 8 * j + e < p.V) tm = fmaxf(tm, acc[4 * j + 2 * h + e]);
          if (tm > m[h]) {  // a new running max: rescale the sum (exp(-inf) = 0 on the first tile)
            s[h] = s[h] * __expf(m[h] - tm);
            m[h] = tm;
          }
#pragma unroll
          for (int j = 0; j < VX_BLOCK_N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = col0 + 8 * j + e;
              const float v = acc[4 * j + 2 * h + e];
              if (col < p.V) s[h] += __expf(v - m[h]);
              if (col == lab[h]) xt[h] = v;
            }
        }
      } else if constexpr (MODE == VX_BEAM) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < VX_BLOCK_N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = col0 + 8 * j + e;
              if (col < p.V)
                vb_insert(bk[h], bi[h], __fadd_rn(__fsub_rn(acc[4 * j + 2 * h + e], lse[h]), sc[h]), col);
            }
      } else {
        const int ncol = min(p.ld_d - (long long)nt * VX_BLOCK_N, (long long)VX_BLOCK_N);  // this tile's columns
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = row + 8 * h;
          if (r >= p.T) continue;
          bf16* drow = p.dl + (long long)r * p.ld_d + col0;
          const bool scored = lab[h] != -1;
#pragma unroll
          for (int j = 0; j < VX_BLOCK_N / 8; ++j) {
            if (8 * j + 2 * q >= ncol) break;  // ld_d is even, so the pair is whole
            float d[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = col0 + 8 * j + e;
              d[e] = 0.f;
              if (scored && col < p.V)
                d[e] = (__expf(acc[4 * j + 2 * h + e] - lse[h]) - (col == lab[h] ? 1.f : 0.f)) * g[h];
            }
            *reinterpret_cast<uint32_t*>(drow + 8 * j) = pack_bf16x2(d[0], d[1]);
          }
        }
      }
    }
    if constexpr (MODE == VX_BEAM) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // merge with the partner lane's list: the top VX_BEAM_MAX of the union in the strict order, so both lanes of
        // the pair (and then all four of the quad) hold the same list
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          float ok[VX_BEAM_MAX];
          int oi[VX_BEAM_MAX];
#pragma unroll
          for (int i = 0; i < VX_BEAM_MAX; ++i) {
            ok[i] = __shfl_xor_sync(0xffffffffu, bk[h][i], o);
            oi[i] = __shfl_xor_sync(0xffffffffu, bi[h][i], o);
          }
#pragma unroll
          for (int i = 0; i < VX_BEAM_MAX; ++i) vb_insert(bk[h], bi[h], ok[i], oi[i]);
        }
        const int r = row + 8 * h;
        if (q == 0 && r < p.T) {
          int2* out = p.cand + ((long long)r * p.chunks + chunk) * VX_BEAM_MAX;
#pragma unroll
          for (int i = 0; i < VX_BEAM_MAX; ++i) out[i] = make_int2(__float_as_int(bk[h][i]), bi[h][i]);
        }
      }
    }
    if constexpr (MODE == VX_FWD) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float mo = __shfl_xor_sync(0xffffffffu, m[h], o);
          const float so = __shfl_xor_sync(0xffffffffu, s[h], o);
          const float xo = __shfl_xor_sync(0xffffffffu, xt[h], o);
          const float mx = fmaxf(m[h], mo);
          const float a = m[h] == -INFINITY ? 0.f : s[h] * __expf(m[h] - mx);
          const float b = mo == -INFINITY ? 0.f : so * __expf(mo - mx);
          m[h] = mx;
          s[h] = a + b;    // commutative: both lanes of the pair get the same bits
          xt[h] += xo;     // one lane of the quad holds the label column, the others add 0
        }
        const int r = row + 8 * h;
        if (q == 0 && r < p.T) p.part[(long long)r * p.chunks + chunk] = make_float4(m[h], s[h], xt[h], 0.f);
      }
    }
  }
}

// Row r (one thread each): fold its chunk records in chunk order into lse[r] = m + log(s) and nll[r] = lse[r] - the
// label logit, taken from the label's chunk.  Rows with label -1 get lse 0, as xent_fwd_kernel gives them.  Without
// labels (null) every row gets its lse and no nll is written.
__global__ void __launch_bounds__(256)
vocab_xent_rows_kernel(const float4* __restrict__ part, const long long* __restrict__ labels, int T, int V, int chunks,
                       int chunk_cols, float* __restrict__ lse_out, float* __restrict__ nll) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T) return;
  const long long lab = labels != nullptr ? labels[r] : 0;
  if (lab == -1) {
    lse_out[r] = 0.f;
    return;
  }
  const float4* pr = part + (long long)r * chunks;
  float4 f = pr[0];
  float m = f.x, s = f.y;
  for (int k = 1; k < chunks; ++k) {
    f = pr[k];
    const float mx = fmaxf(m, f.x);
    s = s * __expf(m - mx) + f.y * __expf(f.x - mx);
    m = mx;
  }
  const float lse = m + __logf(s);
  lse_out[r] = lse;
  if (labels == nullptr) return;
  // a label outside [0, V) scores NaN instead of reading past the row
  nll[r] = (lab >= 0 && lab < V) ? lse - pr[lab / chunk_cols].z : __int_as_float(0x7fc00000);
}

// Per group (one CTA each): the sum of its scored rows' nll and their count, in a fixed order (no float atomics).
constexpr int VX_GROUP_THREADS = 512;
__global__ void __launch_bounds__(VX_GROUP_THREADS)
vocab_xent_group_kernel(const float* __restrict__ nll, const long long* __restrict__ labels, int rows_per_group,
                        float* __restrict__ sum_count, int groups) {
  __shared__ float red[2][VX_GROUP_THREADS];
  const int grp = blockIdx.x;
  float sum = 0.f, cnt = 0.f;
  for (int i = threadIdx.x; i < rows_per_group; i += VX_GROUP_THREADS) {
    const long long r = (long long)grp * rows_per_group + i;
    if (labels[r] == -1) continue;
    sum += nll[r];
    cnt += 1.f;
  }
  red[0][threadIdx.x] = sum;
  red[1][threadIdx.x] = cnt;
  __syncthreads();
  for (int o = VX_GROUP_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] += red[0][threadIdx.x + o];
      red[1][threadIdx.x] += red[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    sum_count[grp] = red[0][0];
    sum_count[groups + grp] = red[1][0];
  }
}

// xent_sum_kernel's arithmetic (csrc/loss.cu): mean over groups of sum / count, 0 / 0 = NaN for a group without a scored row
__global__ void vocab_xent_mean_kernel(const float* __restrict__ sum_count, int groups, float* __restrict__ out) {
  float acc = sum_count[0] / sum_count[groups];
  for (int g = 1; g < groups; ++g) acc += sum_count[g] / sum_count[groups + g];
  *out = groups > 1 ? acc / (float)groups : acc;
}

// Instance i (one CTA each): its n_beam best candidates from the lists of its live rows i n_beam + k, k < n_live[i]
// (clamped to [0, n_beam]), as (key, flat = k V + c) in the beam order.  Round j takes the best candidate after round
// j - 1's in that order: each thread scans a fixed stride of the lists, then a fixed-shape tree picks the block's best,
// so the result is the exact top n_beam whatever the chunking.  Slots without a candidate get (-inf, -1).
constexpr int VB_MERGE_THREADS = 256;
__global__ void __launch_bounds__(VB_MERGE_THREADS)
vocab_beam_merge_kernel(const int2* __restrict__ cand, const int* __restrict__ n_live, int n_beam, int chunks, int V,
                        float* __restrict__ out_key, int* __restrict__ out_index) {
  __shared__ float sk[VB_MERGE_THREADS / 32];
  __shared__ int si[VB_MERGE_THREADS / 32];
  const int inst = blockIdx.x;
  const int live = min(max(__ldg(n_live + inst), 0), n_beam);
  const int per_row = chunks * VX_BEAM_MAX;
  const int n = live * per_row;
  const int2* base = cand + (long long)inst * n_beam * per_row;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float pk = INFINITY;  // the previous round's pick (none yet: every candidate comes after (+inf, -1))
  int pi = -1;
  for (int j = 0; j < n_beam; ++j) {
    float bk = -INFINITY;
    int bi = INT_MAX;
    for (int e = threadIdx.x; e < n; e += VB_MERGE_THREADS) {
      const int2 c = base[e];
      if (c.y == INT_MAX) continue;  // an unfilled slot
      const float k = __int_as_float(c.x);
      const int flat = (e / per_row) * V + c.y;
      if (vb_before(pk, pi, k, flat) && vb_before(k, flat, bk, bi)) {
        bk = k;
        bi = flat;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (vb_before(ok, oi, bk, bi)) {
        bk = ok;
        bi = oi;
      }
    }
    if (lane == 0) {
      sk[warp] = bk;
      si[warp] = bi;
    }
    __syncthreads();
    bk = sk[0];
    bi = si[0];
    for (int w = 1; w < VB_MERGE_THREADS / 32; ++w)
      if (vb_before(sk[w], si[w], bk, bi)) {
        bk = sk[w];
        bi = si[w];
      }
    __syncthreads();
    if (threadIdx.x == 0) {
      out_key[inst * n_beam + j] = bk;
      out_index[inst * n_beam + j] = bi == INT_MAX ? -1 : bi;
    }
    pk = bk;
    pi = bi;
  }
}

// One beam step's bookkeeping for instance i (one CTA each), after vocab_beam_merge_kernel (Beam.advance,
// modules/beam.py:63-87).  A live instance takes its n_beam picks: hypothesis j continues row k = flat / V of the
// instance with word c = flat mod V, score[i n_beam + j] = key, prev_k[t, i, j] = k, word[t, i, j] = c and the row's
// next input token is c; the instance is done when its top pick's word is eos.  A done instance changes none of these.
// Every row r = i n_beam + j then gets its ancestor list for step t + 1: its parent's (row i n_beam + k, or r itself
// when the instance is done) first t + 1 entries, then its own slot (t + 1) R + r, R = n_inst n_beam.
__global__ void __launch_bounds__(128)
beam_advance_kernel(const float* __restrict__ key, const int* __restrict__ index, int n_beam, int V, int t,
                    long long eos, float* __restrict__ score, int* __restrict__ done,
                    int* __restrict__ prev_k, int* __restrict__ word, long long* __restrict__ tokens,
                    const int* __restrict__ anc_in, int* __restrict__ anc_out, int ld_anc) {
  __shared__ int parent[VX_BEAM_MAX];
  const int inst = blockIdx.x, n_inst = gridDim.x;
  const int R = n_inst * n_beam;
  const bool frozen = done[inst] != 0;
  if (threadIdx.x < n_beam) {
    const int j = threadIdx.x, r = inst * n_beam + j;
    int k = j;
    if (!frozen) {
      const int flat = index[r];
      k = flat / V;
      const int c = flat - k * V;
      score[r] = key[r];
      prev_k[((long long)t * n_inst + inst) * n_beam + j] = k;
      word[((long long)t * n_inst + inst) * n_beam + j] = c;
      tokens[r] = c;
    }
    parent[j] = inst * n_beam + k;
  }
  __syncthreads();
  if (threadIdx.x == 0 && !frozen && index[inst * n_beam] % V == eos) done[inst] = 1;
  const int len = min(t + 2, ld_anc);
  for (int e = threadIdx.x; e < n_beam * len; e += blockDim.x) {
    const int j = e / len, pos = e - j * len;
    const int r = inst * n_beam + j;
    anc_out[(long long)r * ld_anc + pos] =
        pos <= t ? anc_in[(long long)parent[j] * ld_anc + pos] : (t + 1) * R + r;
  }
}

// after vx_params, which runs persistent_prepare
template <int MODE>
static const char* vx_name() {
  return MODE == VX_FWD ? "univl_vocab_xent_fwd" : MODE == VX_BWD ? "univl_vocab_xent_bwd" : "univl_vocab_beam_topk";
}

template <int MODE>
static int launch_vocab_xent(const CUtensorMap& ta, const CUtensorMap& tb, const VocabXentParams& p,
                             cudaStream_t stream) {
  const long long work = (long long)p.m_tiles * p.chunks;
  return persistent_launch(vocab_xent_kernel<MODE>, vx_name<MODE>(), work, GemmSmem<VX_BLOCK_N, VX_STAGES>::DYN_BYTES,
                           stream, ta, tb, p, (int)work);
}

}  // namespace univl

using namespace univl;

namespace {
struct GemmPlan {
  int bn, splits, kb_per, kb_seg;
};
// tile width and split-K factor for a problem — a pure function of the arguments, shared by the launcher and by
// univl_gemm_plan
int plan_gemm(int M, int N, int Kc, int epilogue, int block_n, int split_k, GemmPlan* plan) {
  const int total_kb = (Kc + BLOCK_K - 1) / BLOCK_K;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  int bn = block_n;
  if (bn == 0) {
    bn = 256;
    // Without split-K the tile count alone must fill the SMs.  256 -> 128 below two work items per SM: the 128-wide
    // ping-pong tiles then keep both warpgroups of a CTA busy, where a 256-wide grid of 1.1 waves leaves most SMs idle
    // for its second wave (1536 x 3072 x 768, bias + GELU: 0.036 against 0.044 ms).  128 -> 64 only below one item
    // per SM (the caption step, whose 4096-row GEMMs of 768 columns then go to 64, ran 2.6 % slower when they
    // narrowed at two items per SM as well).  A problem with thousands of tiles keeps the cooperative
    // 256-wide tile: it loads the fewest operand bytes per MMA, and on an H100 SXM at a 400 W power limit the
    // 98304-row GEMMs, which run at that cap, were up to 16 % slower with 128-wide ping-pong tiles (a lower SM clock
    // for the same work; the bias + GELU forward was 2 % faster).
    // The fp32 weight gradients keep 256 and take their parallelism from split-K (cross-encoder wgrads, K = 98304:
    // 256 is 20-45 % faster than 128 or 64).  Their split count follows from the tile count, and it sets the order in
    // which the partial sums are added, so a different tile width would change their bits.
    if (epilogue != EPI_ATOMIC_F32) {
      const auto tiles = [&](int w) { return (long long)m_tiles * ((N + w - 1) / w); };
      if (tiles(256) < 2 * PLAN_SMS) bn = 128;
      if (tiles(128) < PLAN_SMS) bn = 64;
    }
    if (N <= 64) bn = 64;
    else if (N <= 128 && bn > 128) bn = 128;
  }
  UNIVL_CHECK_ARG(bn == 64 || bn == 128 || bn == 256, "gemm: block_n must be 64/128/256");
  const int n_tiles = (N + bn - 1) / bn;
  int splits = 1;
  if (epilogue == EPI_ATOMIC_F32) {
    splits = split_k;
    if (splits == 0) {
      const long long tiles = (long long)m_tiles * n_tiles;
      splits = (int)((2 * PLAN_SMS + tiles - 1) / tiles);
      if (splits > total_kb / 2) splits = total_kb / 2;  // keep >= 2 k-blocks per split
      if (splits < 1) splits = 1;
    }
    if (splits > total_kb) splits = total_kb;
  }
  int kb_per = (total_kb + splits - 1) / splits;
  splits = (total_kb + kb_per - 1) / kb_per;  // no empty split
  int kb_seg = kb_per;
  // Below SPLIT_MIN_K the automatic split plan cuts K into 2-6 k-blocks per split, and its scratch partials cost
  // more than the SMs the splits fill.  Such a weight gradient runs unsplit on the 64-wide ping-pong tile instead,
  // summing the same k-segments in registers in the same order (GemmParams::kb_seg), so it computes the bits of the
  // split plan.  On an H100 SXM every 1536- and 1024-row weight gradient of the FT-Align step ran unsplit at 64 wide
  // in about half the time of its split plan (768 x 768 x 1536: 0.014 against 0.027 ms; 3072 x 768 x 1536: 0.026
  // against 0.052).
  if (epilogue == EPI_ATOMIC_F32 && block_n == 0 && split_k == 0 && Kc < SPLIT_MIN_K && splits > 1) {
    bn = 64;
    splits = 1;
    kb_per = total_kb;
  }
  plan->bn = bn; plan->splits = splits; plan->kb_per = kb_per; plan->kb_seg = kb_seg;
  return UNIVL_OK;
}

// the parameters of an unsplit launch (no split-K slots, kb_seg = kb_per), with the epilogue's vector widths read off
// its operands' alignment
GemmParams gemm_params(int M, int N, int Kc, int kb_per, int epilogue, float alpha, void* out, long long ldo,
                       const float* bias, const void* aux_in, long long ld_aux_in, void* aux_out,
                       long long ld_aux_out) {
  GemmParams p;
  p.M = M; p.N = N; p.Kc = Kc;
  p.k_blocks_per_split = kb_per;
  p.epilogue = epilogue;
  p.alpha = alpha;
  p.out = out; p.ldo = ldo;
  p.bias = bias;
  p.aux_in = reinterpret_cast<const bf16*>(aux_in); p.ld_aux_in = ld_aux_in;
  p.aux_out = reinterpret_cast<bf16*>(aux_out); p.ld_aux_out = ld_aux_out;
  // 2-element vector accesses need every epilogue operand's pairs (even columns) aligned to the pair size
  const bool out_f32 = epilogue == EPI_BIAS_F32 || epilogue == EPI_ATOMIC_F32;
  bool vec2 = ((uintptr_t)out % (out_f32 ? 8 : 4)) == 0 && (ldo % 2) == 0;
  if (aux_in != nullptr) vec2 = vec2 && ((uintptr_t)aux_in % 4) == 0 && (ld_aux_in % 2) == 0;
  if (aux_out != nullptr) vec2 = vec2 && ((uintptr_t)aux_out % 4) == 0 && (ld_aux_out % 2) == 0;
  p.vec2 = vec2 ? 1 : 0;
  // 16-byte stores of the bf16 outputs: 8-column groups start at multiples of 8 columns from a 16-byte aligned base
  bool vec8 = !out_f32 && ((uintptr_t)out % 16) == 0 && (ldo % 8) == 0;
  if (aux_out != nullptr) vec8 = vec8 && ((uintptr_t)aux_out % 16) == 0 && (ld_aux_out % 8) == 0;
  p.vec8 = vec8 ? 1 : 0;
  p.slots = nullptr;
  p.arrived = nullptr;
  p.splits = 1;
  p.kb_seg = kb_per;
  return p;
}
}  // namespace

// Which kernel univl_gemm_bf16 launches for this problem: 1 = the persistent wgmma kernel (the only one); negative =
// error.  Stateless (a function of its arguments): bench.py uses it to attribute per-launch CUDA-event times.
extern "C" int univl_gemm_plan(int M, int N, int Kc, int epilogue, int block_n, int split_k) {
  GemmPlan plan;
  if (int rc = plan_gemm(M, N, Kc, epilogue, block_n, split_k, &plan)) return rc;
  return 1;
}

// Aliasing: aux_in may be out itself, with the same leading dimension (an in-place residual add or GELU backward):
// every element is read and then written by the same thread, and epi_tile loads a chunk ahead only elements that thread
// has not written yet.  Any other overlap of aux_in or aux_out with out is a race between threads and is not
// supported.  No caller in ops.py aliases them.
extern "C" int univl_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                               int b_mn_major, int M, int N, int Kc, void* out, long long ldo, int epilogue,
                               const float* bias, const void* aux_in, long long ld_aux_in, void* aux_out,
                               long long ld_aux_out, float alpha, int block_n, int split_k, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UNIVL_CHECK_ARG(M > 0 && N > 0 && Kc > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, Kc);
  UNIVL_CHECK_ARG(A && B && out, "gemm: null operand");
  UNIVL_CHECK_ARG((lda % 8) == 0 && (ldb % 8) == 0, "gemm: lda/ldb must be multiples of 8 elements (got %lld, %lld)",
                  lda, ldb);
  UNIVL_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0, "gemm: operands must be 16-byte aligned");
  UNIVL_CHECK_ARG(epilogue >= 0 && epilogue <= 5, "gemm: unknown epilogue %d", epilogue);
  if (epilogue == EPI_GELU_BWD_BF16 || epilogue == EPI_ADD_BF16)
    UNIVL_CHECK_ARG(aux_in != nullptr, "gemm: epilogue %d needs aux_in", epilogue);
  if (epilogue == EPI_BIAS_GELU_BF16) UNIVL_CHECK_ARG(aux_out != nullptr, "gemm: gelu epilogue needs aux_out");
  UNIVL_CHECK_ARG(split_k >= 0, "gemm: bad split_k");
  if (epilogue != EPI_ATOMIC_F32) UNIVL_CHECK_ARG(split_k <= 1, "gemm: split_k>1 needs the atomic epilogue");

  GemmPlan plan;
  if (int prc = plan_gemm(M, N, Kc, epilogue, block_n, split_k, &plan)) return prc;
  const int bn = plan.bn;

  CUtensorMap ta, tb;
  int rc;
  if (!a_mn_major) rc = make_tmap(&ta, A, M, Kc, lda, BLOCK_M);   // [M, Kc], box {64 k, 128 rows}
  else             rc = make_tmap(&ta, A, Kc, M, lda, BLOCK_K);   // [Kc, M], box {64 m, 64 k-rows}
  if (rc) return rc;
  if (!b_mn_major) rc = make_tmap(&tb, B, N, Kc, ldb, bn);
  else             rc = make_tmap(&tb, B, Kc, N, ldb, BLOCK_K);
  if (rc) return rc;

  GemmParams p = gemm_params(M, N, Kc, plan.kb_per, epilogue, alpha, out, ldo, bias, aux_in, ld_aux_in, aux_out,
                             ld_aux_out);
  p.splits = plan.splits;
  p.kb_seg = plan.kb_seg;
  if (plan.splits > 1) {  // the split-K fix-up's slots and arrival counters, one stream-ordered block
    const long long tiles = (long long)((M + BLOCK_M - 1) / BLOCK_M) * ((N + bn - 1) / bn);
    const size_t slot_bytes = (size_t)tiles * plan.splits * BLOCK_M * bn * sizeof(float);
    const size_t counter_bytes = (size_t)tiles * 8 * sizeof(unsigned);
    if ((rc = scratch_alloc((void**)&p.slots, slot_bytes + counter_bytes, stream))) return rc;
    p.arrived = reinterpret_cast<unsigned*>(p.slots + slot_bytes / sizeof(float));
    const cudaError_t e = cudaMemsetAsync(p.arrived, 0, counter_bytes, stream);
    if (e != cudaSuccess) {
      cudaFreeAsync(p.slots, stream);
      return set_error(UNIVL_ERR_CUDA, "gemm split-K counters: %s", cudaGetErrorString(e));
    }
  }

  const bool amn = a_mn_major != 0, bmn = b_mn_major != 0;
  if (bn == 256) rc = dispatch_major<256, 4>(amn, bmn, ta, tb, p, plan.splits, stream);
  else if (bn == 128) rc = dispatch_major<128, 6>(amn, bmn, ta, tb, p, plan.splits, stream);
  else rc = dispatch_major<64, 8>(amn, bmn, ta, tb, p, plan.splits, stream);
  if (p.slots != nullptr) cudaFreeAsync(p.slots, stream);
  return rc;
}

// FP8 GEMM (see gemm_fp8_kernel).  epilogue 0: out bf16 [M, ldo] = acc + bias; 1: out e4m3 [M, ldo] with out_scale
// [N/128, M] = gelu_erf(acc + bias) quantized per (row, 128-column block).
extern "C" int univl_gemm_fp8(const void* A, long long lda, const float* a_scale, const void* B, long long ldb,
                              const float* b_scale, int M, int N, int Kc, int epilogue, const float* bias, void* out,
                              long long ldo, float* out_scale, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UNIVL_CHECK_ARG(M > 0 && N > 0 && Kc > 0, "univl_gemm_fp8: empty problem M=%d N=%d K=%d", M, N, Kc);
  UNIVL_CHECK_ARG(Kc % 128 == 0, "univl_gemm_fp8: K=%d must be a multiple of 128 (one scale per 128 columns)", Kc);
  UNIVL_CHECK_ARG(N % 128 == 0, "univl_gemm_fp8: N=%d must be a multiple of 128 (one scale per 128 x 128 block)", N);
  UNIVL_CHECK_ARG(epilogue == FP8_EPI_BIAS_BF16 || epilogue == FP8_EPI_GELU_E4M3,
                  "univl_gemm_fp8: unknown epilogue %d", epilogue);
  UNIVL_CHECK_ARG(A && B && a_scale && b_scale && bias && out, "univl_gemm_fp8: null operand, scale, bias or output");
  UNIVL_CHECK_ARG(lda >= Kc && ldb >= Kc && (lda % 16) == 0 && (ldb % 16) == 0,
                  "univl_gemm_fp8: lda/ldb must be >= K and multiples of 16 (got %lld, %lld, K=%d)", lda, ldb, Kc);
  UNIVL_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0,
                  "univl_gemm_fp8: A and B must be 16-byte aligned");
  UNIVL_CHECK_ARG(ldo >= N, "univl_gemm_fp8: ldo=%lld must be >= N=%d", ldo, N);
  if (epilogue == FP8_EPI_GELU_E4M3) {
    UNIVL_CHECK_ARG(out_scale != nullptr, "univl_gemm_fp8: the GELU epilogue needs out_scale");
    UNIVL_CHECK_ARG(((uintptr_t)out & 15) == 0 && (ldo % 16) == 0,
                    "univl_gemm_fp8: the e4m3 output must be 16-byte aligned with ldo a multiple of 16 (got %lld)",
                    ldo);
  }

  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap(&ta, A, M, Kc, lda, BLOCK_M, true))) return rc;
  if ((rc = make_tmap(&tb, B, N, Kc, ldb, FP8_BLOCK_N, true))) return rc;

  const GemmParams p = gemm_params(M, N, Kc, Kc / 128, EPI_BIAS_BF16, 1.f, out, ldo, bias, nullptr, 0, nullptr, 0);
  Fp8Params f;
  f.a_scale = a_scale;
  f.b_scale = b_scale;
  f.out_q = reinterpret_cast<uint8_t*>(out);
  f.out_scale = out_scale;
  const bool pairs = (Kc / 128) % 2 == 0;
  if (epilogue == FP8_EPI_BIAS_BF16)
    return pairs ? launch_gemm_fp8<FP8_EPI_BIAS_BF16, true>(ta, tb, p, f, stream)
                 : launch_gemm_fp8<FP8_EPI_BIAS_BF16, false>(ta, tb, p, f, stream);
  return pairs ? launch_gemm_fp8<FP8_EPI_GELU_E4M3, true>(ta, tb, p, f, stream)
               : launch_gemm_fp8<FP8_EPI_GELU_E4M3, false>(ta, tb, p, f, stream);
}

namespace {
// Chunking of the vocabulary cross-entropy: chunks of whole 128-column tiles (at least VX_MIN_CHUNK_TILES of them, so
// that the per-chunk records stay small), no empty chunk, and among those the fewest chunks that give the shortest
// schedule on an H100 SXM's 132 SMs, counted as (rounds of work items) x (tiles per item): 4 chunks of 60 tiles at
// T = 4096 (one round of 128 items), 30 of 8 at T = 17280 (31 rounds).  A pure function of (T, V), never of the SMs in use: the
// chunk order is the lse's summation order.
constexpr int VX_MIN_CHUNK_TILES = 8;
struct VxPlan {
  int m_tiles, n_tiles, chunks, chunk_tiles;
};
VxPlan vx_plan(int T, int V) {
  VxPlan pl;
  pl.m_tiles = (T + BLOCK_M - 1) / BLOCK_M;
  pl.n_tiles = (V + VX_BLOCK_N - 1) / VX_BLOCK_N;
  long long best = -1;
  for (int c = 1; c <= pl.n_tiles; ++c) {
    const int ct = (pl.n_tiles + c - 1) / c;
    if (ct < VX_MIN_CHUNK_TILES && c > 1) break;
    if (c > 1 && ct == (pl.n_tiles + c - 2) / (c - 1)) continue;  // same tiles per chunk as c - 1 chunks
    const int chunks = (pl.n_tiles + ct - 1) / ct;
    const long long rounds = ((long long)pl.m_tiles * chunks + PLAN_SMS - 1) / PLAN_SMS;
    if (best < 0 || rounds * ct < best) {
      best = rounds * ct;
      pl.chunks = chunks;
      pl.chunk_tiles = ct;
    }
  }
  return pl;
}

int vx_check(const char* name, const void* x, long long ldx, const void* w, long long ldw, const long long* labels,
             int T, int V, int Kc, int groups) {
  UNIVL_CHECK_ARG(T > 0 && V > 0 && Kc > 0, "%s: empty problem T=%d V=%d K=%d", name, T, V, Kc);
  UNIVL_CHECK_ARG(x && w && labels, "%s: null x, W or labels", name);
  UNIVL_CHECK_ARG(ldx >= Kc && ldw >= Kc && (ldx % 8) == 0 && (ldw % 8) == 0,
                  "%s: ldx/ldw must be >= K and multiples of 8 (got %lld, %lld, K=%d)", name, ldx, ldw, Kc);
  UNIVL_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)w & 15) == 0, "%s: x and W must be 16-byte aligned", name);
  UNIVL_CHECK_ARG(groups > 0 && T % groups == 0, "%s: %d groups must divide T=%d", name, groups, T);
  return UNIVL_OK;
}

// Runs persistent_prepare first: a runtime call, which also makes the device's primary context current on this thread
// before the driver encodes the tensor maps (autograd runs backward on a thread of its own, where this may be the
// first call of the process into CUDA).
template <int MODE>
int vx_params(const void* x, long long ldx, const void* w, long long ldw, int T, int V, int Kc, CUtensorMap* ta,
              CUtensorMap* tb, VocabXentParams* p) {
  if (int rc = persistent_prepare(vocab_xent_kernel<MODE>, GemmSmem<VX_BLOCK_N, VX_STAGES>::DYN_BYTES, vx_name<MODE>()))
    return rc;
  const VxPlan pl = vx_plan(T, V);
  int rc;
  if ((rc = make_tmap(ta, x, T, Kc, ldx, BLOCK_M))) return rc;
  if ((rc = make_tmap(tb, w, V, Kc, ldw, VX_BLOCK_N))) return rc;
  *p = VocabXentParams{};
  p->T = T; p->V = V; p->Kc = Kc;
  p->m_tiles = pl.m_tiles; p->n_tiles = pl.n_tiles; p->chunks = pl.chunks; p->chunk_tiles = pl.chunk_tiles;
  return UNIVL_OK;
}


// workspace of univl_vocab_xent_fwd: one 16-byte record per row and vocabulary chunk, then one float per row (the row's
// loss term), padded to 16 bytes
long long vx_workspace_bytes(int T, int V) {
  return (long long)T * vx_plan(T, V).chunks * (long long)sizeof(float4) + ((long long)T * 4 + 15) / 16 * 16;
}
}  // namespace

// bytes of workspace univl_vocab_xent_fwd needs for T rows over a V-word vocabulary; negative = error
extern "C" int univl_vocab_xent_workspace(int T, int V) {
  UNIVL_CHECK_ARG(T > 0 && V > 0, "univl_vocab_xent_workspace: empty problem T=%d V=%d", T, V);
  const long long bytes = vx_workspace_bytes(T, V);
  UNIVL_CHECK_ARG(bytes <= 0x7fffffffLL, "univl_vocab_xent_workspace: T=%d V=%d needs over 2 GiB", T, V);
  return (int)bytes;
}

extern "C" int univl_vocab_xent_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                                    const long long* labels, float* lse, float* sum_count, float* loss,
                                    void* workspace, long long workspace_bytes, int T, int V, int Kc, int groups,
                                    void* stream_) {
  const char* name = "univl_vocab_xent_fwd";
  if (int rc = vx_check(name, x, ldx, w, ldw, labels, T, V, Kc, groups)) return rc;
  UNIVL_CHECK_ARG(lse && sum_count && loss && workspace, "%s: null lse, sum_count, loss or workspace", name);
  UNIVL_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "%s: the workspace must be 16-byte aligned", name);
  const long long need = vx_workspace_bytes(T, V);
  UNIVL_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %lld bytes, needs %lld (univl_vocab_xent_workspace)",
                  name, workspace_bytes, need);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CUtensorMap ta, tb;
  VocabXentParams p;
  if (int rc = vx_params<VX_FWD>(x, ldx, w, ldw, T, V, Kc, &ta, &tb, &p)) return rc;
  p.bias = bias;
  p.labels = labels;
  p.part = reinterpret_cast<float4*>(workspace);
  if (int rc = launch_vocab_xent<VX_FWD>(ta, tb, p, stream)) return rc;
  float* nll = reinterpret_cast<float*>(p.part + (long long)T * p.chunks);
  vocab_xent_rows_kernel<<<(T + 255) / 256, 256, 0, stream>>>(p.part, labels, T, V, p.chunks,
                                                               p.chunk_tiles * VX_BLOCK_N, lse, nll);
  vocab_xent_group_kernel<<<groups, VX_GROUP_THREADS, 0, stream>>>(nll, labels, T / groups, sum_count, groups);
  vocab_xent_mean_kernel<<<1, 1, 0, stream>>>(sum_count, groups, loss);
  UNIVL_CHECK_LAUNCH(name);
  return UNIVL_OK;
}

extern "C" int univl_vocab_xent_bwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                                    const long long* labels, const float* lse, const float* sum_count,
                                    const float* gscale, void* dlogits, long long ld_d, int T, int V, int Kc,
                                    int groups, void* stream_) {
  const char* name = "univl_vocab_xent_bwd";
  if (int rc = vx_check(name, x, ldx, w, ldw, labels, T, V, Kc, groups)) return rc;
  UNIVL_CHECK_ARG(lse && sum_count && dlogits, "%s: null lse, sum_count or dlogits", name);
  const long long cols = (long long)vx_plan(T, V).n_tiles * VX_BLOCK_N;
  UNIVL_CHECK_ARG(ld_d >= V && ld_d <= cols && (ld_d % 2) == 0 && ((uintptr_t)dlogits & 3) == 0,
                  "%s: ld_d=%lld must be even, >= V=%d and <= V rounded up to 128, with dlogits 4-byte aligned", name,
                  ld_d, V);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CUtensorMap ta, tb;
  VocabXentParams p;
  if (int rc = vx_params<VX_BWD>(x, ldx, w, ldw, T, V, Kc, &ta, &tb, &p)) return rc;
  p.bias = bias;
  p.labels = labels;
  p.lse = lse;
  p.count = sum_count + groups;
  p.gscale = gscale;
  p.rows_per_group = T / groups;
  p.groups = groups;
  p.dl = reinterpret_cast<bf16*>(dlogits);
  p.ld_d = ld_d;
  return launch_vocab_xent<VX_BWD>(ta, tb, p, stream);
}

namespace {
// workspace of univl_vocab_beam_topk: the lse pass's 16-byte record per row and chunk, then the selection pass's
// VX_BEAM_MAX 8-byte candidates per row and chunk
long long vb_workspace_bytes(int R, int V) {
  return (long long)R * vx_plan(R, V).chunks * (long long)(sizeof(float4) + VX_BEAM_MAX * sizeof(int2));
}
}  // namespace

extern "C" int univl_vocab_beam_topk_workspace(int n_inst, int n_beam, int V) {
  UNIVL_CHECK_ARG(n_inst > 0 && V > 0 && n_beam >= 1 && n_beam <= VX_BEAM_MAX,
                  "univl_vocab_beam_topk_workspace: n_inst=%d V=%d n_beam=%d (1 <= n_beam <= %d)", n_inst, V, n_beam,
                  VX_BEAM_MAX);
  const long long bytes = vb_workspace_bytes(n_inst * n_beam, V);
  UNIVL_CHECK_ARG(bytes <= 0x7fffffffLL, "univl_vocab_beam_topk_workspace: n_inst=%d V=%d needs over 2 GiB", n_inst, V);
  return (int)bytes;
}

extern "C" int univl_vocab_beam_topk(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                                     const float* score, const int* n_live, int n_inst, int n_beam, int V, int Kc,
                                     float* lse, float* out_key, int* out_index, void* workspace,
                                     long long workspace_bytes, void* stream_) {
  const char* name = "univl_vocab_beam_topk";
  UNIVL_CHECK_ARG(n_beam >= 1 && n_beam <= VX_BEAM_MAX, "%s: n_beam=%d outside [1, %d]", name, n_beam, VX_BEAM_MAX);
  UNIVL_CHECK_ARG(n_inst > 0 && Kc > 0 && V >= n_beam && (long long)n_beam * V <= 0x7fffffffLL,
                  "%s: n_inst=%d K=%d V=%d (n_beam <= V, n_beam V < 2^31)", name, n_inst, Kc, V);
  UNIVL_CHECK_ARG(x && w && score && n_live && lse && out_key && out_index && workspace,
                  "%s: null x, W, score, n_live, lse, out_key, out_index or workspace", name);
  UNIVL_CHECK_ARG(ldx >= Kc && ldw >= Kc && (ldx % 8) == 0 && (ldw % 8) == 0,
                  "%s: ldx/ldw must be >= K and multiples of 8 (got %lld, %lld, K=%d)", name, ldx, ldw, Kc);
  UNIVL_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)w & 15) == 0 && ((uintptr_t)workspace & 15) == 0,
                  "%s: x, W and the workspace must be 16-byte aligned", name);
  const int R = n_inst * n_beam;
  const long long need = vb_workspace_bytes(R, V);
  UNIVL_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %lld bytes, needs %lld (univl_vocab_beam_topk_workspace)",
                  name, workspace_bytes, need);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CUtensorMap ta, tb;
  VocabXentParams p;
  // pass 1: every row's lse, folded as the cross-entropy forward folds it
  if (int rc = vx_params<VX_FWD>(x, ldx, w, ldw, R, V, Kc, &ta, &tb, &p)) return rc;
  p.bias = bias;
  p.part = reinterpret_cast<float4*>(workspace);
  if (int rc = launch_vocab_xent<VX_FWD>(ta, tb, p, stream)) return rc;
  vocab_xent_rows_kernel<<<(R + 255) / 256, 256, 0, stream>>>(p.part, nullptr, R, V, p.chunks,
                                                               p.chunk_tiles * VX_BLOCK_N, lse, nullptr);
  UNIVL_CHECK_LAUNCH(name);
  // pass 2: the logits again, each row's best keys per chunk, then each instance's top n_beam
  float4* part = p.part;
  if (int rc = vx_params<VX_BEAM>(x, ldx, w, ldw, R, V, Kc, &ta, &tb, &p)) return rc;
  p.bias = bias;
  p.lse = lse;
  p.score = score;
  p.cand = reinterpret_cast<int2*>(part + (long long)R * p.chunks);
  if (int rc = launch_vocab_xent<VX_BEAM>(ta, tb, p, stream)) return rc;
  vocab_beam_merge_kernel<<<n_inst, VB_MERGE_THREADS, 0, stream>>>(p.cand, n_live, n_beam, p.chunks, V, out_key,
                                                                   out_index);
  UNIVL_CHECK_LAUNCH(name);
  return UNIVL_OK;
}

extern "C" int univl_beam_advance(const float* key, const int* index, int n_inst, int n_beam, int V, int t,
                                  int max_words, long long eos, float* score, int* done, int* prev_k, int* word,
                                  long long* tokens, const int* anc_in, int* anc_out, void* stream_) {
  const char* name = "univl_beam_advance";
  UNIVL_CHECK_ARG(n_beam >= 1 && n_beam <= VX_BEAM_MAX, "%s: n_beam=%d outside [1, %d]", name, n_beam, VX_BEAM_MAX);
  UNIVL_CHECK_ARG(n_inst > 0 && V > 0 && t >= 0 && t < max_words, "%s: n_inst=%d V=%d t=%d max_words=%d", name, n_inst,
                  V, t, max_words);
  UNIVL_CHECK_ARG((long long)max_words * n_inst * n_beam <= 0x7fffffffLL, "%s: max_words x rows must be < 2^31", name);
  UNIVL_CHECK_ARG(key && index && score && done && prev_k && word && tokens && anc_in && anc_out && anc_in != anc_out,
                  "%s: null pointer, or anc_in == anc_out", name);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  beam_advance_kernel<<<n_inst, 128, 0, stream>>>(key, index, n_beam, V, t, eos, score, done, prev_k, word,
                                                  tokens, anc_in, anc_out, max_words);
  UNIVL_CHECK_LAUNCH(name);
  return UNIVL_OK;
}
