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
// Structure (per CTA, 384 threads, 128 x BLOCK_N output tiles, optional split-K):
//   warpgroup 0      TMA producer : one thread streams 2D boxes (128B swizzle) into a STAGES-deep mbarrier ring
//   warpgroups 1, 2  consumers    : each owns 64 rows of the tile, issues m64 x BLOCK_N x k16 wgmma on the shared stage
//                                   and runs the fused epilogue straight from its accumulator registers
// grid = min(#work items, #SMs); each CTA walks work items round-robin in the order decode_work() defines, and the
// producer's ring runs continuously across tiles, so the next tile's operands load while the epilogue runs.
#include "common.cuh"
#include "tmap.cuh"
#include "wgmma.cuh"

#include <stdio.h>

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
  float* part;  // EPI_ATOMIC_F32 with split-K: [splits][M][N] partial sums, else null
};

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int PLAN_SMS = 132;  // H100 SXM: the tile-width / split-K plan is a pure function of the problem

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

// fused epilogue of the accumulator values of columns (col, col + 1) of one row; col is even.  split: the work item's
// split-K index
__device__ __forceinline__ void epi_pair(const GemmParams& p, int split, int row, int col, float v0, float v1) {
  if (row >= p.M || col >= p.N) return;
  const bool two = col + 1 < p.N;
  const bool vec = two && p.vec2;
  const int epi = p.epilogue;
  v0 *= p.alpha;
  v1 *= p.alpha;
  if (p.bias != nullptr && (epi == EPI_BIAS_BF16 || epi == EPI_BIAS_GELU_BF16 || epi == EPI_BIAS_F32)) {
    v0 += __ldg(p.bias + col);
    if (two) v1 += __ldg(p.bias + col + 1);
  }
  if (epi == EPI_ATOMIC_F32 && p.part != nullptr) {  // this split's partial sums (partials_reduce adds them in order)
    float* o = p.part + ((long long)split * p.M + row) * p.N + col;
    if (two && (p.N & 1) == 0) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
    else {
      o[0] = v0;
      if (two) o[1] = v1;
    }
    return;
  }
  if (epi == EPI_ATOMIC_F32 || epi == EPI_BIAS_F32) {
    float* o = reinterpret_cast<float*>(p.out) + (long long)row * p.ldo + col;
    if (epi == EPI_ATOMIC_F32) {  // one split: this thread is the element's only writer in the launch
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

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const GemmParams p, const int num_work) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int total_kb = (p.Kc + BLOCK_K - 1) / BLOCK_K;
  const int kb_per = p.k_blocks_per_split;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; global memory is touched only from here on

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
        const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, kb_per, BLOCK_N);
        for (int i = 0; i < wi.num_kb; ++i, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], L::STAGE_BYTES);
          const int k_elem = (wi.kb_begin + i) * BLOCK_K;
          if (!A_MN) {
            tma_load_2d(sa, &tmap_a, &full_bar[s], k_elem, wi.m0);  // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c)  // box {64 m, 64 k-rows}
              tma_load_2d(sa + c * (BLOCK_K * 128), &tmap_a, &full_bar[s], wi.m0 + c * 64, k_elem);
          }
          if (!B_MN) {
            tma_load_2d(sb, &tmap_b, &full_bar[s], k_elem, wi.n0);  // box {64 k, BLOCK_N rows}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_N / 64; ++c)
              tma_load_2d(sb + c * (BLOCK_K * 128), &tmap_b, &full_bar[s], wi.n0 + c * 64, k_elem);
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers ------------------------------
    regs_alloc<232>();
    const int c = wg - 1;  // rows [64 c, 64 c + 64) of every tile
    const int t = threadIdx.x & 127;
    const int warp = t >> 5, lane = t & 31;
    uint32_t it = 0;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
      const WorkItem wi = decode_work(w, m_tiles, n_tiles, total_kb, kb_per, BLOCK_N);
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int e = 0; e < BLOCK_N / 2; ++e) acc[e] = 0.f;
      int prev_s = -1;
      for (int i = 0; i < wi.num_kb; ++i, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        // this warpgroup's 64 rows of A start 8 KB into the stage in both layouts (64 rows x 128 B K-major, or the
        // second 64-wide MN block); a k16 step is +32 B K-major, +16 rows of 128 B MN-major
        const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES) + c * (64 * 128);
        const uint32_t sb = smem_u32(smem + s * L::STAGE_BYTES) + L::A_BYTES;
        wgmma_fence();
        fence_regs(acc);
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          const uint64_t da = A_MN ? make_smem_desc_sw128(sa + k * 2048, BLOCK_K * 128, 1024)
                                   : make_smem_desc_sw128(sa + k * 32, 16, 1024);
          const uint64_t db = B_MN ? make_smem_desc_sw128(sb + k * 2048, BLOCK_K * 128, 1024)
                                   : make_smem_desc_sw128(sb + k * 32, 16, 1024);
          WgmmaSS<BLOCK_N>::template mma<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (i > 0 || k > 0) ? 1 : 0);
        }
        wgmma_commit();
        fence_regs(acc);
        wgmma_wait<1>();  // the previous k-block's MMAs have read their stage
        if (prev_s >= 0 && t == 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (t == 0) mbar_arrive(&empty_bar[prev_s]);
      // accumulator fragment: warp w holds rows 16 w + lane / 4 (+ 8); register 4 j + {0, 1} (+ {2, 3} for row + 8) are
      // columns 8 j + 2 (lane % 4) + {0, 1}
      const int row = wi.m0 + c * 64 + warp * 16 + (lane >> 2);
      const int col0 = wi.n0 + 2 * (lane & 3);
      const int split = wi.kb_begin / kb_per;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        if (wi.n0 + j * 8 >= p.N) break;  // warp-uniform
        epi_pair(p, split, row, col0 + j * 8, acc[4 * j], acc[4 * j + 1]);
        epi_pair(p, split, row + 8, col0 + j * 8, acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
}

template <int BLOCK_N, int STAGES, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int splits,
                       cudaStream_t stream) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  auto kern = gemm_wgmma_kernel<BLOCK_N, STAGES, A_MN, B_MN>;
  // per launch: the attribute is per device and callers may drive several devices from one process
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "gemm smem attribute: %s", cudaGetErrorString(e));
  const int sms = usable_sms();
  const long long work =
      (long long)((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N) * (long long)splits;
  if (work > 0x7fffffffLL) return set_error(UNIVL_ERR_ARG, "gemm: too many tiles");
  const int grid = (int)(work < sms ? work : sms);
  e = launch_kernel(kern, dim3(grid), dim3(GEMM_THREADS), (size_t)L::DYN_BYTES, stream, ta, tb, p, (int)work);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "gemm launch: %s", cudaGetErrorString(e));
  UNIVL_CHECK_LAUNCH("gemm_wgmma");
  return UNIVL_OK;
}

template <int BLOCK_N, int STAGES>
static int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          int splits, cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch_gemm<BLOCK_N, STAGES, false, false>(ta, tb, p, splits, stream);
  if (!a_mn && b_mn) return launch_gemm<BLOCK_N, STAGES, false, true>(ta, tb, p, splits, stream);
  if (a_mn && b_mn) return launch_gemm<BLOCK_N, STAGES, true, true>(ta, tb, p, splits, stream);
  return launch_gemm<BLOCK_N, STAGES, true, false>(ta, tb, p, splits, stream);
}

}  // namespace univl

using namespace univl;

namespace {
struct GemmPlan {
  int bn, splits, kb_per;
};
// tile width and split-K factor for a problem — a pure function of the arguments, shared by the launcher and by
// univl_gemm_plan
int plan_gemm(int M, int N, int Kc, int epilogue, int block_n, int split_k, GemmPlan* plan) {
  const int total_kb = (Kc + BLOCK_K - 1) / BLOCK_K;
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  int bn = block_n;
  if (bn == 0) {
    bn = 256;
    // without split-K the tile count alone must fill the SMs; with the atomic epilogue split-K supplies the
    // parallelism, so keep the widest (most operand-bandwidth-efficient) tile
    if (epilogue != EPI_ATOMIC_F32)
      while (bn > 64 && (long long)m_tiles * ((N + bn - 1) / bn) < PLAN_SMS) bn >>= 1;
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
  const int kb_per = (total_kb + splits - 1) / splits;
  splits = (total_kb + kb_per - 1) / kb_per;  // no empty split
  plan->bn = bn; plan->splits = splits; plan->kb_per = kb_per;
  return UNIVL_OK;
}
}  // namespace

// Which kernel univl_gemm_bf16 launches for this problem: 1 = the persistent wgmma kernel (the only one); negative =
// error.  Stateless (a function of its arguments): bench.py uses it to attribute per-launch CUDA-event times.
extern "C" int univl_gemm_plan(int M, int N, int Kc, int epilogue, int block_n, int split_k) {
  GemmPlan plan;
  if (int rc = plan_gemm(M, N, Kc, epilogue, block_n, split_k, &plan)) return rc;
  return 1;
}

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

  GemmParams p;
  p.M = M; p.N = N; p.Kc = Kc;
  p.k_blocks_per_split = plan.kb_per;
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
  p.part = nullptr;
  if (plan.splits > 1)
    if ((rc = scratch_alloc((void**)&p.part, (size_t)plan.splits * M * N * sizeof(float), stream))) return rc;

  const bool amn = a_mn_major != 0, bmn = b_mn_major != 0;
  if (bn == 256) rc = dispatch_major<256, 4>(amn, bmn, ta, tb, p, plan.splits, stream);
  else if (bn == 128) rc = dispatch_major<128, 6>(amn, bmn, ta, tb, p, plan.splits, stream);
  else rc = dispatch_major<64, 8>(amn, bmn, ta, tb, p, plan.splits, stream);
  if (rc != UNIVL_OK || p.part == nullptr) return rc;
  return partials_reduce(p.part, plan.splits, M, N, reinterpret_cast<float*>(out), ldo, stream);
}
