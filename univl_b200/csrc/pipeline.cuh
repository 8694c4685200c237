// univl_b200 — the pipeline skeleton of the warp-specialised wgmma kernels (GEMM, FP8 GEMM, vocabulary
// cross-entropy, fused attention forward and backward).
//
// A CTA of 384 threads: warpgroup 0 is the producer, whose one TMA thread streams operand boxes into a STAGES-deep
// ring of shared-memory stages, and warpgroups 1 and 2 are the consumers, which issue wgmma on each stage and hand it
// back.  Each stage has two mbarriers: `full` (one arrival, the producer's expect_tx, completed by the TMA bytes) and
// `empty` (one arrival per consumer warpgroup that reads the stage).  Producer and consumers walk the same sequence of
// ring positions, it = 0, 1, 2, ...: position it is stage it % STAGES in phase (it / STAGES) & 1.  A kernel is
//   prologue    kernel_prologue: barriers, tensor-map prefetch, the wait for the previous kernel
//   producer    producer_regs(), then Ring::acquire per stage and the TMA loads into it
//   consumers   consumer_regs(), then Ring::wait per stage, the MMAs and Ring::release behind wgmma_wait<1>
// and its host launcher runs persistent_prepare + persistent_launch: grid = min(work items, usable SMs).
#pragma once

#include "common.cuh"
#include "wgmma.cuh"

namespace univl {

constexpr int PIPELINE_THREADS = 384;  // producer warpgroup + two consumer warpgroups

template <int STAGES>
struct Ring {
  uint64_t* full;   // [STAGES]
  uint64_t* empty;  // [STAGES]

  __device__ __forceinline__ static int stage(uint32_t it) { return it % STAGES; }

  __device__ __forceinline__ void init(uint32_t consumer_arrivals) const {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], consumer_arrivals);
    }
    fence_mbar_init();
  }
  // producer: waits until the consumers have released position it's stage (parity flipped: the first pass over the
  // ring finds every stage free), arms its full barrier for tx_bytes of TMA loads and returns the stage
  __device__ __forceinline__ int acquire(uint32_t it, uint32_t tx_bytes) const {
    const int s = stage(it);
    mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&full[s], tx_bytes);
    return s;
  }
  // consumer: waits until position it's loads have landed and returns the stage.  A parity wait cannot tell phases
  // two apart: a wait issued more than one phase ahead of the barrier matches the phase before, which has already
  // completed, and reads the stage before its load lands.  So no consumer may wait on position it + STAGES before
  // every wait on position it has passed — each consumer's own waits are in order, and consumers that split the
  // positions between them (the GEMM's ping-pong schedule) must take turns.
  __device__ __forceinline__ int wait(uint32_t it) const {
    const int s = stage(it);
    mbar_wait(&full[s], (it / STAGES) & 1);
    return s;
  }
  // consumer: one warpgroup's arrival (call from one thread) — it no longer reads the stage
  __device__ __forceinline__ void release(int s) const { mbar_arrive(&empty[s]); }
};

// Kernel prologue: lets the next kernel launch (PDL), aligns dynamic shared memory to 1024 bytes (the 128B swizzle),
// sets up the ring whose barriers lie at bar_offset from that base, prefetches the tensor maps (m2 may be null) and
// waits for the previous kernel.  Returns the aligned base.  Everything before pdl_wait() overlaps the previous
// kernel's tail, so nothing here touches global memory before it.
template <int STAGES>
__device__ __forceinline__ uint8_t* kernel_prologue(Ring<STAGES>& ring, int bar_offset, uint32_t consumer_arrivals,
                                                    const CUtensorMap* m0, const CUtensorMap* m1,
                                                    const CUtensorMap* m2 = nullptr) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  ring.full = reinterpret_cast<uint64_t*>(smem + bar_offset);
  ring.empty = ring.full + STAGES;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(m0);
    tma_prefetch_desc(m1);
    if (m2 != nullptr) tma_prefetch_desc(m2);
    ring.init(consumer_arrivals);
  }
  __syncthreads();
  pdl_wait();
  return smem;
}

// register budgets of the warp roles: the producer warpgroup gives its registers to the two consumer warpgroups.
// producer_regs() returns true on the producer's one TMA thread.
__device__ __forceinline__ bool producer_regs() {
  regs_dealloc<40>();
  return threadIdx.x == 0;
}
__device__ __forceinline__ void consumer_regs() { regs_alloc<232>(); }

// bf16 k-block mainloop of one consumer warpgroup: issues k-blocks [i0, i1) at ring positions it, it + 1, ... (it
// advances past them) into HALVES accumulator blocks of 64 rows x N.  A stage holds A (128 rows x 128 B of K) at its
// start and B at B_OFFSET; accumulator block h reads A rows from byte a_off + h * 8 KB, the 64-row offset in both
// operand layouts (64 rows x 128 B K-major, or the second 64-wide MN block).  Per k-block: four k16 wgmmas (a k16 step
// is +32 B K-major, +16 rows of 128 B MN-major), commit, and wgmma_wait<1>, after which the previous k-block's MMAs
// have read their stage and `leader` (one thread of the warpgroup) releases it.  The MMAs restart from zero at i0.
// Returns the last k-block's stage, which mma_drain releases.
template <int N, int HALVES, bool A_MN, bool B_MN, int STAGE_BYTES, int B_OFFSET, int STAGES>
__device__ __forceinline__ int mma_kblocks(const Ring<STAGES>& ring, uint8_t* smem, uint32_t a_off,
                                           float (&acc)[HALVES][N / 2], int i0, int i1, uint32_t& it, bool leader) {
  int prev_s = -1;
  for (int i = i0; i < i1; ++i, ++it) {
    const int s = ring.wait(it);
    const uint32_t sa = smem_u32(smem + s * STAGE_BYTES) + a_off;
    const uint32_t sb = smem_u32(smem + s * STAGE_BYTES) + B_OFFSET;
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < HALVES; ++h) fence_regs(acc[h]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t db = B_MN ? make_smem_desc_sw128(sb + k * 2048, 64 * 128, 1024)
                               : make_smem_desc_sw128(sb + k * 32, 16, 1024);
#pragma unroll
      for (int h = 0; h < HALVES; ++h) {
        const uint32_t sah = sa + h * (64 * 128);
        const uint64_t da = A_MN ? make_smem_desc_sw128(sah + k * 2048, 64 * 128, 1024)
                                 : make_smem_desc_sw128(sah + k * 32, 16, 1024);
        WgmmaSS<N>::template mma<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[h], da, db, (i > i0 || k > 0) ? 1 : 0);
      }
    }
    wgmma_commit();
#pragma unroll
    for (int h = 0; h < HALVES; ++h) fence_regs(acc[h]);
    wgmma_wait<1>();
    if (prev_s >= 0 && leader) ring.release(prev_s);
    prev_s = s;
  }
  return prev_s;
}
// one 64-row accumulator block
template <int N, bool A_MN, bool B_MN, int STAGE_BYTES, int B_OFFSET, int STAGES>
__device__ __forceinline__ int mma_kblocks(const Ring<STAGES>& ring, uint8_t* smem, uint32_t a_off,
                                           float (&acc)[N / 2], int i0, int i1, uint32_t& it, bool leader) {
  return mma_kblocks<N, 1, A_MN, B_MN, STAGE_BYTES, B_OFFSET>(ring, smem, a_off,
                                                             reinterpret_cast<float (&)[1][N / 2]>(acc), i0, i1, it,
                                                             leader);
}

// the end of a mainloop: waits for its last MMAs and releases their stage
template <int HALVES, int R, int STAGES>
__device__ __forceinline__ void mma_drain(const Ring<STAGES>& ring, int last_s, float (&acc)[HALVES][R], bool leader) {
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < HALVES; ++h) fence_regs(acc[h]);
  if (leader) ring.release(last_s);
}
template <int R, int STAGES>
__device__ __forceinline__ void mma_drain(const Ring<STAGES>& ring, int last_s, float (&acc)[R], bool leader) {
  mma_drain(ring, last_s, reinterpret_cast<float (&)[1][R]>(acc), leader);
}

// Host side of a persistent kernel, in two steps.  persistent_prepare sets the kernel's dynamic shared-memory size: on
// every launch, since the attribute is per device and callers may drive several devices from one process.  It is
// also a runtime call that makes the device's primary context current on the calling thread, which a launcher that
// encodes tensor maps from a thread of its own (autograd's backward) needs first.  persistent_launch then runs
// grid = min(items, usable SMs) CTAs of PIPELINE_THREADS; each walks its share of the items.  `name`: the entry point,
// for the error messages.
template <typename Kern>
static int persistent_prepare(Kern kern, int smem_bytes, const char* name) {
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "%s smem attribute: %s", name, cudaGetErrorString(e));
  return UNIVL_OK;
}
template <typename Kern, typename... Args>
static int persistent_launch(Kern kern, const char* name, long long items, int smem_bytes, cudaStream_t stream,
                             Args... args) {
  if (items > 0x7fffffffLL) return set_error(UNIVL_ERR_ARG, "%s: too many work items", name);
  const int sms = usable_sms();
  const int grid = (int)(items < sms ? items : sms);
  const cudaError_t e = launch_kernel(kern, dim3(grid), dim3(PIPELINE_THREADS), (size_t)smem_bytes, stream, args...);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "%s launch: %s", name, cudaGetErrorString(e));
  UNIVL_CHECK_LAUNCH(name);
  return UNIVL_OK;
}

}  // namespace univl
