// univl_b200 — exact streaming top-k of the mean-pooled text x video similarity (retrieval shortlists).
//
// For each text row i, the k videos j with the largest sim[i, j] = t[i, :] . v[j, :], in one strict total order: score
// descending, then video index ascending.  The [Nt, Nv] matrix is never written.
//
// Scores.  Every score has the bits loss.cu's sim_fwd_kernel gives the same entry, so a shortlist agrees exactly with
// the similarity matrix a caller would otherwise rank (UniVL._mean_pool_similarity).  That kernel's lane l forms the
// partial acc_l = fma(t[c], v[c], acc_l) over c = l, l + 32, ... in increasing c, and warp_sum combines the 32
// partials with a butterfly (xor 16, 8, 4, 2, 1).  Here lane l of a warp forms the same partial acc_l for each of the
// warp's 8 x 8 entries, with its t and v columns staged in shared memory, so each loaded value feeds 8 FMAs instead of
// one.  The 64 partial sets are then combined by a reduce-scatter over the same xor distances in the same order: at
// distance o a lane keeps half of its entries and adds the partner's copy of them, which is the sum the butterfly forms
// at that step (fp32 addition is commutative), so each entry ends with the butterfly's bits.  Tensor cores would sum in
// another order, so the values stay on the FMA pipe.
//
// Ranking.  A CTA owns BT text rows and a contiguous share of the gallery, which it streams in tiles of BV videos in
// increasing index order, keeping a sorted running top-k per text row in shared memory.  A candidate enters when it beats
// the current k-th entry; since every listed entry has a lower index, an equal score never does.  When the gallery is
// split over several CTAs (to fill the GPU when there are few text rows), each writes its sorted list to stream-ordered
// scratch, and a merge kernel folds the lists in split order by rank (each element's position in the merged list is its
// own index plus the number of elements of the other list ranked above it).  The order is a strict total order, so the
// result does not depend on the tiling or the split: every launch writes the same bits.  No floating-point atomics.
//
// Ground-truth ranks.  sim_best_positive_kernel scores each query's positives with sim_dot (sim_fwd_kernel's own dot
// product); sim_rank_kernel runs the same scoring engine as sim_topk_kernel and counts, per tile, the videos that rank
// above that best positive with one ballot per row instead of keeping a list.
#include <climits>

#include "common.cuh"

namespace univl {

constexpr int TK_BT = 16;       // text rows per CTA
constexpr int TK_BV = 32;       // videos per gallery tile (one candidate per lane when ranking)
constexpr int TK_KC = 128;      // columns per staged chunk of a video tile
constexpr int TK_THREADS = 256; // 8 warps: 2 (text halves of 8 rows) x 4 (video quarters of 8)
constexpr int TK_MAX_K = 256;

__device__ __forceinline__ void tk_cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void tk_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tk_cp_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// key order of the ranking: (s1, i1) ranks above (s2, i2)
__device__ __forceinline__ bool tk_above(float s1, int i1, float s2, int i2) {
  return s1 > s2 || (s1 == s2 && i1 < i2);
}

// one reduce-scatter step over xor distance O on N values per lane: the lanes with bit O set keep the upper half
template <int N, int O>
__device__ __forceinline__ void tk_reduce_step(float (&r)[64], int lane) {
  constexpr int HALF = N / 2;
  const bool up = (lane & O) != 0;
#pragma unroll
  for (int e = 0; e < HALF; ++e) {
    const float send = up ? r[e] : r[e + HALF];
    const float keep = up ? r[e + HALF] : r[e];
    r[e] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}

// Shared memory of the scoring engine, in floats: sT [BT][Hp] (zero beyond H and past Nt), sV [2][BV][KC], sS [BT][BV]
__host__ __device__ constexpr int tk_engine_floats(int Hp) { return TK_BT * Hp + 2 * TK_BV * TK_KC + TK_BT * TK_BV; }

// The scoring engine of sim_topk_kernel and sim_rank_kernel.  The CTA stages text rows [row0, row0 + BT) in smem and
// streams videos [vbeg, vend) through it in tiles of BV, in increasing index order.  After each tile it calls
// on_tile(sS, j0) with every thread of the CTA: sS[r * BV + c] is the score of text row row0 + r against video j0 + c,
// with the bits of sim_dot, for j0 + c < vend (entries past vend are not scores).  sS is only read inside the call.
template <class OnTile>
__device__ __forceinline__ void tk_score_tiles(const float* __restrict__ t, const float* __restrict__ v, int Nt, int H,
                                               int Hp, int row0, int vbeg, int vend, float* smem, OnTile&& on_tile) {
  float* sT = smem;
  float* sV = sT + TK_BT * Hp;
  float* sS = sV + 2 * TK_BV * TK_KC;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wt = warp & 1, wv = warp >> 1;
  const int nch = Hp / TK_KC;
  const int ntile = vend > vbeg ? (vend - vbeg + TK_BV - 1) / TK_BV : 0;
  const int steps = ntile * nch;

  for (int idx = tid; idx < TK_BT * (Hp / 4); idx += TK_THREADS) {
    const int r = idx / (Hp / 4), c = (idx - r * (Hp / 4)) * 4;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < Nt && c < H) x = *reinterpret_cast<const float4*>(t + (long long)(row0 + r) * H + c);
    *reinterpret_cast<float4*>(sT + r * Hp + c) = x;
  }
  // step s = (tile s / nch, chunk s % nch) into stage s & 1
  auto load = [&](int s) {
    const int tile = s / nch, ch = s - tile * nch;
    float* dst = sV + (s & 1) * TK_BV * TK_KC;
    for (int idx = tid; idx < TK_BV * (TK_KC / 4); idx += TK_THREADS) {
      const int r = idx / (TK_KC / 4), c = (idx - r * (TK_KC / 4)) * 4;
      const int j = vbeg + tile * TK_BV + r, col = ch * TK_KC + c;
      if (j < vend && col < H) tk_cp_async16(dst + r * TK_KC + c, v + (long long)j * H + col);
      else *reinterpret_cast<float4*>(dst + r * TK_KC + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };

  float acc[64];
  if (steps > 0) load(0);
  tk_cp_commit();
  for (int s = 0; s < steps; ++s) {
    if (s + 1 < steps) load(s + 1);
    tk_cp_commit();
    tk_cp_wait1();
    __syncthreads();
    const int tile = s / nch, ch = s - tile * nch;
    if (ch == 0) {
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.f;
    }
    const float* tb = sT + (wt * 8) * Hp + ch * TK_KC + lane;
    const float* vb = sV + (s & 1) * TK_BV * TK_KC + (wv * 8) * TK_KC + lane;
#pragma unroll
    for (int m = 0; m < TK_KC / 32; ++m) {
      if (ch * TK_KC + m * 32 + lane < H) {  // columns past H add nothing (not even a signed zero)
        float tv[8], vv[8];
#pragma unroll
        for (int a = 0; a < 8; ++a) tv[a] = tb[a * Hp + m * 32];
#pragma unroll
        for (int b = 0; b < 8; ++b) vv[b] = vb[b * TK_KC + m * 32];
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
          for (int b = 0; b < 8; ++b) acc[a * 8 + b] = fmaf(tv[a], vv[b], acc[a * 8 + b]);
      }
    }
    if (ch == nch - 1) {
      tk_reduce_step<64, 16>(acc, lane);
      tk_reduce_step<32, 8>(acc, lane);
      tk_reduce_step<16, 4>(acc, lane);
      tk_reduce_step<8, 2>(acc, lane);
      tk_reduce_step<4, 1>(acc, lane);
      // lane holds entries 2 lane and 2 lane + 1 of the warp's 8 x 8 (entry e = 8 a + b): the step at distance o
      // kept the upper half, 2 o entries further on, in the lanes with bit o set
      const int e0 = 2 * lane;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int e = e0 + q;
        sS[(wt * 8 + (e >> 3)) * TK_BV + wv * 8 + (e & 7)] = acc[q];
      }
      __syncthreads();
      on_tile(static_cast<const float*>(sS), vbeg + tile * TK_BV);
    }
    __syncthreads();
  }
}

// Grid (ceil(Nt / BT), splits); CTA (x, y) ranks text rows [x BT, x BT + BT) against videos [y per, min(Nv, y per + per)).
// out_s / out_i: [splits][Nt][k] (the final [Nt, k] when splits == 1); a split with fewer than k videos pads its list
// with (-inf, INT_MAX), which ranks below every video.
__global__ void __launch_bounds__(TK_THREADS)
sim_topk_kernel(const float* __restrict__ t, const float* __restrict__ v, int Nt, int Nv, int H, int Hp, int k, int per,
                float* __restrict__ out_s, int* __restrict__ out_i) {
  extern __shared__ __align__(16) float tk_smem[];
  float* lsc = tk_smem + tk_engine_floats(Hp);  // [BT][k] running lists, sorted
  int* lid = reinterpret_cast<int*>(lsc + TK_BT * k);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * TK_BT;
  const int vbeg = blockIdx.y * per, vend = min(Nv, vbeg + per);

  int cnt0 = 0, cnt1 = 0;  // listed entries of this warp's rows 2 warp and 2 warp + 1
  tk_score_tiles(t, v, Nt, H, Hp, row0, vbeg, vend, tk_smem, [&](const float* sS, int j0) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = warp * 2 + rr;
      int cnt = rr ? cnt1 : cnt0;
      float* ls = lsc + r * k;
      int* li = lid + r * k;
      const float sc = sS[r * TK_BV + lane];
      const bool enter = j0 + lane < vend && (cnt < k || sc > ls[k - 1]);
      unsigned m = __ballot_sync(0xffffffffu, enter);
      while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const float cs = __shfl_sync(0xffffffffu, sc, src);
        // every listed entry has a lower index: it ranks above the candidate iff its score is >= cs
        int pos = 0;
        for (int q = lane; q < cnt; q += 32) pos += ls[q] >= cs ? 1 : 0;
        pos = __reduce_add_sync(0xffffffffu, pos);
        if (pos >= k) continue;
        const int last = min(cnt, k - 1);  // entries [pos, last) move down by one, from the tail
        for (int base = last - 1; base >= pos; base -= 32) {
          const int q = base - lane;
          float ms = 0.f;
          int mi = 0;
          if (q >= pos) { ms = ls[q]; mi = li[q]; }
          __syncwarp();
          if (q >= pos) { ls[q + 1] = ms; li[q + 1] = mi; }
          __syncwarp();
        }
        if (lane == 0) { ls[pos] = cs; li[pos] = j0 + src; }
        __syncwarp();
        cnt = min(cnt + 1, k);
      }
      if (rr) cnt1 = cnt; else cnt0 = cnt;
    }
  });

  const long long ob = (long long)blockIdx.y * Nt;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = warp * 2 + rr, row = row0 + r;
    const int cnt = rr ? cnt1 : cnt0;
    if (row >= Nt) continue;
    for (int q = lane; q < k; q += 32) {
      out_s[(ob + row) * k + q] = q < cnt ? lsc[r * k + q] : -INFINITY;
      out_i[(ob + row) * k + q] = q < cnt ? lid[r * k + q] : INT_MAX;
    }
  }
}

// Grid and CTA as sim_topk_kernel: CTA (x, y) adds to rank[row] (zeroed beforehand), for each of its query rows, the
// number of its videos that rank above the row's (best_s, best_i).  A tile is counted with one ballot per row, so
// nothing is listed; the splits' counts are integers, so the order of their atomic adds does not change the result.
__global__ void __launch_bounds__(TK_THREADS)
sim_rank_kernel(const float* __restrict__ t, const float* __restrict__ v, int Nt, int Nv, int H, int Hp, int per,
                const float* __restrict__ best_s, const int* __restrict__ best_i,
                unsigned long long* __restrict__ rank) {
  extern __shared__ __align__(16) float tk_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * TK_BT;
  const int vbeg = blockIdx.y * per, vend = min(Nv, vbeg + per);

  float bs[2];
  int bi[2];
  unsigned cnt[2] = {0u, 0u};
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int row = row0 + warp * 2 + rr;
    bs[rr] = row < Nt ? best_s[row] : 0.f;
    bi[rr] = row < Nt ? best_i[row] : 0;
  }
  tk_score_tiles(t, v, Nt, H, Hp, row0, vbeg, vend, tk_smem, [&](const float* sS, int j0) {
    const int j = j0 + lane;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const bool above = j < vend && tk_above(sS[(warp * 2 + rr) * TK_BV + lane], j, bs[rr], bi[rr]);
      cnt[rr] += __popc(__ballot_sync(0xffffffffu, above));
    }
  });
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int row = row0 + warp * 2 + rr;
    if (lane == 0 && row < Nt && cnt[rr]) atomicAdd(rank + row, (unsigned long long)cnt[rr]);
  }
}

// One warp per query row i: the best of its positives perm[lo[i]:hi[i]] under the key order, each scored by sim_dot;
// (-inf, INT_MAX) when it has none.
__global__ void __launch_bounds__(256)
sim_best_positive_kernel(const float* __restrict__ t, const float* __restrict__ v, int Nt, int H,
                         const int* __restrict__ perm, const int* __restrict__ lo, const int* __restrict__ hi,
                         float* __restrict__ best_s, int* __restrict__ best_i) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= Nt) return;
  float bs = -INFINITY;
  int bi = INT_MAX;
  for (int p = lo[row], end = hi[row]; p < end; ++p) {
    const int j = perm[p];
    const float s = sim_dot(t + (long long)row * H, v + (long long)j * H, H, lane);
    if (tk_above(s, j, bs, bi)) { bs = s; bi = j; }
  }
  if (lane == 0) { best_s[row] = bs; best_i[row] = bi; }
}

// number of the first n entries of sorted list (ls, li) that rank above (s, i), or also those equal to it
__device__ __forceinline__ int tk_rank(const float* ls, const int* li, int n, float s, int i, bool or_equal) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const bool in = tk_above(ls[mid], li[mid], s, i) || (or_equal && ls[mid] == s && li[mid] == i);
    if (in) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One CTA per text row: the splits' sorted lists part_s / part_i [splits][Nt][k] merged in split order into the row's
// top k.  An element's merged position is its own index plus the count of the other list's elements above it (ties,
// which only padding entries have, go to the earlier list), so each position is written once.
__global__ void __launch_bounds__(TK_MAX_K)
topk_merge_kernel(const float* __restrict__ part_s, const int* __restrict__ part_i, int splits, int Nt, int k,
                  float* __restrict__ out_s, int* __restrict__ out_i) {
  __shared__ float ms[3][TK_MAX_K];
  __shared__ int mi[3][TK_MAX_K];
  const int row = blockIdx.x, tid = threadIdx.x;
  int cur = 0;
  if (tid < k) { ms[0][tid] = part_s[(long long)row * k + tid]; mi[0][tid] = part_i[(long long)row * k + tid]; }
  for (int s = 1; s < splits; ++s) {
    const int nxt = cur == 0 ? 1 : 0;
    if (tid < k) {
      ms[2][tid] = part_s[((long long)s * Nt + row) * k + tid];
      mi[2][tid] = part_i[((long long)s * Nt + row) * k + tid];
    }
    __syncthreads();
    if (tid < k) {
      const float as = ms[cur][tid], bs = ms[2][tid];
      const int ai = mi[cur][tid], bi = mi[2][tid];
      const int pa = tid + tk_rank(ms[2], mi[2], k, as, ai, false);
      const int pb = tid + tk_rank(ms[cur], mi[cur], k, bs, bi, true);
      if (pa < k) { ms[nxt][pa] = as; mi[nxt][pa] = ai; }
      if (pb < k) { ms[nxt][pb] = bs; mi[nxt][pb] = bi; }
    }
    __syncthreads();
    cur = nxt;
  }
  if (tid < k) { out_s[(long long)row * k + tid] = ms[cur][tid]; out_i[(long long)row * k + tid] = mi[cur][tid]; }
}

// Split the gallery only when the text blocks alone leave SMs idle; each split keeps at least 8 tiles.  -> splits, and
// the videos per split `per` (a multiple of BV)
static int tk_gallery_splits(int bx, int Nv, int& per) {
  const int max_splits = (Nv + 8 * TK_BV - 1) / (8 * TK_BV);
  int splits = (2 * usable_sms() + bx - 1) / bx;
  splits = splits < 1 ? 1 : splits > max_splits ? max_splits : splits;
  per = ((Nv + splits - 1) / splits + TK_BV - 1) / TK_BV * TK_BV;
  return (Nv + per - 1) / per;
}

}  // namespace univl

using namespace univl;

extern "C" int univl_sim_topk(const float* t, const float* v, float* scores, int* index, int Nt, int Nv, int H, int k,
                              void* stream) {
  UNIVL_CHECK_ARG(t && v && scores && index, "sim_topk: null pointer");
  UNIVL_CHECK_ARG(Nt >= 0 && Nv > 0 && H > 0 && (H % 4) == 0,
                  "sim_topk: bad shape Nt=%d Nv=%d H=%d (H must be a positive multiple of 4)", Nt, Nv, H);
  UNIVL_CHECK_ARG(k >= 1 && k <= TK_MAX_K && k <= Nv, "sim_topk: k=%d must be in [1, min(%d, Nv=%d)]", k, TK_MAX_K,
                  Nv);
  UNIVL_CHECK_ARG(((uintptr_t)t & 15) == 0 && ((uintptr_t)v & 15) == 0, "sim_topk: t and v must be 16-byte aligned");
  if (Nt == 0) return UNIVL_OK;
  const int Hp = (H + TK_KC - 1) / TK_KC * TK_KC;
  const size_t smem = (size_t)tk_engine_floats(Hp) * sizeof(float) + (size_t)TK_BT * k * (sizeof(float) + sizeof(int));
  UNIVL_CHECK_ARG(smem <= 227 * 1024, "sim_topk: H=%d with k=%d needs %zu bytes of shared memory", H, k, smem);
  const cudaStream_t st = (cudaStream_t)stream;
  const int bx = (Nt + TK_BT - 1) / TK_BT;
  int per;
  const int splits = tk_gallery_splits(bx, Nv, per);
  cudaError_t e = cudaFuncSetAttribute(sim_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "sim_topk smem attribute: %s", cudaGetErrorString(e));
  if (splits == 1) {
    sim_topk_kernel<<<dim3(bx, 1), TK_THREADS, smem, st>>>(t, v, Nt, Nv, H, Hp, k, per, scores, index);
    UNIVL_CHECK_LAUNCH("sim_topk");
    return UNIVL_OK;
  }
  void* part = nullptr;
  const size_t n = (size_t)splits * Nt * k;
  if (int rc = scratch_alloc(&part, n * (sizeof(float) + sizeof(int)), st)) return rc;
  float* ps = (float*)part;
  int* pi = (int*)(ps + n);
  sim_topk_kernel<<<dim3(bx, splits), TK_THREADS, smem, st>>>(t, v, Nt, Nv, H, Hp, k, per, ps, pi);
  e = cudaGetLastError();
  if (e == cudaSuccess) {
    topk_merge_kernel<<<Nt, TK_MAX_K, 0, st>>>(ps, pi, splits, Nt, k, scores, index);
    e = cudaGetLastError();
  }
  cudaFreeAsync(part, st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "sim_topk launch: %s", cudaGetErrorString(e));
  return UNIVL_OK;
}

extern "C" int univl_sim_best_positive(const float* t, const float* v, const int* perm, const int* lo, const int* hi,
                                       float* best_s, int* best_i, int Nt, int Nv, int H, void* stream) {
  UNIVL_CHECK_ARG(t && v && perm && lo && hi && best_s && best_i, "sim_best_positive: null pointer");
  UNIVL_CHECK_ARG(Nt >= 0 && Nv > 0 && H > 0, "sim_best_positive: bad shape Nt=%d Nv=%d H=%d", Nt, Nv, H);
  if (Nt == 0) return UNIVL_OK;
  sim_best_positive_kernel<<<(int)(((long long)Nt * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      t, v, Nt, H, perm, lo, hi, best_s, best_i);
  UNIVL_CHECK_LAUNCH("sim_best_positive");
  return UNIVL_OK;
}

extern "C" int univl_sim_rank(const float* t, const float* v, const float* best_s, const int* best_i, long long* rank,
                              int Nt, int Nv, int H, void* stream) {
  UNIVL_CHECK_ARG(t && v && best_s && best_i && rank, "sim_rank: null pointer");
  UNIVL_CHECK_ARG(Nt >= 0 && Nv > 0 && H > 0 && (H % 4) == 0,
                  "sim_rank: bad shape Nt=%d Nv=%d H=%d (H must be a positive multiple of 4)", Nt, Nv, H);
  UNIVL_CHECK_ARG(((uintptr_t)t & 15) == 0 && ((uintptr_t)v & 15) == 0, "sim_rank: t and v must be 16-byte aligned");
  if (Nt == 0) return UNIVL_OK;
  const int Hp = (H + TK_KC - 1) / TK_KC * TK_KC;
  const size_t smem = (size_t)tk_engine_floats(Hp) * sizeof(float);
  UNIVL_CHECK_ARG(smem <= 227 * 1024, "sim_rank: H=%d needs %zu bytes of shared memory", H, smem);
  const cudaStream_t st = (cudaStream_t)stream;
  const int bx = (Nt + TK_BT - 1) / TK_BT;
  int per;
  const int splits = tk_gallery_splits(bx, Nv, per);
  cudaError_t e = cudaFuncSetAttribute(sim_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "sim_rank smem attribute: %s", cudaGetErrorString(e));
  e = cudaMemsetAsync(rank, 0, (size_t)Nt * sizeof(long long), st);
  if (e != cudaSuccess) return set_error(UNIVL_ERR_CUDA, "sim_rank memset: %s", cudaGetErrorString(e));
  sim_rank_kernel<<<dim3(bx, splits), TK_THREADS, smem, st>>>(t, v, Nt, Nv, H, Hp, per, best_s, best_i,
                                                             (unsigned long long*)rank);
  UNIVL_CHECK_LAUNCH("sim_rank");
  return UNIVL_OK;
}
