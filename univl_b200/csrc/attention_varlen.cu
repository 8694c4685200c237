// univl_b200 — variable-length attention forward and the row gather of the packed pair layout.
//
// Packed evaluation of the cross encoder (UNIVL_EVAL_LAYOUT=packed) computes every (text, video) pair on its valid
// tokens alone: sequence p is len_a(p) text tokens then len_b(p) video tokens, stored back to back, every one of them a
// real key.  Its first layer reads Q/K/V from the per-source projections through index lists (pair addressing, as
// univl_attention_pair_fwd reads them through i * Wa + r / j * Fb + r - Wa), the later layers from the packed rows
// (packed addressing).  Sequences of different lengths share one launch of attention.cu's forward kernel (longest
// sequence <= 256 keys) or attention_long.cu's (<= 1024): each CTA takes its own sequence's length, with the row
// addressing as a compile-time variant (attention_common.cuh VarlenSrc).
#include <climits>

#include "attention_common.cuh"

namespace univl {

constexpr int GATHER_THREADS = 128;

// one CTA per sequence: its rows (row 0 only under q_first) copied in 16-byte vectors to out[cu[p] + r] (out[p])
__global__ void __launch_bounds__(GATHER_THREADS)
gather_rows_varlen_kernel(const bf16* __restrict__ a, long long lda, const bf16* __restrict__ b, long long ldb,
                          const VarlenSrc vl, int cols, bf16* __restrict__ out, long long ldo) {
  pdl_trigger();
  pdl_wait();
  const int seq = blockIdx.x;
  const int rows = vl.q_first ? min(1, vl.cu[seq + 1] - vl.cu[seq]) : vl.cu[seq + 1] - vl.cu[seq];
  const long long obase = vl.q_first ? seq : vl.cu[seq];
  const int vec = cols >> 3;
  for (int idx = threadIdx.x; idx < rows * vec; idx += blockDim.x) {
    const int r = idx / vec, c = idx - r * vec;
    const uint4 v = *reinterpret_cast<const uint4*>(varlen_row(vl, a, lda, b, ldb, seq, r) + c * 8);
    *reinterpret_cast<uint4*>(out + (obase + r) * ldo + c * 8) = v;
  }
}

// the VarlenSrc argument checks both entries share
static int fill_varlen(VarlenSrc& vl, const void* a, long long lda, const void* b, long long ldb, const int* idx_a,
                       const int* idx_b, const int* start_a, const int* start_b, const int* len_a,
                       const int* cu_seqlens, int n_seq, int q_first, const char* what) {
  UNIVL_CHECK_ARG(n_seq >= 0 && cu_seqlens != nullptr, "%s: bad n_seq=%d or null cu_seqlens", what, n_seq);
  UNIVL_CHECK_ARG(q_first == 0 || q_first == 1, "%s: q_first must be 0 or 1 (got %d)", what, q_first);
  UNIVL_CHECK_ARG(a != nullptr && (lda % 8) == 0 && ((uintptr_t)a & 15) == 0,
                  "%s: the first source must be 16-byte aligned with a row stride that is a multiple of 8", what);
  const bool pair = idx_a != nullptr;
  if (pair) {
    UNIVL_CHECK_ARG(idx_b && start_a && start_b && len_a,
                    "%s: pair addressing needs idx_a, idx_b, start_a, start_b and len_a", what);
    UNIVL_CHECK_ARG(b != nullptr && (ldb % 8) == 0 && ((uintptr_t)b & 15) == 0,
                    "%s: the second source must be 16-byte aligned with a row stride that is a multiple of 8", what);
  } else {
    UNIVL_CHECK_ARG(!idx_b && !start_a && !start_b && !len_a,
                    "%s: packed addressing takes no index lists (idx_a is null)", what);
  }
  vl.cu = cu_seqlens;
  vl.idx_a = idx_a; vl.idx_b = idx_b; vl.start_a = start_a; vl.start_b = start_b; vl.len_a = len_a;
  vl.q_first = q_first;
  return UNIVL_OK;
}

}  // namespace univl

using namespace univl;

extern "C" int univl_attention_varlen_fwd(const void* qa, long long ldqa, const void* ka, long long ldka,
                                          const void* va, long long ldva, const void* qb, long long ldqb,
                                          const void* kb, long long ldkb, const void* vb, long long ldvb,
                                          const int* idx_a, const int* idx_b, const int* start_a, const int* start_b,
                                          const int* len_a, const int* cu_seqlens, int n_seq, int max_sk, int heads,
                                          int q_first, void* o, long long ldo, float* lse, float scale, void* stream) {
  UNIVL_CHECK_ARG(heads == 12, "attention_varlen_fwd: heads must be 12 (got %d)", heads);
  UNIVL_CHECK_ARG((long long)n_seq * heads <= INT_MAX, "attention_varlen_fwd: too many sequences (%d)", n_seq);
  VarlenSrc vl{};
  if (int rc = fill_varlen(vl, ka, ldka, kb, ldkb, idx_a, idx_b, start_a, start_b, len_a, cu_seqlens, n_seq, q_first,
                           "attention_varlen_fwd"))
    return rc;
  AttnParams p = {};
  if (int rc = fill_common(p, qa, ldqa, ka, ldka, va, ldva, nullptr, nullptr, 0, 0, 0, 0, n_seq, heads,
                           q_first ? 1 : max_sk, max_sk, 0, scale, 0.f, nullptr, 0, 1024))
    return rc;
  PairSrc pb{};
  if (idx_a != nullptr)
    if (int rc = fill_pair_src(pb, qb, ldqb, kb, ldkb, vb, ldvb, "attention_varlen_fwd")) return rc;
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_varlen_fwd: bad output");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  const Addr addr = idx_a != nullptr ? ADDR_VARLEN_PAIR : ADDR_VARLEN_PACKED;
  return attention_fwd_any_launch(p, addr, pb, vl, (cudaStream_t)stream);
}

extern "C" int univl_gather_rows_varlen(const void* a, long long lda, const void* b, long long ldb, const int* idx_a,
                                        const int* idx_b, const int* start_a, const int* start_b, const int* len_a,
                                        const int* cu_seqlens, int n_seq, int q_first, int cols, void* out,
                                        long long ldo, void* stream) {
  VarlenSrc vl{};
  if (int rc = fill_varlen(vl, a, lda, b, ldb, idx_a, idx_b, start_a, start_b, len_a, cu_seqlens, n_seq, q_first,
                           "gather_rows_varlen"))
    return rc;
  UNIVL_CHECK_ARG(cols > 0 && (cols % 8) == 0, "gather_rows_varlen: cols must be a positive multiple of 8 (got %d)",
                  cols);
  UNIVL_CHECK_ARG(out != nullptr && (ldo % 8) == 0 && ((uintptr_t)out & 15) == 0,
                  "gather_rows_varlen: out must be 16-byte aligned with a row stride that is a multiple of 8");
  if (n_seq == 0) return UNIVL_OK;
  launch_kernel(gather_rows_varlen_kernel, dim3(n_seq), dim3(GATHER_THREADS), 0, (cudaStream_t)stream, (const bf16*)a,
                lda, (const bf16*)b, ldb, vl, cols, (bf16*)out, ldo);
  UNIVL_CHECK_LAUNCH("gather_rows_varlen");
  return UNIVL_OK;
}
