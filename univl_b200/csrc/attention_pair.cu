// univl_b200 — attention core over (text, video) pair sequences, Q/K/V rows read from per-source projections.
//
// In evaluation (no dropout) the first cross layer's Q/K/V projections act on each token alone, and the token's input
// (the CrossEmbeddings LayerNorm of text i's or video j's row) does not depend on the pair.  So the projections are
// computed once per source row, and this entry reads them in place: sequence p = i * Nb + j (the all-pairs pairing of
// common.cuh pair_sources) takes rows r < Wa from the text source at row i * Wa + r and rows r >= Wa from the video
// source at row j * Fb + r - Wa.  The kernels are attention.cu's (S <= 256) and attention_long.cu's (S <= 1024) forward
// kernels with the pair row addressing (load_rows) as a compile-time variant, so the context equals that of
// univl_attention_fwd / univl_attention_long_fwd on the materialised per-pair q/k/v bit for bit.
//
// univl_attention_pair_list_fwd runs the same kernels on a list of pairs (sequence p = (text_index[p],
// video_index[p])), the pair's rows addressed as above (ADDR_PAIR_LIST), so a listed pair's context equals the
// all-pairs entry's for the same (i, j) bit for bit.  Its masks are the listed pairs' own rows, read aligned.
#include <climits>

#include "attention_common.cuh"

using namespace univl;

extern "C" int univl_attention_pair_fwd(const void* qa, long long ldqa, const void* ka, long long ldka, const void* va,
                                        long long ldva, const void* qb, long long ldqb, const void* kb, long long ldkb,
                                        const void* vb, long long ldvb, void* o, long long ldo, float* lse,
                                        const long long* mask_a, const long long* mask_b, int Na, int Wa, int Nb,
                                        int Fb, int heads, int Sq, float scale, void* stream) {
  UNIVL_CHECK_ARG(Na >= 0 && Wa > 0 && Nb > 0 && Fb >= 0,
                  "attention_pair_fwd: bad source shape Na=%d Wa=%d Nb=%d Fb=%d", Na, Wa, Nb, Fb);
  UNIVL_CHECK_ARG(heads == 12, "attention_pair_fwd: heads must be 12 (got %d)", heads);
  const int S = Wa + Fb;
  UNIVL_CHECK_ARG(Sq == 1 || Sq == S, "attention_pair_fwd: Sq must be 1 or Wa + Fb = %d (got %d)", S, Sq);
  UNIVL_CHECK_ARG((long long)Na * Nb * heads <= INT_MAX, "attention_pair_fwd: too many pairs (%d x %d)", Na, Nb);
  UNIVL_CHECK_ARG(Fb == 0 || (mask_a != nullptr && mask_b != nullptr),
                  "attention_pair_fwd: both mask parts are needed when Fb > 0");
  PairSrc pb{};
  if (Fb > 0)
    if (int rc = fill_pair_src(pb, qb, ldqb, kb, ldkb, vb, ldvb, "attention_pair_fwd")) return rc;
  const int n_seq = Na * Nb;
  AttnParams p = {};
  if (int rc = fill_common(p, qa, ldqa, ka, ldka, va, ldva, mask_a, mask_b, Wa, Fb, Nb, 1, n_seq, heads, Sq, S, 0,
                           scale, 0.f, nullptr, 0, 1024))
    return rc;
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_pair_fwd: bad output");
  if (n_seq == 0) return UNIVL_OK;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  return attention_fwd_any_launch(p, ADDR_PAIR, pb, VarlenSrc{}, (cudaStream_t)stream);
}

extern "C" int univl_attention_pair_list_fwd(const void* qa, long long ldqa, const void* ka, long long ldka,
                                             const void* va, long long ldva, const void* qb, long long ldqb,
                                             const void* kb, long long ldkb, const void* vb, long long ldvb, void* o,
                                             long long ldo, float* lse, const int* text_index, const int* video_index,
                                             const long long* mask_a, const long long* mask_b, int n_pairs, int Wa,
                                             int Fb, int heads, int Sq, float scale, void* stream) {
  UNIVL_CHECK_ARG(n_pairs >= 0 && Wa > 0 && Fb > 0, "attention_pair_list_fwd: bad shape n_pairs=%d Wa=%d Fb=%d",
                  n_pairs, Wa, Fb);
  UNIVL_CHECK_ARG(heads == 12, "attention_pair_list_fwd: heads must be 12 (got %d)", heads);
  const int S = Wa + Fb;
  UNIVL_CHECK_ARG(Sq == 1 || Sq == S, "attention_pair_list_fwd: Sq must be 1 or Wa + Fb = %d (got %d)", S, Sq);
  UNIVL_CHECK_ARG((long long)n_pairs * heads <= INT_MAX, "attention_pair_list_fwd: too many pairs (%d)", n_pairs);
  UNIVL_CHECK_ARG(text_index && video_index && mask_a && mask_b,
                  "attention_pair_list_fwd: the index lists and both mask parts are needed");
  PairSrc pb;
  if (int rc = fill_pair_src(pb, qb, ldqb, kb, ldkb, vb, ldvb, "attention_pair_list_fwd")) return rc;
  AttnParams p = {};
  // masks [n_pairs, Wa] / [n_pairs, Fb]: aligned pairing (row p of each part)
  if (int rc = fill_common(p, qa, ldqa, ka, ldka, va, ldva, mask_a, mask_b, Wa, Fb, n_pairs, 0, n_pairs, heads, Sq, S,
                           0, scale, 0.f, nullptr, 0, 1024))
    return rc;
  UNIVL_CHECK_ARG(o != nullptr && (ldo % 2) == 0, "attention_pair_list_fwd: bad output");
  if (n_pairs == 0) return UNIVL_OK;
  VarlenSrc vl{};
  vl.idx_a = text_index;
  vl.idx_b = video_index;
  p.o = (bf16*)o; p.ldo = ldo; p.lse = lse;
  return attention_fwd_any_launch(p, ADDR_PAIR_LIST, pb, vl, (cudaStream_t)stream);
}
