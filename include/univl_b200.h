/* univl_b200 — C ABI of the H100-native UniVL hot path (libunivl_b200.so, sm_90a).
 *
 * The reference (microsoft/UniVL) has no FFI: its "plugin API" is the Python class surface of
 * modules/modeling.py (UniVL.forward :188-271 etc.), which univl_b200/modules/ mirrors.  This header is the new
 * boundary UNDER that surface: one entry point per fused kernel, each replacing the aten-op sequence of the
 * reference lines cited beside it.  Conventions (SURVEY.md §8b):
 *   - plain pointers (device memory owned by the caller) and sizes; no torch types; `stream` is a cudaStream_t
 *   - no allocation, no synchronisation, no global mutable state inside; safe to call under CUDA-graph capture
 *   - return 0 on success, negative on error (univl_last_error_string() describes it); never a silent fallback
 *   - activations bf16 row-major; parameters / statistics / losses fp32; ids, masks, labels int64 (as the
 *     reference dataloaders emit them)
 *   - dropout masks are Philox4x32-10(seed, stream, element index), regenerated in backward, never stored;
 *     `rng_state` points to device memory {uint64 seed, uint64 epoch} and the kernels use stream = stream_id +
 *     (epoch << 20), so a captured CUDA graph draws fresh masks on every replay once univl_rng_advance ran
 */
#ifndef UNIVL_B200_H_
#define UNIVL_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

const char* univl_last_error_string(void);
int univl_abi_version(void);
/* Number of SMs a concurrent collective kernel (NCCL all-reduce on another stream) occupies while the kernels enqueued
 * from now on run; persistent grids (GEMM, fused attention) are sized to the remaining SMs.  0 = none
 * (default).  Process-wide; read at enqueue time (captured graphs keep their grids).
 * No reference counterpart: DDP's overlapped bucket all-reduce (main_task_retrieval.py:197) leaves this to cuBLAS. */
int univl_set_reserved_sms(int n);
/* dst[r * ld + c] += sum over k of part[k][r][c] (fp32, part [nparts][rows][cols] contiguous, left unchanged): the
 * ordered reduction every deterministic cross-block sum of the library ends in.  Each element's rows are added in
 * ascending k (t = 0; t += part[k]), then t is added into dst, so the bits depend only on the inputs. */
int univl_partials_reduce(const float* part, int nparts, long long rows, long long cols, float* dst, long long ld,
                          void* stream);

/* ---- GEMM (wgmma / TMA) ---------------------------------------------------------------------------------
 * D[M,N] = epilogue(sum_k A(m,k) B(n,k)), bf16 operands, fp32 accumulation.
 * A is [M,Kc] row-major (a_mn_major=0) or [Kc,M] row-major (a_mn_major=1); likewise B with N.
 * Replaces every nn.Linear forward / dgrad / wgrad of the hot path:
 *   module_bert.py:172-174 (q,k,v), :208 (attention output), :234 (intermediate), :247 (output),
 *   module_visual.py:122 (1024->768), module_bert.py:327-330 + module_decoder.py:180-182 (vocab projection),
 *   module_visual.py:308-311 (MFM projection), modeling.py:285 (MFM logits), module_cross.py:284 (pooler).
 * epilogue: 0 out(bf16)=alpha*acc+bias | 1 aux_out(bf16)=acc+bias, out(bf16)=gelu_erf(.) (until_module.py:28-33)
 *           2 out(bf16)=acc*gelu'(aux_in) | 3 out(bf16)=alpha*acc+aux_in | 4 out(f32)=alpha*acc+bias
 *           5 out(f32)+=alpha*acc (gradient accumulation; split-K partials are summed in split order)
 * block_n: 0 = auto | 64 | 128 | 256.  split_k: 0 = auto (epilogue 5 only).
 * Aliasing: aux_in may be out itself (the same pointer and the same leading dimension, computed in place); any other
 * overlap of aux_in or aux_out with out is undefined. */
int univl_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                    int M, int N, int Kc, void* out, long long ldo, int epilogue, const float* bias,
                    const void* aux_in, long long ld_aux_in, void* aux_out, long long ld_aux_out, float alpha,
                    int block_n, int split_k, void* stream);
/* kernel variant univl_gemm_bf16 launches for this problem: 1 = the persistent wgmma kernel (the only one); a pure
 * function of its arguments (measurement aid: bench.py attributes launch times to the dominant kernel with it) */
int univl_gemm_plan(int M, int N, int Kc, int epilogue, int block_n, int split_k);

/* ---- FP8 (e4m3) forward GEMM with block scaling (cross-encoder evaluation) ------------------------------------
 * A block of e4m3 codes q with its fp32 scale s stands for q * s.  s = 2^ceil(log2(amax / 448)) of the block's largest
 * magnitude (1 for an all-zero block, at least 2^-126); codes round to nearest even and saturate at +-448.
 * univl_quantize_e4m3_rows:   x bf16 [M, K] (ldx) -> q e4m3 [M, K] (ldq), scale fp32 [K/128, M]: 1 x 128 blocks.
 * univl_quantize_e4m3_blocks: w fp32 [N, K] (ldw) -> q e4m3 [N, K] (ldq), scale fp32 [N/128, K/128]: 128 x 128 blocks.
 * univl_gemm_fp8: D[M,N] = epilogue(sum_kb a_scale[kb, m] b_scale[n/128, kb] sum_{k in kb} A(m,k) B(n,k)),
 *   A e4m3 [M, Kc] (lda) with a_scale [Kc/128, M], B e4m3 [N, Kc] (ldb) with b_scale [N/128, Kc/128], both K-major;
 *   Kc and N multiples of 128; each 128-wide K block accumulates apart and is added in fp32 with its two scales.
 *   epilogue 0: out bf16 [M, ldo] = D + bias      (module_bert.py:208 attention output, :247 FFN output, K/V)
 *            1: out e4m3 [M, ldo] with out_scale [N/128, M] = gelu_erf(D + bias) quantized per (row, 128 columns)
 *               (module_bert.py:234 intermediate; no pre-activation is written: forward only) */
int univl_quantize_e4m3_rows(const void* x, long long ldx, void* q, long long ldq, float* scale, int M, int K,
                             void* stream);
int univl_quantize_e4m3_blocks(const float* w, long long ldw, void* q, long long ldq, float* scale, int N, int K,
                               void* stream);
int univl_gemm_fp8(const void* A, long long lda, const float* a_scale, const void* B, long long ldb,
                   const float* b_scale, int M, int N, int Kc, int epilogue, const float* bias, void* out,
                   long long ldo, float* out_scale, void* stream);

/* ---- LayerNorm family (until_module.py:49-53; eps inside sqrt) ---------------------------------------------
 * drop_mode 1: y = LN(dropout(x) + res)   (module_bert.py:207-211, :246-250)
 * drop_mode 2: y = dropout(LN(x + res))   (embeddings; head transforms use p = 0) */
int univl_layernorm_fwd(const void* x, const void* res, const float* gamma, const float* beta, void* y, float* mean,
                        float* rstd, int rows, int cols, float eps, float p_drop, int drop_mode,
                        const unsigned long long* rng_state, unsigned long long stream_id, void* stream);
int univl_layernorm_bwd(const void* dy, const void* dy2, const void* x, const void* res, const float* gamma,
                        const float* mean, const float* rstd, void* dx_res, void* dx_dense, float* dgamma,
                        float* dbeta, float* dbias, int rows, int cols, float p_drop, int drop_mode,
                        const unsigned long long* rng_state, unsigned long long stream_id, void* stream);
/* NormalizeVideo (modeling.py:88-92): fp32 rows in, bf16 out; backward yields parameter gradients only */
int univl_layernorm_f32_fwd(const float* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                            int rows, int cols, float eps, void* stream);
int univl_layernorm_f32_bwd(const void* dy, const float* x, const float* gamma, const float* mean, const float* rstd,
                            float* dgamma, float* dbeta, int rows, int cols, void* stream);

/* ---- embeddings ---------------------------------------------------------------------------------------------
 * text: word[id] + pos[s] (+ type[t]) -> LN -> dropout   (module_bert.py:132-146; module_decoder.py:309-320) */
int univl_embed_text_fwd(const long long* ids, const long long* type_ids, const float* word, const float* pos,
                         const float* type, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                         int n_seq, int S, int H, int vocab, float eps, float p_drop, const unsigned long long* rng_state,
                         unsigned long long stream_id, void* stream);
int univl_embed_text_bwd(const void* dy, const long long* ids, const long long* type_ids, const float* word,
                         const float* pos, const float* type, const float* gamma, const float* mean,
                         const float* rstd, float* dword, float* dpos, float* dtype, float* dgamma, float* dbeta,
                         int n_seq, int S, int H, int vocab, float p_drop, const unsigned long long* rng_state,
                         unsigned long long stream_id, void* stream);
/* activation sources a[Na,Wa,H] (+ b[Nb,Fb,H]) + pos[s] (+ type[s>=Wa]) -> LN -> dropout
 * (module_visual.py:118-131; module_cross.py:123-138 with modeling.py:315-325).  `all_pairs` is the number of pairing
 * groups: 0 = aligned (sequence p reads a[p], b[p]; Na == Nb); 1 = the B x B text-video pairing of
 * modeling.py:341-375 without materialising the repeats (p = i * Nb + j); G > 1 = G independent micro-batches, group g
 * pairing a rows [g Na/G, (g+1) Na/G) with b rows [g Nb/G, (g+1) Nb/G): Na Nb / G sequences, sequence p of group
 * g = p / (Gt Gv), r = p mod (Gt Gv), reads a[g Gt + r / Gv], b[g Gv + r % Gv] with Gt = Na/G, Gv = Nb/G (G must divide
 * Na and Nb).  The backward sums a source row's gradient over the pairs of its own group only. */
int univl_embed_src_fwd(const void* a, const void* b, const float* pos, const float* type, const float* gamma,
                        const float* beta, void* y, float* mean, float* rstd, int Na, int Wa, int Nb, int Fb,
                        int all_pairs, int H, float eps, float p_drop, const unsigned long long* rng_state,
                        unsigned long long stream_id, void* stream);
int univl_embed_src_bwd(const void* dy, const void* a, const void* b, const float* pos, const float* type,
                        const float* gamma, const float* mean, const float* rstd, void* da, void* db, float* dpos,
                        float* dtype, float* dgamma, float* dbeta, int Na, int Wa, int Nb, int Fb, int all_pairs,
                        int H, float p_drop, const unsigned long long* rng_state, unsigned long long stream_id, void* stream);

/* ---- attention core (module_bert.py:176-196; module_decoder.py:225-245, mask :385-396) -------------------------
 * ctx = dropout(softmax(Q K^T * scale + mask)) V per (sequence, head), head dim 64.
 * mask = -10000 * (key padded [or key > query if causal]); key padding = concat(mask_a[i,:Wa], mask_b[j,:Fb]) with
 * (i, j) the sources of the sequence under `all_pairs` pairing groups as in univl_embed_src_fwd (here Gv = Nb / G and
 * Gt = n_seq / Nb; G > 1 needs G | Nb and Nb | n_seq).
 * univl_attention_fwd / _bwd take Sq, Sk <= 256 (whole K/V of a head in shared memory); univl_attention_long_fwd /
 * _bwd take the same arguments for 0 < Sq, Sk <= 1024 with 12 heads (key-tiled; rng_layout must be 0), which covers
 * the model's position tables: text, visual and decoder <= 512 tokens, cross encoder <= 1024.  Both draw the same
 * dropout mask for the same (seed, stream, sequence, head, query, key). */
int univl_attention_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                        void* o, long long ldo, float* lse, const long long* mask_a, const long long* mask_b, int Wa,
                        int Fb, int Nb, int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal, float scale,
                        float p_drop, const unsigned long long* rng_state, unsigned long long stream_id, void* stream);
int univl_attention_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                        const void* o, long long ldo, const float* lse, const void* d_o, long long lddo, void* dq,
                        long long lddq, void* dk, long long lddk, void* dv, long long lddv, const long long* mask_a,
                        const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs, int n_seq, int heads, int Sq,
                        int Sk, int causal, float scale, float p_drop, const unsigned long long* rng_state,
                        unsigned long long stream_id, int rng_layout, float* dbq, float* dbk, float* dbv, void* stream);
int univl_attention_long_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                             void* o, long long ldo, float* lse, const long long* mask_a, const long long* mask_b,
                             int Wa, int Fb, int Nb, int all_pairs, int n_seq, int heads, int Sq, int Sk, int causal,
                             float scale, float p_drop, const unsigned long long* rng_state,
                             unsigned long long stream_id, void* stream);
int univl_attention_long_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                             const void* o, long long ldo, const float* lse, const void* d_o, long long lddo, void* dq,
                             long long lddq, void* dk, long long lddk, void* dv, long long lddv,
                             const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs,
                             int n_seq, int heads, int Sq, int Sk, int causal, float scale, float p_drop,
                             const unsigned long long* rng_state, unsigned long long stream_id, int rng_layout,
                             float* dbq, float* dbk, float* dbv, void* stream);
/* Forward only, no dropout: the attention core of the Na x Nb sequences concat(a_i, b_j), p = i * Nb + j (all_pairs
 * = 1 above), with Q/K/V read from per-source projections instead of per-pair copies.  Row r < Wa of sequence p reads
 * row i * Wa + r of (qa, ka, va); row r >= Wa reads row j * Fb + (r - Wa) of (qb, kb, vb).  The cross encoder's eval
 * similarity (modeling.py:355-373 under model.eval() / no_grad) computes its first layer's projections once per text
 * row and once per video row and scores every pair through this entry.  Sq = Wa + Fb (every query row) or 1 (token 0
 * only, from a_i); the context is [Na * Nb * Sq, heads * 64] as univl_attention_fwd writes it; lse is nullable.  Masks
 * as above (both parts needed when Fb > 0); 12 heads, 0 < Wa + Fb <= 1024; row strides multiples of 8 and 16-byte
 * aligned q/k/v.  Runs univl_attention_fwd's kernel up to 256 tokens and univl_attention_long_fwd's above, and gives
 * the same bits as they do on the materialised per-pair q/k/v. */
int univl_attention_pair_fwd(const void* qa, long long ldqa, const void* ka, long long ldka, const void* va,
                             long long ldva, const void* qb, long long ldqb, const void* kb, long long ldkb,
                             const void* vb, long long ldvb, void* o, long long ldo, float* lse,
                             const long long* mask_a, const long long* mask_b, int Na, int Wa, int Nb, int Fb,
                             int heads, int Sq, float scale, void* stream);
/* Forward only, no dropout, no mask: the attention core of n_seq variable-length sequences in one launch.  Sequence p
 * has Sk_p = cu_seqlens[p + 1] - cu_seqlens[p] keys (int32 [n_seq + 1], ascending), all of them real.  Two row
 * addressings of q/k/v:
 *   - pair (idx_a non-null): row r < len_a[p] of sequence p is row idx_a[start_a[p] + r] of (qa, ka, va), row
 *     r >= len_a[p] is row idx_b[start_b[p] + r - len_a[p]] of (qb, kb, vb) — univl_attention_pair_fwd's two sources
 *     with per-row index lists (int32) in place of i * Wa + r / j * Fb + r - Wa;
 *   - packed (idx_a, idx_b, start_a, start_b, len_a all null): row r of sequence p is row cu_seqlens[p] + r of
 *     (qa, ka, va); qb / kb / vb are ignored.
 * q_first = 0: every row queries and the context row of (p, r) is o[cu_seqlens[p] + r]; q_first = 1: one query per
 * sequence, its row 0 (under packed addressing: row p of qa instead), context in o[p].  lse (nullable) is fp32
 * [context rows, heads].  max_sk >= every Sk_p, 0 < max_sk <= 1024, sizes the launch: univl_attention_fwd's kernel up to
 * 256 keys, univl_attention_long_fwd's above; a sequence computes exactly what those kernels compute for it alone.  A
 * sequence without keys writes nothing.  12 heads; row strides multiples of 8 and 16-byte aligned q/k/v. */
int univl_attention_varlen_fwd(const void* qa, long long ldqa, const void* ka, long long ldka, const void* va,
                               long long ldva, const void* qb, long long ldqb, const void* kb, long long ldkb,
                               const void* vb, long long ldvb, const int* idx_a, const int* idx_b, const int* start_a,
                               const int* start_b, const int* len_a, const int* cu_seqlens, int n_seq, int max_sk,
                               int heads, int q_first, void* o, long long ldo, float* lse, float scale, void* stream);
/* The rows of univl_attention_varlen_fwd's sequences gathered into packed order: with the same addressing (pair: a, b
 * and the index lists; packed: a alone), row r of sequence p is copied to out[cu_seqlens[p] + r], or with q_first = 1
 * only row 0, to out[p].  bf16 [*, cols], cols a multiple of 8, 16-byte aligned rows (16-byte vectors). */
int univl_gather_rows_varlen(const void* a, long long lda, const void* b, long long ldb, const int* idx_a,
                             const int* idx_b, const int* start_a, const int* start_b, const int* len_a,
                             const int* cu_seqlens, int n_seq, int q_first, int cols, void* out, long long ldo,
                             void* stream);
/* Forward only, no mask, no dropout: attention of n_q single-token queries over indexed key rows (one decoder token per
 * hypothesis, module_decoder.py:225-245 at Sq = 1).  q bf16 [n_q, 768] (ldq), 12 heads of 64.  Keys come from ONE K|V
 * buffer kv: row x holds k in columns [0, 768) and v in [768, 1536) (ldkv >= 1536).  Query r attends to the n_keys[c]
 * rows key_rows[c * ld_rows + 0 .. n_keys[c] - 1] of kv, c = list_of_query[r] (list_of_query null: c = r); every
 * listed row is a real key and no other row is read.  Lists hold 0 to 1024 keys; a query whose list is empty writes
 * nothing.  Output o bf16 [n_q, 768] (ldo), lse (nullable) fp32 [n_q, 12].  fp32 accumulation; the key splits are
 * merged in a fixed order (no floating-point atomics) and the launch does not depend on the SM count, so the bits
 * depend on the inputs alone.  16-byte aligned q / kv with row strides multiples of 8. */
int univl_attention_decode_fwd(const void* q, long long ldq, const void* kv, long long ldkv, const int* key_rows,
                               long long ld_rows, const int* n_keys, const int* list_of_query, int n_q, int heads,
                               void* o, long long ldo, float* lse, float scale, void* stream);
/* ---- fused QKV projection + self-attention, forward (wgmma / TMA; module_bert.py:171-197 as ONE kernel) --------------
 * ctx[T,H] = merge_heads(dropout(softmax((x Wq^T + bq)(x Wk^T + bk)^T * scale + mask)) (x Wv^T + bv)), T = n_seq * S,
 * H = heads * 64 = 768.  wqkv: bf16 [3H, H] (query | key | value rows), bias fp32 [3H].  The [T,3H] projections and the
 * score matrices stay on chip; qkv_out (nullable) additionally receives bf16 q | k | v for the backward pass.  Supported
 * when univl_fused_qkv_attention_supported(...) == 1 (12 heads, S % 16 == 0, 16 <= S <= 128); masks as above.  Dropout
 * masks use the row-major layout that univl_attention_bwd regenerates with rng_layout = 1. */
int univl_fused_qkv_attention_supported(int n_seq, int heads, int S, int H);
int univl_fused_qkv_attention_fwd(const void* x, long long ldx, const void* wqkv, long long ldw, const float* bias,
                                  void* qkv_out, long long ld_qkv, void* o, long long ldo, float* lse,
                                  const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb,
                                  int all_pairs, int n_seq, int heads, int S, int causal, float scale, float p_drop,
                                  const unsigned long long* rng_state, unsigned long long stream_id, void* stream);
/* backward of the attention core for the same shapes, on wgmma (S, dP, dS, P in registers / shared memory only):
 * dqkv[T,3H] = d(q | k | v) from the saved qkv, the context o, d_o and lse; dbias (nullable, fp32 [3H]) accumulates the
 * projection-bias gradients (column sums).  Masks / dropout as the fused forward (row-major dropout layout). */
int univl_fused_attention_bwd(const void* qkv, long long ld_qkv, const void* o, long long ldo, const float* lse,
                              const void* d_o, long long lddo, void* dqkv, long long ld_dqkv, float* dbias,
                              const long long* mask_a, const long long* mask_b, int Wa, int Fb, int Nb, int all_pairs,
                              int n_seq, int heads, int S, int causal, float scale, float p_drop,
                              const unsigned long long* rng_state, unsigned long long stream_id, void* stream);

/* ---- utilities ------------------------------------------------------------------------------------------------ */
int univl_colsum_bf16(const void* x, long long ld, float* out, int rows, int cols, void* stream); /* bias grads */
int univl_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream);
int univl_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream); /* bf16 gradient payload -> fp32 */
int univl_multi_cast_f32_to_bf16(const unsigned long long* device_table, int n_tensors, int blocks_per_tensor,
                                 void* stream);
int univl_fill_f32(float* p, float value, long long n, void* stream);
int univl_rng_advance(unsigned long long* rng_state, void* stream); /* ++epoch (device side) */
/* elementwise bf16: out = dy * gelu_erf'(pre) (head transforms, module_bert.py:308-312); tanh and its backward
 * (poolers, module_bert.py:290-296) */
int univl_gelu_fwd_bf16(const void* x, void* out, long long n, void* stream);
int univl_gelu_bwd_bf16(const void* dy, const void* pre, void* out, long long n, void* stream);
int univl_tanh_fwd_bf16(const void* x, void* out, long long n, void* stream);
int univl_tanh_bwd_bf16(const void* dy, const void* y, void* out, long long n, void* stream);
int univl_scale_f32(float* dst, const float* src, long long n, const float* gscale, void* stream);

/* ---- pooling, similarity, losses -------------------------------------------------------------------------------
 * masked mean pooling (modeling.py:327-339) [+ F.normalize, :386-388] */
int univl_meanpool_fwd(const void* x, const long long* mask, float* out, float* norm_out, int N, int S, int H,
                       int skip_first, int guard_zero, int l2norm, void* stream);
int univl_meanpool_bwd(const float* dy, const float* y, const float* norm, const long long* mask, void* dx, int N,
                       int S, int H, int skip_first, int guard_zero, int l2norm, void* stream);
/* sim = T V^T (modeling.py:389).  groups = G >= 1: t [G Bt, H], v [G Bv, H] and sim the block diagonal [G, Bt, Bv],
 * sim[g] = t[g Bt : (g+1) Bt] v[g Bv : (g+1) Bv]^T (one similarity matrix per micro-batch) */
int univl_sim_matmul_fwd(const float* t, const float* v, float* sim, int Bt, int Bv, int H, int groups, void* stream);
int univl_sim_matmul_bwd(const float* dsim, const float* t, const float* v, float* dt, float* dv, int Bt, int Bv,
                         int H, int groups, void* stream);
/* losses on sim[G,B,B] (until_module.py:182-251): loss = mean over the G groups of the reference loss of sim[g]; each
 * also writes dsim for an upstream gradient of 1.  One CTA per group, the group losses averaged in group order: no
 * floating-point atomics across groups, deterministic.  G = 1 is the single [B, B] loss. */
int univl_maxmargin_loss(const float* sim, float* loss, float* dsim, int B, float margin, int n_pair, float w_same,
                         float w_diff, int groups, void* stream);
int univl_crossen_loss(const float* sim, float* loss, float* dsim, int B, int groups, void* stream);
int univl_milnce_loss(const float* sim, float* loss, float* dsim, int batch_size, int n_pair, int groups,
                      void* stream);
/* CrossEntropyLoss(ignore_index) over wide rows (modeling.py:253, :275) and the MFM NCE (modeling.py:278-297:
 * target_mode 1 = diagonal target, pair_mask adds (1 - m_r m_c) * -1e8).  groups = G >= 1 splits the T rows into G
 * consecutive micro-batches of R = T / G rows: loss = mean over groups of (sum / count of the group's scored rows), a
 * group without a scored row giving NaN like the reference's mean of an empty selection; the backward scales row r by
 * (gscale / G) / count[group(r)].  Grouped target_mode 1 takes V = R: row r of group g holds its logits against the
 * group's own R frames, target r - g R, mask columns pair_mask[g R + c].  sum_count: 2 G floats (sums, then counts). */
int univl_softmax_xent_fwd(const float* logits, long long ld, const long long* labels, const long long* pair_mask,
                           float* lse, float* sum_count, float* loss, int T, int V, int target_mode,
                           long long ignore_index, int groups, void* stream);
int univl_softmax_xent_bwd(const float* logits, long long ld, const long long* labels, const long long* pair_mask,
                           const float* lse, const float* sum_count, const float* gscale, void* dlogits,
                           long long ld_d, int T, int V, int target_mode, long long ignore_index, int groups,
                           void* stream);
/* The same CrossEntropyLoss(ignore_index = -1) for target_mode 0 over the tied vocabulary projection, with the logits
 * never written to memory (module_bert.py:327-330 + modeling.py:253, :275):
 *   logit[r, c] = x[r, :] . W[c, :] + bias[c]   (x bf16 [T, Kc], W bf16 [V, Kc], both K-major; bias fp32 [V], nullable)
 * computed by the wgmma GEMM's mainloop with EPI_BIAS_F32's bits.
 * univl_vocab_xent_fwd: loss, lse [T] (0 for unscored rows) and sum_count [2 G] as univl_softmax_xent_fwd defines them;
 *   the per-group sums are taken in a fixed order (no floating-point atomics), so the result is deterministic.
 *   workspace: device memory of at least univl_vocab_xent_workspace(T, V) bytes, 16-byte aligned, used within the call
 *   on `stream` only (so one buffer per stream; safe under CUDA-graph capture).  Labels must be -1 or in [0, V); any
 *   other label makes the loss NaN.
 * univl_vocab_xent_bwd: recomputes the logits and writes dlogits bf16 [T, ld_d] = univl_softmax_xent_bwd's result from
 *   them: (exp(logit - lse) - onehot) (gscale / G) / count[group] for scored rows, 0 for unscored rows and columns
 *   [V, ld_d); V <= ld_d <= V rounded up to 128, ld_d even.  The dgrad, wgrad and bias gradient then read dlogits.
 * univl_vocab_xent_workspace: bytes (>= 0) of that workspace, or negative on error. */
int univl_vocab_xent_workspace(int T, int V);
int univl_vocab_xent_fwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                         const long long* labels, float* lse, float* sum_count, float* loss, void* workspace,
                         long long workspace_bytes, int T, int V, int Kc, int groups, void* stream);
int univl_vocab_xent_bwd(const void* x, long long ldx, const void* w, long long ldw, const float* bias,
                         const long long* labels, const float* lse, const float* sum_count, const float* gscale,
                         void* dlogits, long long ld_d, int T, int V, int Kc, int groups, void* stream);
/* cross pooler tanh + similarity_dense (module_cross.py:281-287; modeling.py:371): out[r] = tanh(u[r,:]).w + b */
int univl_pooler_sim_fwd(const void* u, const float* w, const float* b, float* out, int N, int H, void* stream);
int univl_pooler_sim_bwd(const void* u, const float* w, const float* dout, void* du, float* dw, float* db, int N,
                         int H, void* stream);

/* ---- optimizer (modules/optimization.py:103-167 + driver clip main_task_retrieval.py:347) --------------------- */
int univl_bert_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, const void* segs, int n_chunks,
                         int n_tensors, float* scratch, long long* step, float b1, float b2, float eps,
                         float max_grad_norm, float global_clip_norm, float warmup, long long t_total,
                         float grad_scale, void* stream);
/* the same step reading the gradients from a bf16 buffer (the summed all-reduce payload; same element offsets as p) */
int univl_bert_adam_step_bf16grad(float* p, const void* g_bf16, float* m, float* v, void* p_bf16, const void* segs,
                                  int n_chunks, int n_tensors, float* scratch, long long* step, float b1, float b2,
                                  float eps, float max_grad_norm, float global_clip_norm, float warmup,
                                  long long t_total, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UNIVL_B200_H_ */
