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
 * block_n: 0 = auto | 64 | 128 | 256.  split_k: 0 = auto (epilogue 5 only). */
int univl_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                    int M, int N, int Kc, void* out, long long ldo, int epilogue, const float* bias,
                    const void* aux_in, long long ld_aux_in, void* aux_out, long long ld_aux_out, float alpha,
                    int block_n, int split_k, void* stream);
/* kernel variant univl_gemm_bf16 launches for this problem: 1 = the persistent wgmma kernel (the only one); a pure
 * function of its arguments (measurement aid: bench.py attributes launch times to the dominant kernel with it) */
int univl_gemm_plan(int M, int N, int Kc, int epilogue, int block_n, int split_k);

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
 * (module_visual.py:118-131; module_cross.py:123-138 with modeling.py:315-325; all_pairs=1 realises the B x B
 *  text-video pairing of modeling.py:341-375 without materialising the repeats) */
int univl_embed_src_fwd(const void* a, const void* b, const float* pos, const float* type, const float* gamma,
                        const float* beta, void* y, float* mean, float* rstd, int Na, int Wa, int Nb, int Fb,
                        int all_pairs, int H, float eps, float p_drop, const unsigned long long* rng_state,
                        unsigned long long stream_id, void* stream);
int univl_embed_src_bwd(const void* dy, const void* a, const void* b, const float* pos, const float* type,
                        const float* gamma, const float* mean, const float* rstd, void* da, void* db, float* dpos,
                        float* dtype, float* dgamma, float* dbeta, int Na, int Wa, int Nb, int Fb, int all_pairs,
                        int H, float p_drop, const unsigned long long* rng_state, unsigned long long stream_id, void* stream);

/* ---- attention core (module_bert.py:176-196; module_decoder.py:225-245, mask :385-396) -------------------------
 * ctx = dropout(softmax(Q K^T * scale + mask)) V per (sequence, head), head dim 64, S <= 256.
 * mask = -10000 * (key padded [or key > query if causal]); key padding = concat(mask_a[i,:Wa], mask_b[j,:Fb]). */
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
/* sim = T V^T (modeling.py:389) */
int univl_sim_matmul_fwd(const float* t, const float* v, float* sim, int Bt, int Bv, int H, void* stream);
int univl_sim_matmul_bwd(const float* dsim, const float* t, const float* v, float* dt, float* dv, int Bt, int Bv,
                         int H, void* stream);
/* losses on sim[B,B]; each also writes dsim for an upstream gradient of 1 (until_module.py:182-251) */
int univl_maxmargin_loss(const float* sim, float* loss, float* dsim, int B, float margin, int n_pair, float w_same,
                         float w_diff, void* stream);
int univl_crossen_loss(const float* sim, float* loss, float* dsim, int B, void* stream);
int univl_milnce_loss(const float* sim, float* loss, float* dsim, int batch_size, int n_pair, void* stream);
/* CrossEntropyLoss(ignore_index) over wide rows (modeling.py:253, :275) and the MFM NCE (modeling.py:278-297:
 * target_mode 1 = diagonal target, pair_mask adds (1 - m_r m_c) * -1e8) */
int univl_softmax_xent_fwd(const float* logits, long long ld, const long long* labels, const long long* pair_mask,
                           float* lse, float* sum_count, float* loss, int T, int V, int target_mode,
                           long long ignore_index, void* stream);
int univl_softmax_xent_bwd(const float* logits, long long ld, const long long* labels, const long long* pair_mask,
                           const float* lse, const float* sum_count, const float* gscale, void* dlogits,
                           long long ld_d, int T, int V, int target_mode, long long ignore_index, void* stream);
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
