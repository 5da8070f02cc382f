/* dalm_b200 — C ABI of the H100-native (sm_90a) RAG-e2e / retriever-only training-step kernels.
 *
 * The reference (arcee-ai/DALM) has no FFI: its hot path is Python calling PyTorch/HF/PEFT library kernels. Each entry
 * point below cites the reference call site whose library work it replaces (paths relative to the reference root).
 *
 * Conventions: plain pointers to DEVICE memory + sizes, a cudaStream_t passed as void*, no torch types. Every function
 * returns 0 on success; on failure it returns non-zero and dalm_b200_last_error() holds the message. Functions never
 * allocate or free caller memory. bf16 = raw 16-bit bfloat16; "token-major" = row index b*L + l.
 */
#ifndef DALM_B200_H
#define DALM_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- library plumbing ---- */
const char* dalm_b200_last_error(void);
const char* dalm_b200_version(void);
long long   dalm_b200_launch_count(void);          /* kernels launched by this library since the last reset */
void        dalm_b200_reset_launch_count(void);
int         dalm_b200_probe_device(void);          /* 0 iff the current device is sm_90 (H100) */

/* ---- loss path ----
 * marginal_counts: c_b / N of marginalize_log_probs + the mask normaliser
 *   (dalm/training/utils/train_utils.py:96-110,135-136). */
int dalm_b200_marginal_counts(const int64_t* gen_mask, const int64_t* qlen, int B, int L, float* cvec, float* nsum,
                              void* stream);
/* inbatch_loss_fwd_bwd: get_cosine_sim + get_nt_xent_loss(S) + get_nt_xent_loss(S^T), the doc log-prob
 *   log_softmax(S,1).diag() and the backward of all of them in ONE launch
 *   (train_utils.py:76-88,124; loop body dalm/training/rag_e2e/train_rage2e.py:441-446,
 *    dalm/training/retriever_only/train_retriever_only.py:371-373).
 *   losses[4] = {Lc, doc_term, Lc+doc_term, N}. cvec/nsum NULL => retriever-only (no marginal term). dQ/dP NULL => fwd only. */
int dalm_b200_inbatch_loss_fwd_bwd(const float* Q, const float* P, int B, int D, float logit_scale, const float* cvec,
                                   const float* nsum, float* S, float* dlp, float* losses, float* dQ, float* dP,
                                   float grad_out, void* stream);
/* ce_marginal_fwd_bwd: log_softmax over the vocabulary + gather + mask weights + d(logits)
 *   (train_utils.py:113-138). dtype 0 = bf16, 1 = fp32. dlogits may alias logits or be NULL. tok_lp: [B,L]. */
int dalm_b200_ce_marginal_fwd_bwd(const void* logits, void* dlogits, int dtype, const int64_t* ids, const int64_t* mask,
                                  const float* nsum, float* tok_lp, int B, int L, int V, long long ld, float grad_out,
                                  void* stream);
/* ce_marginal_rows: the same pass over token rows [row0, row0 + nrows) of the flattened [B*L] rows only; logits / dlogits
 *   point at row `row0` (a scratch holding just that chunk), tok_lp is still the whole [B,L] table. This is what lets the
 *   lm_head GEMM, the vocabulary CE and the head's dgrad run chunk by chunk over an L2-sized scratch, so the [B,L,V]
 *   logits of train_utils.py:113-138 (590 MB fp32 + three more copies in the reference) never exist in HBM. */
int dalm_b200_ce_marginal_rows(const void* logits, void* dlogits, int dtype, const int64_t* ids, const int64_t* mask,
                               const float* nsum, float* tok_lp, int B, int L, int V, long long ld, float grad_out,
                               int row0, int nrows, void* stream);
/* finalize_loss: out4 = {Lc, Lm, Lc+Lm, N}; combined_loss of train_rage2e.py:467. */
int dalm_b200_finalize_loss(const float* tok_lp, const int64_t* mask, int B, int L, const float* nsum,
                            const float* inbatch_losses, float* out4, void* stream);

/* small_matmul_f32: stand-alone get_cosine_sim forward / backward (train_utils.py:76-77) for callers that do not use the
 *   fused in-batch kernel. C[M,N] = alpha * opA(A) * opB(B), row-major fp32. */
int dalm_b200_small_matmul_f32(const float* A, const float* B, float* C, int M, int N, int K, int transA, int transB,
                               float alpha, void* stream);

/* ---- dropout (reference trains under model.train(): BERT hidden / attention-probability dropout 0.1, peft LoRA input
 * dropout 0.05). Counter-based Philox4x32-10 keyed by (seed, stream id, element index); masks are never stored, backward
 * kernels regenerate them. Entry points that can apply dropout take (drop_p, drop_seed, drop_stream_id, drop_offset):
 * drop_p = 0 disables it; drop_offset is an optional DEVICE uint64 added to the stream id (bumped once per step by
 * dalm_b200_bump_counter so that a CUDA-graph replay draws fresh masks). ---- */
int dalm_b200_bump_counter(void* counter, void* stream);
int dalm_b200_dropout_scale(float* out, long long n, float p, unsigned long long seed, unsigned long long stream_id,
                            const void* offset, void* stream);
/* dh[m,k] += mask(m,k)/(1-p) * sum_r G[m,r] A[r,k]: backward of the LoRA input dropout (the p = 0 case is folded into the
 * dgrad GEMM instead) */
int dalm_b200_lora_dx(void* dh, long long lddh, const void* G, long long ldg, const void* A, long long lda, int M, int K,
                      int R, float p, unsigned long long seed, unsigned long long stream_id, const void* offset,
                      void* stream);

/* ---- dense contractions (wgmma / TMA) ----
 * out[M,N] = act(alpha * A[M,K] B[N,K]^T + bias) + resid. Replaces every nn.Linear forward / dgrad reached through
 * dalm/models/rag_e2e_base_model.py:93,105 and dalm/models/retriever_only_base_model.py:58 (HF modeling code -> cuBLAS).
 * Either operand is read K-major or MN-major straight from its row-major buffer (nothing is transposed in HBM):
 *   layout 0: A[M,K], B[N,K]  "TN", both K-contiguous: forward y = x W^T, and dgrad against resident W^T copies
 *   layout 1: A[M,K], B[K,N]  dgrad dx = dy W against W[out,in] itself — full fine-tuning (reference default use_peft=None,
 *                             dalm/training/rag_e2e/train_rage2e.py:229-260,336) where weights change every step
 *   layout 2: A[K,M], B[K,N]  wgrad dW[out,in] = dy^T x, contraction over token rows (autograd of nn.Linear.weight) */
int dalm_b200_gemm_bf16(int layout, const void* A, long long lda, const void* B, long long ldb, void* out, long long ldo,
                        int out_f32, int M, int N, int K, float alpha, const float* bias, int act, const void* resid,
                        long long ldr, int resid_f32, int block_n, int max_ctas, float drop_p, unsigned long long drop_seed,
                        unsigned long long drop_stream_id, const void* drop_offset, void* stream);
/* LlamaMLP gate|up projection with SiLU(gate) * up fused into the epilogue: B = the gate / up weight rows interleaved in blocks of
 * 128 features ([gate blk | up blk | ...], N = 2F rows), so one 128 x 256 accumulator tile holds both halves of 128 features.
 * Writes gu[M, N] (interleaved, bf16: the backward's input) AND act[M, N/2] = silu(gate) * up (bf16). N % 256 == 0. Replaces
 * gate_proj / up_proj / act_fn of HF LlamaMLP reached through dalm/models/rag_e2e_base_model.py:105. */
int dalm_b200_gemm_bf16_swiglu(const void* A, long long lda, const void* B, long long ldb, void* gu, long long ldgu, void* act,
                               long long ldact, int M, int N, int K, void* stream);
/* fused q|k|v projection + rotary position embedding (HF rotate_half, head_dim 128) on output columns [0, rope_cols); cos / sin
 * fp32 [L, 64]; output row m is at position m % L. Replaces q_proj / k_proj / v_proj + apply_rotary_pos_emb of HF LlamaAttention.
 * bias: fp32 [N] or NULL (Qwen2's q/k/v biases): added to the fp32 accumulator before the rotation and the single bf16 rounding,
 * on every column; NULL leaves the results bit-identical to a bias-free projection. */
/* q_norm != NULL (Qwen3): every 128-column head of [0, rope_cols) is RMS-normalised before the rotation, all in fp32 before the
 * single bf16 store: x * rsqrt(mean(x^2) + eps) * w, with w = q_norm (fp32 [128]) on heads [0, nq_heads) and k_norm on the
 * rest. pre_out (bf16 [M, rope_cols], row stride ld_pre) receives the pre-norm columns (bias included) and rstd_out (fp32
 * [M, rope_cols / 128], row stride ld_rstd) each head's rstd, when non-NULL. q_norm == NULL requires k_norm, pre_out and
 * rstd_out NULL and computes exactly the norm-free projection. */
int dalm_b200_gemm_bf16_rope(const void* A, long long lda, const void* B, long long ldb, void* out, long long ldo, int M, int N,
                             int K, const float* bias, const float* cos_t, const float* sin_t, int L, int rope_cols,
                             const float* q_norm, const float* k_norm, int nq_heads, float eps, void* pre_out, long long ld_pre,
                             float* rstd_out, long long ld_rstd, void* stream);
/* gemm_bf16_gelu: pre[M,N] = A B^T + bias (bf16) AND act[M,N] = gelu_erf(pre) (bf16) from one launch: BertIntermediate
 * (dense + GELU, HF modeling_bert) / Falcon's dense_h_to_4h + act; the backward multiplies by gelu'(pre) inside the next dgrad
 * GEMM (gemm_bf16 with act = 2 and resid = pre), so neither direction runs a separate activation kernel. */
int dalm_b200_gemm_bf16_gelu(const void* A, long long lda, const void* B, long long ldb, void* pre, long long ldpre, void* act,
                             long long ldact, int M, int N, int K, const float* bias, void* stream);
void dalm_b200_gemm_clear_cache(void);
/* tile rasterisation of the persistent GEMM (tuning / test hook): -1 = m-fastest order, 0 = automatic (default: m-fastest
 * while A [M,K] stays L2-resident next to a bf16 output, else bands with a ~square wave footprint walked serpentine),
 * -2 = bands for every multi-wave problem, > 0 = bands of that many 128-row m-tiles. Env DALM_B200_GEMM_RASTER seeds it. */
void dalm_b200_gemm_set_raster(int group_m);
/* L2 eviction priorities on the GEMM's TMA traffic: -1 = automatic (default: mask 7 for multi-wave m-fastest problems whose
 * A operand stays L2-resident, else 0), or a bit mask applied to every launch: 1 = A loads evict_last, 2 = B loads evict_first,
 * 4 = output stores evict_first. Env DALM_B200_GEMM_L2_HINTS seeds it. Results never depend on it. */
void dalm_b200_gemm_set_l2_hints(int mask);

/* ---- attention (same call sites; HF eager/SDPA attention) ---- */
/* window: 0 = no window; > 0 = sliding window, counted in the padded row. Causal: query i sees key j iff
 * i - window < j <= i (Mistral; Qwen2 / Qwen3 with use_sliding_window). Bidirectional: iff |i - j| < window (ModernBERT's
 * local layers, window = local_attention / 2 + 1). Both combine with the key-padding mask; a query row that sees no key
 * gets output 0, lse = +inf and contributes nothing to dQ / dK / dV. Probability dropout is not built with a window. */
int dalm_b200_attention_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                            const int64_t* mask, void* out, long long ldo, float* lse, int B, int L, int Hq, int Hkv,
                            int D, float scale, int causal, int window, float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);
int dalm_b200_attention_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                            const int64_t* mask, const void* out, long long ldo, const float* lse, const void* d_out,
                            long long lddo, float* delta, void* dq, long long lddq, void* dk, long long lddk, void* dv,
                            long long lddv, int B, int L, int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);

/* wgmma / TMA attention (Hopper tensor cores): head_dim 128 (Llama decoder) or 64 (bge-large encoder incl.
 * attention-probability dropout; Falcon MQA decoder). Same arguments, outputs, mask semantics and dropout element indexing
 * as dalm_b200_attention_fwd / _bwd (the mma.sync kernels, kept for head_dim 32 and as a cross-check). */
int dalm_b200_attention_tc_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                               const int64_t* mask, void* out, long long ldo, float* lse, int B, int L, int Hq, int Hkv,
                               int D, float scale, int causal, int window, float drop_p, unsigned long long drop_seed,
                               unsigned long long drop_stream_id, const void* drop_offset, void* stream);
int dalm_b200_attention_tc_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                               const int64_t* mask, const void* out, long long ldo, const float* lse, const void* d_out,
                               long long lddo, float* delta, void* dq, long long lddq, void* dk, long long lddk, void* dv,
                               long long lddv, int B, int L, int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p,
                               unsigned long long drop_seed, unsigned long long drop_stream_id, const void* drop_offset,
                               void* stream);

/* ---- row-wise pieces of the encoder / decoder blocks ---- */
int dalm_b200_layernorm_fwd(const float* z, const float* gamma, const float* beta, float* y32, void* y16, long long ld16,
                            float* mean, float* rstd, int M, int H, float eps, float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);
int dalm_b200_layernorm_bwd(const float* z, const float* gamma, const float* mean, const float* rstd, const float* dy_f32,
                            const void* dy_bf16, long long ldb, float* dz32, void* dz16, long long ld16, int M, int H,
                            float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);
/* pre-LN blocks (Falcon): dz = LayerNorm-backward(dy) + dres, the gradient arriving around the norm; dres may alias dz32 */
int dalm_b200_layernorm_bwd_res(const float* z, const float* gamma, const float* mean, const float* rstd, const float* dy_f32,
                                const void* dy_bf16, long long ldb, const float* dres, float* dz32, void* dz16, long long ld16,
                                int M, int H, void* stream);
int dalm_b200_rmsnorm_fwd(const float* x, const float* g, void* h, long long ldh, float* rstd, int M, int H, float eps,
                          void* stream);
int dalm_b200_rmsnorm_bwd(const float* x, const float* g, const float* rstd, const void* dh, long long lddh,
                          const float* dres_in, float* dres_out, void* dres16, long long ld16, int M, int H, void* stream);
int dalm_b200_bert_embed(const int64_t* ids, const void* word, const void* pos, const void* type0, float* z, int M, int L,
                         int H, int V, void* stream);
/* RoBERTa / XLM-RoBERTa (HF create_position_ids_from_input_ids): position = pad_id + (id != pad_id) * (count of non-pad ids in
 * columns 0..l of the row), clamped into [0, P); z = word[id] + pos[position] + type0 (fp32, bert_embed's order of additions).
 * ids [B,L] dense; pos_ids_out int64 [B*L] (may be NULL) receives the positions. No allocation, no host synchronisation. */
int dalm_b200_roberta_embed(const int64_t* ids, const void* word, const void* pos, const void* type0, int pad_id, float* z,
                            int64_t* pos_ids_out, int B, int L, int H, int V, int P, void* stream);
int dalm_b200_embed_gather(const int64_t* ids, const void* table, float* x, int M, int H, int V, void* stream);
int dalm_b200_rope(void* buf, long long ld, int col0, int nheads, int D, const float* cos_t, const float* sin_t, int M,
                   int L, int backward, void* stream);
/* gu = [gate | up] of LlamaMLP. interleave == 0: columns [gate 0..F | up 0..F] (HF order); interleave == k: blocks of k features
 * alternate [gate blk | up blk | ...] (the layout dalm_b200_gemm_bf16_swiglu produces) */
int dalm_b200_swiglu_fwd(const void* gu, long long ldgu, void* act, long long lda, int M, int F, int interleave, void* stream);
int dalm_b200_swiglu_bwd(void* gu, long long ldgu, const void* dact, long long ldd, int M, int F, int interleave, void* stream);
/* x = [input | gate] = Wi(h).chunk(2) of ModernBertMLP (bf16 [M, 2F], any 16-byte-aligned row stride):
 * act = gelu_erf(input) * gate. The backward works in place, x <- [d_input | d_gate], fp32 math. */
int dalm_b200_geglu_fwd(const void* x, long long ldx, void* act, long long lda, int M, int F, void* stream);
int dalm_b200_geglu_bwd(void* x, long long ldx, const void* dact, long long ldd, int M, int F, void* stream);
int dalm_b200_gelu_fwd(const void* pre, long long ldp, void* act, long long lda, int M, int F, void* stream);
int dalm_b200_gelu_bwd(const void* pre, long long ldp, void* dact, long long ldd, int M, int F, void* stream);
/* mean_pooling + F.normalize (rag_e2e_base_model.py:96-97,108-111; retriever_only_base_model.py:60-68) */
int dalm_b200_pool_norm_fwd(const float* hidden, const int64_t* mask, float* pooled, float* emb, float* norm, int B, int L,
                            int H, int normalize, void* stream);
int dalm_b200_pool_norm_bwd(const float* emb, const float* norm, const float* d_emb, const int64_t* mask, float* d_hidden,
                            int B, int L, int H, int normalize, void* stream);

/* ---- LoRA (peft.LoraConfig r=8 alpha=16: rag_e2e_base_model.py:144-160) and optimizer (train_rage2e.py:336) ---- */
/* out0[r*so_r + k*so_k] += scale * sum_m G[m,r] X[m,k]  (r < 8; rows 8..15 of an R=16 call go to out1): dA = g^T x, dB^T = u^T dY */
int dalm_b200_lora_wgrad(const void* X, long long ldx, const void* G, long long ldg, float* out0, float* out1,
                         long long so_r, long long so_k, int M, int K, int R, float scale, float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);
/* out[M,R] (bf16) = X[M,K] . W[R,K]^T, R in {8,16}: LoRA down-projection u = x A^T and mid-gradient g = dY (sB) */
int dalm_b200_skinny_gemm(const void* X, long long ldx, const void* W, long long ldw, void* out, long long ldo, int M,
                          int K, int R, float drop_p, unsigned long long drop_seed,
    unsigned long long drop_stream_id, const void* drop_offset, void* stream);
int dalm_b200_pack_scaled_bf16(const float* in, long long si_r, long long si_c, void* out, long long ldo, int rows,
                               int cols, float scale, void* stream);
/* one launch for a whole table of pack jobs (device array of 56-byte records, see csrc/rowwise.cu PackEntry) */
int dalm_b200_pack_table(const void* table, int n_entries, void* stream);
int dalm_b200_cast_f32_bf16(const float* in, long long ldi, void* out, long long ldo, int rows, int cols, void* stream);
int dalm_b200_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                        float eps, int step, float grad_scale, void* stream);


/* ---- full fine-tuning: parameter gradients that are not GEMMs, and the optimizer over the fp32 master buffer ----
 * (autograd of nn.Linear.bias / nn.LayerNorm / LlamaRMSNorm / nn.Embedding under the reference's `accelerator.backward(loss)`,
 *  dalm/training/rag_e2e/train_rage2e.py:466, and torch.optim.Adam.step, :336,467)
 * col_reduce: out_sum[h] += sum_m dy[m,h]; out_prod[h] += sum_m dy[m,h] * (z[m,h] - mean[m]) * rstd[m]; dy = dy_f32 + dy_bf16
 * (either may be NULL), mean NULL for RMSNorm. */
int dalm_b200_col_reduce(const float* dy_f32, const void* dy_bf16, long long lddy, const float* z, const float* mean,
                         const float* rstd, float* out_sum, float* out_prod, int M, int H, void* stream);
/* dword[ids[m],:] += d[m,:]; dpos[pos_ids[m],:] += d[m,:] (dpos may be NULL; pos_ids NULL: position m % L). pad_id >= 0:
 * tokens with id == pad_id add nothing to dword and positions == pad_id nothing to dpos (nn.Embedding padding_idx); -1: none */
int dalm_b200_embed_scatter_add(const float* d, const int64_t* ids, const int64_t* pos_ids, float* dword, float* dpos, int M,
                                int H, int L, int V, int pad_id, void* stream);
/* out = (a_f32 + b_bf16) * dropout_scale  (gradient through the embedding dropout; out may alias a) */
int dalm_b200_masked_add(const float* a, const void* b, long long ldb, float* out, int M, int H, float p,
                         unsigned long long seed, unsigned long long stream_id, const void* offset, void* stream);
/* Adam on a flat fp32 buffer (n % 4 == 0) + refresh of the bf16 shadow the GEMMs read (shadow may be NULL) */
int dalm_b200_adam_step_shadow(float* p, const float* g, float* m, float* v, void* shadow_bf16, long long n, float lr,
                               float beta1, float beta2, float eps, int step, float grad_scale, void* stream);

/* ---- evaluation: exact maximum-inner-product top-k over the resident passage embeddings ----
 * replaces hnswlib.Index(space="ip").knn_query of dalm/eval/utils.py:18-66 (approximate: M=100, ef 100) with an exact
 * sweep. out_scores [nq,K] = inner products in descending order (hnswlib's distance is 1 - score), out_idx [nq,K] int32 row
 * ids (-1 past the end when N < K); ties -> lower row id first. workspace: dalm_b200_topk_ip_workspace(nq, K) bytes. */
long long dalm_b200_topk_ip_workspace(int nq, int K);
int dalm_b200_topk_ip(const float* Q, const float* P, long long ldp, int nq, int N, int D, int K, float* out_scores,
                      int* out_idx, void* workspace, void* stream);

/* ---- use_bnb: NF4 quantise -> dequantise of a weight, in place, at load time ----
 * what BitsAndBytesConfig(load_in_4bit, nf4, compute bf16) makes the matmuls see (dalm/models/rag_e2e_base_model.py:136-142,
 * retriever_only_base_model.py:85-91): fp16 cast, blocks of 64, absmax, 16 NormalFloat levels, dequantised to fp16.
 * codes (uint8 [n]) / absmax (fp32 [ceil(n/64)]) are optional outputs. */
int dalm_b200_nf4_roundtrip(float* w, long long n, void* codes, float* absmax, void* stream);
/* 4-bit STORAGE of the same quantisation (what bitsandbytes' Linear4bit keeps resident): nf4_quantize packs two codes per byte
 * (first element in the high nibble) + fp32 absmax per block of 64; nf4_dequant_bf16 expands a [rows, cols] weight (cols % 64
 * == 0) to bf16(fp16(code * absmax)) right before the GEMM that reads it - bnb's dequantize_4bit -> matmul forward - and copies
 * an optional bf16 tail (the LoRA block of a K-augmented weight) behind each row. */
int dalm_b200_nf4_quantize(const float* w, long long n, void* packed, float* absmax, void* stream);
int dalm_b200_nf4_dequant_bf16(const void* packed, const float* absmax, long long rows, int cols, void* out, long long ldo,
                               const void* tail, long long ldt, int tail_cols, void* stream);

/* ---- evaluation: greedy autoregressive decoding of the generator ----
 * replaces `model.generate(**inputs, max_length=max_length, early_stopping=True)` of run_generator_on_prompts
 * (dalm/eval/eval_rag.py:126-140; HF GenerationMixin greedy search with a KV cache).
 * rope_pos: RoPE at explicit position ids pos[M] (HF generate: cumsum(attention_mask) - 1), tables cos/sin [T, D/2].
 * attention_decode: one query token per sequence (row b of qkv: q | k | v at the given columns, already rotated) against
 *   the bf16 KV cache [B][T][Hkv*D] (batch stride cache_sb, token stride cache_st, in elements); keys t < cur are visible
 *   iff mask[b*ldm + t] != 0, the token itself (column cur) always; its K / V rows are appended to the cache at column cur.
 *   window > 0: only columns t > cur - window are visible (the sliding window of the training kernels).
 * greedy_step: next token = argmax(logits[b, 0..V)) for unfinished rows, pad_id for finished ones; writes tokens[b, col],
 *   mask[b, col] = 1, next_ids[b], pos[b] += 1; a row finishes when it emits one of eos_ids; alive[col] += #unfinished
 *   rows after this step (alive: int32 [T], zeroed by the caller).
 * Device-column mode (cur_dev != NULL, int32 [B]): attention_decode takes cur = cur_dev[b], greedy_step writes column
 *   cur_dev[b] + 1 and advances cur_dev[b]; the host `cur` / `col` arguments are ignored, so the launch sequence of a
 *   decode step has identical arguments for every token and can be captured once in a CUDA graph and replayed. */
/* decode_gemm: out[M,N] = act(A[M,K] W[N,K]^T + bias) + resid for the M <= 16 token rows of a decode step (every nn.Linear of
 *   the generator once per generated token): weight-streaming mma.sync kernel, each weight read once. act 0 none / 1 gelu;
 *   bias fp32 [N] or NULL; out / resid bf16 or fp32 (resid may be NULL). Same order of operations as gemm_bf16. */
int dalm_b200_decode_gemm(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldo, int out_f32,
                          const float* bias, const void* resid, long long ldr, int resid_f32, int act, int M, int N, int K,
                          void* stream);
int dalm_b200_rope_pos(void* buf, long long ld, int col0, int nheads, int D, const float* cos_t, const float* sin_t,
                       const int64_t* pos, int M, int T, void* stream);
/* qk_norm_rope: Qwen3's per-head q/k RMSNorm followed by RoPE (head_dim 128, HF rotate_half), in place on heads [0, nheads) of
 * a token-major bf16 buffer [M, ld] (heads [0, nq_heads) use q_norm, the rest k_norm; both fp32 [128]). Position of row m:
 * clamp(pos[m], 0, T-1) when pos != NULL, else m % L; cos / sin fp32 [T, 64]. pre (bf16, ld_pre) and rstd (fp32 [M, nheads],
 * ld_rstd) optionally receive the pre-norm values and each head's rstd. No allocation, no host synchronisation.
 * qk_norm_rope_bwd: in place on d(out) of the same heads (positions m % L): un-rotates, then the RMSNorm backward from the
 * saved pre / rstd, dx = rstd (w dy - x_hat mean(w dy x_hat)), x_hat = pre rstd; dw_q / dw_k (fp32 [128], both or neither)
 * accumulate sum(dy x_hat) over rows and heads with atomics. */
int dalm_b200_qk_norm_rope(void* buf, long long ld, int nheads, int nq_heads, const float* q_norm, const float* k_norm, float eps,
                           const float* cos_t, const float* sin_t, int T, int L, const int64_t* pos, int M, void* pre,
                           long long ld_pre, float* rstd, long long ld_rstd, void* stream);
int dalm_b200_qk_norm_rope_bwd(void* dbuf, long long ld, int nheads, int nq_heads, const float* q_norm, const float* k_norm,
                               const float* cos_t, const float* sin_t, int L, const void* pre, long long ld_pre, const float* rstd,
                               long long ld_rstd, int M, float* dw_q, float* dw_k, void* stream);
int dalm_b200_attention_decode(const void* qkv, long long ldq, int q_col, int k_col, int v_col, void* cache_k, void* cache_v,
                               long long cache_sb, long long cache_st, const int64_t* mask, long long ldm, void* out,
                               long long ldo, int B, int Hq, int Hkv, int D, int cur, const int* cur_dev, int T, float scale,
                               int window, void* stream);
int dalm_b200_greedy_step(const void* logits, long long ld, int B, int V, const int64_t* eos_ids, int n_eos,
                          long long pad_id, int* unfinished, int64_t* tokens, long long ldt, int64_t* mask, long long ldm,
                          int col, int* cur_dev, int T, int64_t* next_ids, int64_t* pos, int* alive, void* stream);
/* sample_step: greedy_step with the token drawn instead of taken by argmax (HF _sample, do_sample=True), same arguments and
 * the same bookkeeping after the choice. The warpers run in HF's order on fp32 scores x = float(logit) / temperature
 * (IEEE division, so kept scores equal HF's bit for bit):
 *   top-k (0 < top_k < V; 0 or >= V is off): remove x < the k-th largest x; ties at the k-th value are all kept;
 *   top-p (top_p < 1): order the survivors ascending by (x, index) and remove while the cumulative softmax share is
 *     <= 1 - top_p, always keeping the last one. HF sorts with an unstable sort; the (x, index) order is this library's
 *     deterministic rule for a tie group that straddles the cut;
 *   draw: u in [0, 1) from Philox keyed by seed with counter (column, row) -- the same token for an eager launch and a CUDA
 *     graph replay; the token is the first kept index, ascending, whose inclusive prefix sum of exp(x - max) exceeds u * Z
 *     (prefix sums and Z in fp64).
 * Requires temperature > 0 and finite, 0 < top_p <= 1, top_k >= 0, V <= 2^20. Test hooks (NULL in production): u
 * (fp64 [B]) replaces the Philox draw; scores_out (fp32, row stride ld) receives the warped scores of every unfinished row,
 * -inf where a token was removed. Finished rows emit pad_id and are not scored. */
int dalm_b200_sample_step(const void* logits, long long ld, int B, int V, const int64_t* eos_ids, int n_eos,
                          long long pad_id, int* unfinished, int64_t* tokens, long long ldt, int64_t* mask, long long ldm,
                          int col, int* cur_dev, int T, int64_t* next_ids, int64_t* pos, int* alive, float temperature,
                          int top_k, float top_p, unsigned long long seed, const double* u, float* scores_out, void* stream);


/* ---- routed mixture-of-experts MLP (Qwen3-MoE Qwen3MoeSparseMoeBlock: softmax router, top-k, SwiGLU experts) ----
 * The experts run as grouped GEMMs over rows permuted so that each expert's (token, slot) pairs are contiguous, in pair order
 * (by token, then slot), each segment padded to the 128-row M tile. Nothing needs a host synchronisation: the live M-tile
 * count stays in device memory and every launch is sized for the static bound of n_tiles = ceil((P + 127 E) / 128) tiles,
 * P = M k pairs. No floating-point atomics: every result is the same bits from run to run.
 * gemm_bf16_grouped: out[M,N] (bf16) = A[M,K] B[e]^T (layout 0, B dense [E, N, K]) or A[M,K] B[e] (layout 1, B dense
 *   [E, K, N], K % 64 == 0: the down / gate|up dgrads read the forward weights, no transposed copy), e = tile_expert[m / 128];
 *   only the first *live_tiles M tiles run. swiglu = 1 (layout 0, N % 256 == 0): B[e]'s gate / up rows interleaved in
 *   128-feature blocks, out = gate|up and out2 [M, N/2] = silu(gate) * up, as gemm_bf16_swiglu. max_ctas: 0 = all SMs. */
int dalm_b200_gemm_bf16_grouped(int layout, int swiglu, const void* A, long long lda, const void* B, int E, void* out,
                                long long ldo, void* out2, long long ldo2, int M, int N, int K, const int* tile_expert,
                                const int* live_tiles, int max_ctas, void* stream);
/* moe_router: fp32 logits [M, E] (row stride ld) -> softmax (fp32) -> top-k by logit (descending, ties to the lower index):
 *   ids int32 [M, k], w fp32 [M, k] = the probabilities, divided by their sum when norm_topk. E <= 256, k <= min(E, 16). */
int dalm_b200_moe_router(const float* logits, long long ld, int M, int E, int k, int norm_topk, int* ids, float* w, void* stream);
/* moe_router_bwd: dlogits (bf16 [M, E], row stride ldd) from dw (fp32 [M, k]) through the renormalisation, the top-k
 *   selection (ids) and the softmax, recomputed from the logits. */
int dalm_b200_moe_router_bwd(const float* logits, long long ld, const int* ids, const float* w, const float* dw, int M, int E,
                             int k, int norm_topk, void* dlogits, long long ldd, void* stream);
/* moe_permute: ids int32 [P] -> counts [E], seg_off [E + 1] (padded row offsets), tile_expert [n_tiles] (-1 after the live
 *   tiles), live [1] (live M tiles), pair_row [P] (row of each pair; -1 for an id outside [0, E)), row_pair [128 n_tiles]
 *   (pair of each live row, -1 on padding rows). chunk_counts: int32 workspace [ceil(P / 1024) E]. */
int dalm_b200_moe_permute(const int* ids, int P, int E, int n_tiles, int* chunk_counts, int* counts, int* seg_off,
                          int* tile_expert, int* live, int* pair_row, int* row_pair, void* stream);
/* moe_gather: out[r] (bf16 [n_rows, H]) = x[row_pair[r] / k] (bf16, or fp32 when x_f32), 0 on padding rows; rows from
 *   128 *live on are not written. */
int dalm_b200_moe_gather(const void* x, long long ldx, int x_f32, int H, const int* row_pair, int k, const int* live, int n_rows,
                         void* out, long long ldo, void* stream);
/* moe_combine: out[t] = resid[t] + sum_s w[t, s] y[pair_row[t, s]] in fp32, slots in order; y bf16 [rows, H]; resid / out
 *   fp32 when f32 else bf16 [M, H], resid may alias out or be NULL; w NULL = weights of 1 (the sum of a token's k rows of
 *   the gate|up dgrad). */
int dalm_b200_moe_combine(const void* y, long long ldy, const int* pair_row, const float* w, int M, int k, int H, const void* resid,
                          long long ldr, void* out, long long ldo, int f32, void* stream);
/* moe_down_bwd: per pair p with row r = pair_row[p]: dw[p] = <da[r], act[r]> (fp32) and d_act[r] = w[p] da[r] (bf16; d_act may
 *   be act itself), where
 *   da = dy_rows W_down[e] is the down projection's dgrad of the token's unweighted output gradient. */
int dalm_b200_moe_down_bwd(const void* da, long long ldda, const void* act, long long ldact, const int* pair_row, const float* w,
                           int P, int I, float* dw, void* d_act, long long ldd, void* stream);
#ifdef __cplusplus
}
#endif
#endif /* DALM_B200_H */
