/* b2_ddp_bert.h — C ABI of libb2ddpbert.so: the sm_90a (H100) kernels behind the DDP BERT fine-tuning step.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference (taishan1994/pytorch-distributed-NLP) has no
 * native code; the work these entry points replace is issued by third-party Python modules that
 * `multi-gpu-distributed-cls.py` drives.  Each declaration cites the reference-side call it stands in for
 * (paths relative to the reference tree, or `SP/` = site-packages of the pinned dependencies).
 *
 * Conventions
 *   - plain C: device pointers (borrowed; the library never allocates tensors), int64 sizes, explicit stream
 *     (`cudaStream_t` passed as void*).  No torch types.  No CPU fallback of any kind.
 *   - every function returns 0 on success, negative on error; `b2_last_error()` returns a thread-local message.
 *     The Python host turns a non-zero status into `RuntimeError(b2_last_error())`.
 *   - re-entrant: forward runs on the main thread, backward / DDP hooks on the autograd thread.
 *   - bf16 activations / weights / gradients, fp32 accumulation and statistics, fp32 master weights and
 *     AdamW moments.
 */
#ifndef B2_DDP_BERT_H_
#define B2_DDP_BERT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------ */
/* library                                                                                                */
/* ------------------------------------------------------------------------------------------------------ */
const char* b2_last_error(void);
int32_t b2_abi_version(void);             /* bumped when a struct below changes */
#define B2_ABI_VERSION 23
int64_t b2_launch_count(void);            /* kernels launched by this library so far (process-wide) */

/* ------------------------------------------------------------------------------------------------------ */
/* GEMM (wgmma + TMA)                                                                                     */
/*   replaces: cuBLAS addmm issued by SP/transformers/models/bert/modeling_bert.py:179-181 (Q,K,V),       */
/*   :295 (attention output dense), :340 (intermediate dense), :353 (output dense) and the dgrad/wgrad    */
/*   GEMMs autograd runs for them inside `loss.backward()` (multi-gpu-distributed-cls.py:173).            */
/* ------------------------------------------------------------------------------------------------------ */
enum { B2_MAJOR_K = 0, B2_MAJOR_MN = 1 };
enum {
  B2_EPI_NONE = 0,                  /* D = acc                                  (dgrad / wgrad)               */
  B2_EPI_BIAS = 1,                  /* D = acc + bias[n]                        (QKV projection)              */
  B2_EPI_BIAS_GELU = 2,             /* aux_out = acc + bias; D = gelu_erf(aux_out)   (BertIntermediate)       */
  B2_EPI_BIAS_DROPOUT_RESIDUAL = 3, /* D = dropout(acc + bias) + aux_in         (BertSelfOutput / BertOutput) */
  B2_EPI_RESIDUAL = 4,              /* D = acc + aux_in                         (dgrad joining a residual)    */
  B2_EPI_GELU_BWD = 5,              /* D = acc * gelu_erf'(aux_in)              (dgrad through GELU)          */
  B2_EPI_RESIDUAL_F32 = 6,          /* D(fp32) = acc + aux_in(fp32); ldd / ld_aux_in count fp32 elements      */
  B2_EPI_ACCUM_F32 = 7,             /* D(fp32) += acc (vector reductions at L2; D holds the residual stream;   */
                                    /* split-K slices add in place, summation order unspecified)               */
  B2_EPI_PARTIAL_F32 = 100          /* internal: split-K partials                                           */
};

typedef struct b2_gemm_args {
  int64_t M, N, K;        /* D is [M,N]; K is the contraction length                                         */
  const void* A;          /* bf16. a_major K : A[m*lda + k];  MN : A[k*lda + m]                              */
  int64_t lda;
  int32_t a_major;
  const void* B;          /* bf16. b_major K : B[n*ldb + k];  MN : B[k*ldb + n]                              */
  int64_t ldb;
  int32_t b_major;
  /* Every leading dimension covers the row it describes: lda >= K (a_major K) or >= M (MN); ldb >= K (K) or
     >= N (MN); ldd >= N; ld_aux_in / ld_aux_out >= N where the epilogue reads / writes them (not read otherwise). */
  void* D;                /* bf16 [M, ldd]                                                                   */
  int64_t ldd;
  int32_t epilogue;
  const void* bias;       /* bf16 [N], 16-byte aligned: required by (1,2,3), must be NULL otherwise           */
  const void* aux_in;     /* bf16 [M, ld_aux_in]: residual (3,4) or saved pre-activation (5); fp32 for (6);
                             16-byte aligned; required by (3,4,5,6)                                          */
  int64_t ld_aux_in;
  void* aux_out;          /* bf16 [M, ld_aux_out], 16-byte aligned: pre-activation saved by (2); required by (2),
                             must be NULL otherwise                                                          */
  int64_t ld_aux_out;
  float dropout_p;        /* [0, 1) for (3); must be 0 otherwise                                             */
  const void* rng_state;  /* device uint64[2] = {seed, step}; see b2_rng_*.  Required by (3) with p > 0; may be
                             set (and is not read) otherwise                                                 */
  uint32_t rng_site;      /* distinct per dropout site                                                       */
  void* workspace;        /* fp32 scratch for split-K of (0) (may be NULL -> never split; may be set on
                             problems that do not split)                                                     */
  int64_t workspace_bytes;
  int32_t force_bn;       /* 0 = auto, else 128 / 256 (tests, tuning)                                        */
  int32_t force_splits;   /* 0 = auto, else >= 1; > 1 needs (7), or (0) with a workspace of force_splits*M*N*4
                             bytes and no colsum_out                                                         */
  int32_t force_kernel;   /* kernel choice (tests, tuning); the H100 build has one GEMM kernel and ignores it       */
  void* debug_timing;     /* unused (may be set, is not read)                                                     */
  float* colsum_out;      /* NULL, or fp32 [N]: += column sums of the (bf16-rounded) output D, by atomic add.  Only
                             with the bf16-output epilogues (0-5); a problem with it is never split               */
} b2_gemm_args_t;

int32_t b2_gemm_bf16(const b2_gemm_args_t* args, void* stream);

/* `count` independent problems behind one launch where they allow it (all TN = both operands MN-major, plain bf16
 * output, N % 256 == 0, one K; at most 4): the four weight-gradient GEMMs of an encoder layer (autograd's
 * addmm backward nodes for BertSelfAttention/BertSelfOutput/BertIntermediate/BertOutput, modeling_bert.py:179-356).
 * Other mixes are issued one by one; results are identical either way.                                         */
int32_t b2_gemm_bf16_grouped(const b2_gemm_args_t* args, int32_t count, void* stream);

/* BertSelfOutput.forward / BertOutput.forward in ONE launch (SP/transformers/models/bert/modeling_bert.py:294-298,
 * :352-356): y = LayerNorm(dropout(x W^T + b) + residual).  `args` as for b2_gemm_bf16 with epilogue
 * B2_EPI_BIAS_DROPOUT_RESIDUAL, NT layouts, N = hidden in {768, 1024} -- EXCEPT that args->aux_in is the residual as
 * FP32 [M, N] (ld_aux_in in elements): the residual stream stays in fp32 end to end.  D receives the pre-LayerNorm sum
 * rounded to bf16 (kept for the backward), y the normalised output as bf16 (the next GEMM's operand), y_f32 (optional)
 * the same as fp32 (the next block's residual), mean / rstd (fp32 [M]) the row statistics -- computed from the
 * UNROUNDED fp32 sum.  A row's N columns are spread over a cluster of N / 256 CTAs; the row statistics travel
 * through distributed shared memory.  Leading dimensions as for b2_gemm_bf16 (lda, ldb >= K; ldd, ld_aux_in >= N),
 * and ldy >= N, ldyf >= N when y_f32 is set.  Rejected, because the kernel would not honour them: colsum_out,
 * aux_out, force_splits > 1, force_bn other than 0 / 256, a workspace.  force_kernel and debug_timing are accepted
 * and not read.
 * b2_gemm_ln_max_clusters(hidden): how many such clusters the device can hold at once (0 = shape / device not
 * supported: issue b2_gemm_bf16 + b2_layernorm_fwd instead).                                                    */
int32_t b2_gemm_ln_fwd(const b2_gemm_args_t* args, const void* gamma, const void* beta, float eps, void* y,
                       int64_t ldy, float* y_f32, int64_t ldyf, float* mean, float* rstd, void* stream);
int32_t b2_gemm_ln_max_clusters(int64_t hidden);

/* ------------------------------------------------------------------------------------------------------ */
/* memory-bound kernels                                                                                   */
/* ------------------------------------------------------------------------------------------------------ */

/* BertEmbeddings.forward (SP/transformers/models/bert/modeling_bert.py:72-112): word + position + token-type
 * gather, add, LayerNorm(eps), dropout.  ids are the int64 tensors the reference's Collate produces
 * (multi-gpu-distributed-cls.py:88-97).  Writes y (bf16 [rows,H]), the pre-LN sum (bf16, for backward),
 * mean/rstd (fp32 [rows]) and ids32/tt32 (int32 copies used by the backward scatter).                      */
int32_t b2_embed_fwd(const int64_t* input_ids, const int64_t* token_type_ids, int64_t batch, int64_t seq,
                     const void* word_emb, const void* pos_emb, const void* type_emb, const void* gamma,
                     const void* beta, int64_t hidden, int64_t vocab, int64_t type_vocab, float eps, float dropout_p,
                     const void* rng_state, uint32_t rng_site, void* y, float* y_f32 /* optional fp32 copy of y: first residual of the fp32 stream */, void* pre_ln, float* mean, float* rstd,
                     int32_t* ids32, int32_t* tt32, void* stream);

/* arms the owner table used by b2_embed_bwd (int32[vocab] = INT_MAX); call once after allocation */
int32_t b2_embed_owner_init(int32_t* owner, int64_t vocab, void* stream);

/* backward of the above: LN backward, then the three scatter-adds.  Word rows are keyed by an owner token per
 * touched vocabulary row; when the scratch holds [tokens + seq * type_vocab][hidden] fp32 (and type_vocab <= 3) every
 * token adds its row into the owner's fp32 accumulator with L2 reductions, so the summation order of a row that
 * occurs more than once varies from run to run.  Otherwise one owner CTA sums the duplicates in token order.
 * d_word must be zeroed by the caller (b2_zero).  The row `pad_token_id` gets no gradient (nn.Embedding padding_idx
 * semantics, modeling_bert.py:58).  b2_embed_bwd_ordered: the same, with the word rows always summed by the owner
 * CTA in token order: bitwise reproducible (torch.use_deterministic_algorithms).  Its fused position / token-type pass
 * needs seq * type_vocab * hidden fp32 of scratch.                                                        */
int32_t b2_embed_bwd(const void* dy /* bf16, or fp32 when dy_fp32 */, int32_t dy_fp32, const void* pre_ln, const float* mean, const float* rstd, const void* gamma,
                     const int32_t* ids32, const int32_t* tt32, int64_t batch, int64_t seq, int64_t hidden,
                     int64_t vocab, int64_t type_vocab, int64_t pad_token_id /* -1: none */, float dropout_p,
                     const void* rng_state, uint32_t rng_site, void* d_word, void* d_pos, void* d_type, void* d_gamma, void* d_beta, void* scratch_dx,
                     float* scratch_partials, int64_t scratch_partials_bytes, int32_t* owner, void* stream);
int32_t b2_embed_bwd_ordered(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean, const float* rstd,
                             const void* gamma, const int32_t* ids32, const int32_t* tt32, int64_t batch, int64_t seq,
                             int64_t hidden, int64_t vocab, int64_t type_vocab, int64_t pad_token_id, float dropout_p,
                             const void* rng_state, uint32_t rng_site, void* d_word, void* d_pos, void* d_type,
                             void* d_gamma, void* d_beta, void* scratch_dx, float* scratch_partials,
                             int64_t scratch_partials_bytes, int32_t* owner, void* stream);

/* LayerNorm over the last dim (BertSelfOutput / BertOutput LayerNorm, modeling_bert.py:297,355).
 * x is the already-summed (dropout(dense)+residual) input produced by the GEMM epilogue.                   */
int32_t b2_layernorm_fwd(const void* x, const void* gamma, const void* beta, int64_t rows, int64_t hidden,
                         float eps, void* y, float* mean, float* rstd, void* stream);

/* LayerNorm backward.  dy: grad wrt LN output.  Produces
 *   dx        grad wrt LN input (goes to the residual branch),
 *   dx_drop   dx * dropout-mask / (1-p) of the dense output that fed this LN (NULL when p == 0: use dx),
 *   d_gamma, d_beta, d_bias (bias grad of that dense = column sums of dx_drop)  — all bf16 [hidden].
 * `dy_add` (optional) is added to dy first (second consumer of the LN output, e.g. a residual path).       */
int32_t b2_layernorm_bwd(const void* dy, const void* dy_add, const void* x, const float* mean, const float* rstd,
                         const void* gamma, int64_t rows, int64_t hidden, float dropout_p, const void* rng_state,
                         uint32_t rng_site, int32_t grad_fp32 /* 1: dy, dy_add, dx are fp32 (dx_drop stays bf16 and
                         is then always written: it is what the GEMMs consume) */,
                         void* dx, void* dx_drop, void* d_gamma, void* d_beta, void* d_bias,
                         float* scratch_partials, int64_t scratch_partials_bytes,
                         int32_t* deferred_nparts /* host pointer or NULL.  NULL: d_gamma/d_beta/d_bias are final in
                         stream order.  Else only the per-block partials are written, *deferred_nparts receives their
                         count and the caller finishes with b2_colsum_finish (takes the reduction off the critical
                         path, e.g. onto another stream) */,
                         void* stream);

/* The training engine's form of b2_layernorm_bwd (fp32 gradient stream: dy fp32 in, dx fp32 out, dx_drop bf16 out,
 * dropout mask on the input branch): the three column-sum sets are ADDED into accum (fp32 [3][hidden]: d_gamma,
 * d_beta, d_bias) instead of going through partials + b2_colsum_finish; the caller converts them with
 * b2_accum_finish.                                                                                             */
int32_t b2_layernorm_bwd_accum(const float* dy, const void* x, const float* mean, const float* rstd,
                               const void* gamma, int64_t rows, int64_t hidden, float dropout_p,
                               const void* rng_state, uint32_t rng_site, float* dx, void* dx_drop, float* accum,
                               void* stream);

/* partials [nparts][nsets][cols] fp32 -> up to three bf16 [cols] outputs (the second half of b2_layernorm_bwd) */
int32_t b2_colsum_finish(const float* partials, int32_t nparts, int32_t nsets, int64_t cols, void* out0, void* out1,
                         void* out2, void* stream);

/* column sums of a bf16 [rows, cols] matrix -> bf16 [cols]   (bias gradients of QKV / intermediate dense)  */
int32_t b2_colsum(const void* x, int64_t rows, int64_t cols, int64_t ldx, void* out, float* scratch_partials,
                  int64_t scratch_partials_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* attention (BertSelfAttention core, modeling_bert.py:115-140 eager_attention_forward + :206 head merge)    */
/*   qkv  bf16 [batch*seq, 3*hidden]  (Q | K | V column blocks, heads of 64 inside each)                    */
/*   mask int64 [batch, seq] of {0,1} as produced by the reference Collate, or NULL (= all ones)            */
/*   ctx  bf16 [batch*seq, hidden]    lse fp32 [batch, heads, seq]                                          */
/*   lse  natural-log log-sum-exp of each query row's masked, scaled scores, for the backward.  A row with no */
/*        visible key (all-zero mask row) gets finfo(fp32).min * ln2 (~ -2.4e38, below -1e38 as no row with  */
/*        a visible key can be): HF's softmax is uniform there (every score is finfo.min), ctx = mean of V,  */
/*        and the backward recognises the value and gives every key P = 1/seq.                               */
/*   keep_bits  NULL, or uint64 [batch, heads, seq, seq/64]: cache of the forward's dropout decisions; used  */
/*              (written by fwd, read by bwd instead of regenerating Philox) when seq == 128 and dropout_p > 0,*/
/*              ignored otherwise.  Pass the same buffer to both calls of a step, or NULL to both.            */
/* ------------------------------------------------------------------------------------------------------ */
int32_t b2_attention_fwd(const void* qkv, const int64_t* attention_mask, int64_t batch, int64_t seq,
                         int64_t heads, int64_t head_dim, float dropout_p, const void* rng_state,
                         uint32_t rng_site, void* ctx, float* lse, uint64_t* keep_bits, void* stream);
int32_t b2_attention_bwd(const void* qkv, const int64_t* attention_mask, const void* ctx, const void* d_ctx,
                         const float* lse, int64_t batch, int64_t seq, int64_t heads, int64_t head_dim,
                         float dropout_p, const void* rng_state, uint32_t rng_site, void* d_qkv,
                         float* dq_accum /* fp32 [batch*seq, hidden], only for seq > 128 */,
                         float* dbias_accum /* NULL, or fp32 [3*hidden]: += column sums of d_qkv (QKV bias grad) */,
                         const uint64_t* keep_bits, void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* head: BertPooler (modeling_bert.py:462-468) + dropout + classifier (:1123-1124) + CrossEntropyLoss       */
/*   (multi-gpu-distributed-cls.py:169,343).  fp32 logits/loss as the reference exposes them.               */
/* ------------------------------------------------------------------------------------------------------ */
int32_t b2_head_fwd(const void* hidden_states /* bf16 [batch*seq, hidden] */, int64_t batch, int64_t seq,
                    int64_t hidden, const void* pool_w, const void* pool_b, const void* cls_w, const void* cls_b,
                    int64_t num_labels, float dropout_p, const void* rng_state, uint32_t rng_site,
                    void* pooled /* bf16 [batch, hidden] */, float* logits /* [batch, num_labels] */,
                    void* stream);
/* mean cross-entropy and d(loss)/d(logits); labels int64 [batch]; loss_scale multiplies dlogits (DDP: 1)    */
int32_t b2_ce_fwd_bwd(const float* logits, const int64_t* labels, int64_t batch, int64_t num_labels,
                      float* loss /* scalar */, float* dlogits /* [batch, num_labels] or NULL */, void* stream);
/* the losses of HF's three problem types and the options of torch's CrossEntropyLoss, all with reduction "mean":   */
/*   B2_LOSS_CE   CrossEntropyLoss(weight, ignore_index, label_smoothing)   labels int64 [batch]                    */
/*   B2_LOSS_MSE  MSELoss()                                                  labels fp32 [batch, num_labels]         */
/*   B2_LOSS_BCE  BCEWithLogitsLoss(pos_weight)                              labels fp32 [batch, num_labels]         */
/* CE with the defaults (no weight, ignore_index -100, no smoothing) computes exactly what b2_ce_fwd_bwd does.      */
/* A degenerate CE batch (every row ignored, or zero total weight) gives loss nan and dlogits 0.                    */
enum { B2_LOSS_CE = 0, B2_LOSS_MSE = 1, B2_LOSS_BCE = 2 };
typedef struct b2_loss_params {
  const float* weight;       /* CE: device fp32 [num_labels] class weights, or NULL                              */
  const float* pos_weight;   /* BCE: device fp32 [num_labels], or NULL                                           */
  int64_t ignore_index;      /* CE: rows with this label count for nothing (torch's default -100)                */
  float label_smoothing;     /* CE: in [0, 1]                                                                    */
} b2_loss_params_t;
int32_t b2_loss_fwd_bwd(const float* logits, const void* labels, int64_t batch, int64_t num_labels, int32_t mode,
                        const b2_loss_params_t* params /* NULL: the defaults */, float* loss /* scalar */,
                        float* dlogits /* [batch, num_labels] or NULL */, void* stream);
/* backward of b2_head_fwd: from dlogits to d(hidden_states[:,0]) and the four head parameter grads (bf16)  */
int32_t b2_head_bwd(const float* dlogits, const void* hidden_states, const void* pooled, int64_t batch,
                    int64_t seq, int64_t hidden, const void* pool_w, const void* cls_w, int64_t num_labels,
                    float dropout_p, const void* rng_state, uint32_t rng_site, void* d_pool_w, void* d_pool_b,
                    void* d_cls_w, void* d_cls_b, void* d_hidden /* [batch*seq, hidden], rows != CLS zeroed */,
                    int32_t d_hidden_fp32 /* 0: bf16, 1: fp32 */, float* scratch /* fp32 [2, batch, hidden] */,
                    void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* packed bins (SURVEY.md §8 f3): the reference tokenises with padding="max_length" (multi-gpu-distributed-cls.py */
/* :76) although its rows average 18 of 128 tokens.  The host packs the valid prefixes of several sequences into  */
/* 128-token bins (pytorch-distributed-nlp_b200/packing.py); these variants of the entry points above take        */
/*   position_ids  int64 [bins * 128]   position of every token inside its own sequence                           */
/*   segments      int32 [bins * 128]   lo | hi << 16: the row may attend to rows [lo, hi) of its bin only        */
/*   cls_rows      int64 [batch]        flat row of every sequence's first token (what the pooler reads)          */
/* Everything else (GEMMs, LayerNorm, GELU) is token-wise and simply runs on bins * 128 rows.                     */
/* ------------------------------------------------------------------------------------------------------ */
int32_t b2_embed_fwd_packed(const int64_t* input_ids, const int64_t* token_type_ids, const int64_t* position_ids,
                            int64_t max_positions, int64_t bins, int64_t seq, const void* word_emb,
                            const void* pos_emb, const void* type_emb, const void* gamma, const void* beta,
                            int64_t hidden, int64_t vocab, int64_t type_vocab, float eps, float dropout_p,
                            const void* rng_state, uint32_t rng_site, void* y, float* y_f32, void* pre_ln, float* mean,
                            float* rstd, int32_t* ids32, int32_t* tt32, int32_t* pos32, void* stream);
int32_t b2_embed_bwd_packed(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean, const float* rstd,
                            const void* gamma, const int32_t* ids32, const int32_t* tt32, const int32_t* pos32,
                            int64_t bins, int64_t seq, int64_t hidden, int64_t vocab, int64_t type_vocab,
                            int64_t pad_token_id, float dropout_p, const void* rng_state, uint32_t rng_site,
                            void* d_word, void* d_pos, void* d_type, void* d_gamma, void* d_beta, void* scratch_dx,
                            float* scratch_partials, int64_t scratch_partials_bytes, int32_t* owner, void* stream);
int32_t b2_attention_fwd_packed(const void* qkv, const int32_t* segments, int64_t bins, int64_t heads,
                                int64_t head_dim, float dropout_p, const void* rng_state, uint32_t rng_site,
                                void* ctx, float* lse, uint64_t* keep_bits, void* stream);
int32_t b2_attention_bwd_packed(const void* qkv, const int32_t* segments, const void* ctx, const void* d_ctx,
                                const float* lse, int64_t bins, int64_t heads, int64_t head_dim, float dropout_p,
                                const void* rng_state, uint32_t rng_site, void* d_qkv, float* dbias_accum,
                                const uint64_t* keep_bits, void* stream);
/* Bins of `seq` tokens (a multiple of 128, at most 512); segments int32 [bins * seq].  The segments of a bin must be  */
/* contiguous with every row inside its own (pack_batch builds them so): above 128 the kernels visit only the 128-row */
/* blocks a segment reaches; other segment words give wrong results for their bin, never an access outside it.      */
/* At seq == 128 these are b2_attention_{fwd,bwd}_packed.  Above 128 the backward takes                              */
/* the fp32 dq_accum [bins * seq, heads * 64] as b2_attention_bwd does, dbias_accum must be null (b2_colsum), and     */
/* keep_bits is not used (the backward regenerates the dropout decisions).                                           */
int32_t b2_attention_fwd_packed_seq(const void* qkv, const int32_t* segments, int64_t bins, int64_t seq, int64_t heads,
                                    int64_t head_dim, float dropout_p, const void* rng_state, uint32_t rng_site,
                                    void* ctx, float* lse, uint64_t* keep_bits, void* stream);
int32_t b2_attention_bwd_packed_seq(const void* qkv, const int32_t* segments, const void* ctx, const void* d_ctx,
                                    const float* lse, int64_t bins, int64_t seq, int64_t heads, int64_t head_dim,
                                    float dropout_p, const void* rng_state, uint32_t rng_site, void* d_qkv,
                                    float* dq_accum, float* dbias_accum, const uint64_t* keep_bits, void* stream);
/* The ordered dQ of the seq > 128 backward (torch.use_deterministic_algorithms): instead of adding every key block's
 * dQ contribution into dq_accum with atomics, the CTA of key block jb stores it into slice jb of
 *   dq_partials  fp32 [seq / 128][bins * seq, heads * 64]   (4 slices x 25.2 MB at 16 x 512 tokens, hidden 768)
 * and a second kernel sums the slices in ascending jb into d_qkv's Q columns: dQ is bitwise the same on every run.
 * dK and dV are those of the atomic form, bit for bit.  A slice a CTA never visits (packed bins skip blocks) is never
 * read, so the buffer needs no clearing.  Rejected: seq <= 128 (whose backward has no cross-CTA dQ sum) and a null
 * dq_partials.  No fused bias sums (b2_colsum) and no keep_bits, as for the atomic form above 128.              */
int32_t b2_attention_bwd_ordered(const void* qkv, const int64_t* attention_mask, const void* ctx, const void* d_ctx,
                                 const float* lse, int64_t batch, int64_t seq, int64_t heads, int64_t head_dim,
                                 float dropout_p, const void* rng_state, uint32_t rng_site, void* d_qkv,
                                 float* dq_partials, void* stream);
int32_t b2_attention_bwd_packed_seq_ordered(const void* qkv, const int32_t* segments, const void* ctx,
                                            const void* d_ctx, const float* lse, int64_t bins, int64_t seq,
                                            int64_t heads, int64_t head_dim, float dropout_p, const void* rng_state,
                                            uint32_t rng_site, void* d_qkv, float* dq_partials, void* stream);
/* b2_embed_bwd_ordered for packed bins (type_vocab <= 3)                                                          */
int32_t b2_embed_bwd_packed_ordered(const void* dy, int32_t dy_fp32, const void* pre_ln, const float* mean,
                                    const float* rstd, const void* gamma, const int32_t* ids32, const int32_t* tt32,
                                    const int32_t* pos32, int64_t bins, int64_t seq, int64_t hidden, int64_t vocab,
                                    int64_t type_vocab, int64_t pad_token_id, float dropout_p, const void* rng_state,
                                    uint32_t rng_site, void* d_word, void* d_pos, void* d_type, void* d_gamma,
                                    void* d_beta, void* scratch_dx, float* scratch_partials,
                                    int64_t scratch_partials_bytes, int32_t* owner, void* stream);
int32_t b2_head_fwd_packed(const void* hidden_states, const int64_t* cls_rows, int64_t batch, int64_t hidden,
                           const void* pool_w, const void* pool_b, const void* cls_w, const void* cls_b,
                           int64_t num_labels, float dropout_p, const void* rng_state, uint32_t rng_site,
                           void* pooled, float* logits, void* stream);
int32_t b2_head_bwd_packed(const float* dlogits, const void* hidden_states, const void* pooled,
                           const int64_t* cls_rows, int64_t tokens, int64_t batch, int64_t hidden,
                           const void* pool_w, const void* cls_w, int64_t num_labels, float dropout_p,
                           const void* rng_state, uint32_t rng_site, void* d_pool_w, void* d_pool_b, void* d_cls_w,
                           void* d_cls_b, void* d_hidden, int32_t d_hidden_fp32, float* scratch, void* stream);

/* b2_head_bwd / b2_head_bwd_packed (cls_rows NULL: row of sequence b = b * seq) with the two parameter-gradient
 * kernels launched on `weight_stream` (ordered behind the data-gradient part by an event; the same stream when NULL): they
 * are off the critical path of the backward.  Whatever reads the four head gradients must be ordered behind
 * `weight_stream`.                                                                                               */
int32_t b2_head_bwd_split(const float* dlogits, const void* hidden_states, const void* pooled,
                          const int64_t* cls_rows, int64_t tokens, int64_t batch, int64_t seq, int64_t hidden,
                          const void* pool_w, const void* cls_w, int64_t num_labels, float dropout_p,
                          const void* rng_state, uint32_t rng_site, void* d_pool_w, void* d_pool_b, void* d_cls_w,
                          void* d_cls_b, void* d_hidden, int32_t d_hidden_fp32, float* scratch, void* stream,
                          void* weight_stream);

/* token-classification head (HF BertForTokenClassification: no pooler; dropout + Linear on every token), over the
 * `tokens` rows of the last hidden state (batch x seq, or bins x bin_len when packed); 256 <= hidden <= 1024 a
 * multiple of 256, 1 <= num_labels <= 64, tokens <= 131072.  Dropout: Philox key (seed, step, rng_site,
 * (m * hidden + h) / 8), regenerated by the backward.
 *   logits[m, c] = cls_b[c] + sum_h drop(x[m, h]) cls_w[c, h]      (fp32 [tokens, num_labels])                   */
int32_t b2_token_head_fwd(const void* hidden_states, int64_t tokens, int64_t hidden, const void* cls_w,
                          const void* cls_b, int64_t num_labels, float dropout_p, const void* rng_state,
                          uint32_t rng_site, float* logits, void* stream);
/* backward: d_hidden[m, h] = keep(m, h) / (1 - p) sum_c dlogits[m, c] cls_w[c, h] (fp32, every row) on `stream`;
 * d_cls_w = sum_m dlogits[m]^T drop(x[m]) and d_cls_b = sum_m dlogits[m] (bf16) on `weight_stream` (ordered behind
 * `stream` by an event; `stream` when NULL), summed as fp32 partials per row block added in ascending block order:
 * bitwise repeatable, no atomics.  scratch: fp32, at least b2_token_head_scratch_floats(tokens, hidden, num_labels)
 * floats.  Whatever reads d_cls_w / d_cls_b must be ordered behind `weight_stream`.                              */
int32_t b2_token_head_bwd_split(const float* dlogits, const void* hidden_states, int64_t tokens, int64_t hidden,
                                const void* cls_w, int64_t num_labels, float dropout_p, const void* rng_state,
                                uint32_t rng_site, void* d_cls_w, void* d_cls_b, float* d_hidden, float* scratch,
                                int64_t scratch_floats, void* stream, void* weight_stream);
/* the fp32 scratch b2_token_head_bwd_split needs (a count, not a status)                                         */
int64_t b2_token_head_scratch_floats(int64_t tokens, int64_t hidden, int64_t num_labels);

/* ------------------------------------------------------------------------------------------------------ */
/* masked-language-model head (csrc/mlm_head.cu, HF BertForMaskedLM's cls.predictions)                     */
/* ------------------------------------------------------------------------------------------------------ */
/* The head runs on the labelled rows only, listed into `capacity` rows (capacity <= tokens).  b2_mlm_compact:
 * rows[i] = the i-th token (in token order) whose label is not ignore_index, slot_labels[i] its label, slot[m] = the
 * row of token m or -1, *count the number of them; the capacity rows past *count get row 0 and label -1.  A label
 * outside [0, vocab) that is not ignore_index, or more labelled tokens than the capacity, traps.               */
int32_t b2_mlm_compact(const int64_t* labels, int64_t tokens, int64_t ignore_index, int64_t vocab, int64_t capacity,
                       int32_t* rows, int32_t* slot, int32_t* slot_labels, int32_t* count, void* stream);
/* out[i] = x[rows[i]] (bf16 [capacity, hidden]) for i < *count, zero rows after it                              */
int32_t b2_mlm_gather_rows(const void* x, const int32_t* rows, const int32_t* count, int64_t capacity, int64_t hidden,
                           void* out, void* stream);
/* dx[m] = src[slot[m]] (fp32) for slot[m] >= 0, a zero row otherwise: every row of dx [tokens, hidden] is written  */
int32_t b2_mlm_scatter_rows(const float* src, const int32_t* slot, int64_t tokens, int64_t hidden, float* dx,
                            void* stream);
/* du = bf16(dg * gelu'(u)) elementwise, n a multiple of 8 (dg fp32, u bf16: the transform's pre-activation)      */
int32_t b2_mlm_gelu_bwd(const float* dg, const void* u, int64_t n, void* du, void* stream);
/* logits[r, c] = bias[c] (fp32 [rows, vocab_pad]), vocab_pad a multiple of 64: EPI_ACCUM_F32 then adds x W^T    */
int32_t b2_mlm_bias_fill(const void* bias, int64_t rows, int64_t vocab_pad, float* logits, void* stream);
/* Vocabulary cross-entropy over fp32 logits [rows, vocab_pad], one block per row.  labels int32 [rows] (NULL: all
 * -1), -1 = no loss term; rows at or past *n_rows (NULL: none) are capacity padding.  For each row:
 *   row_loss[r] = logsumexp(x[r, :vocab]) - x[r, y]   (0 without a label),   pred[r] = argmax (-1 without a label)
 *   d_logits[r, c] = bf16(d_extra[r, c] + (softmax - onehot) * (*d_loss) / (*n_labelled)) for c < vocab, 0 above
 * (d_loss NULL: 1; d_extra NULL: 0; pred / d_logits NULL: not written; padding rows get zero rows).  loss (NULL: not
 * written) = sum of row_loss / *n_labelled, summed in a fixed order: nan when *n_labelled is 0.  A label outside
 * [-1, vocab) traps.                                                                                           */
int32_t b2_mlm_ce(const float* logits, int64_t rows, int64_t vocab, int64_t vocab_pad, const int32_t* labels,
                  const int32_t* n_rows, const int32_t* n_labelled, const float* d_loss, const float* d_extra,
                  int64_t ld_extra, float* row_loss, int32_t* pred, void* d_logits, float* loss, void* stream);
/* grad = bf16(grad + dec) over n elements (a multiple of 8): the tied decoder's fp32 part of the word-embedding
 * gradient added onto the embedding backward's rows                                                           */
int32_t b2_mlm_tied_add(const float* dec, void* grad, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* question-answering span loss (csrc/qa_head.cu, HF BertForQuestionAnswering's loss)                       */
/* ------------------------------------------------------------------------------------------------------ */
/* The head is the token head with num_labels = 2 and no dropout: logits fp32 [rows, 2], column 0 the start logit and
 * column 1 the end logit of every row.  Sequence b covers rows [seq_first[b], seq_first[b] + seq_len[b]) (both NULL:
 * padded, rows [b * ignored_index, (b + 1) * ignored_index)), 1 to 512 rows each.  Its targets are HF's
 * clamp(0, ignored_index) of the raw int64 start_positions[b] / end_positions[b]; a target equal to ignored_index
 * (the padded length) is ignored.  Per sequence and column, a softmax over the sequence's own rows:
 *   seq_loss[2b + c] = logsumexp_r x[r, c] - x[t_c, c]   (0 when ignored)
 *   loss = (sum_b seq_loss[2b] / n_start + sum_b seq_loss[2b + 1] / n_end) / 2   (nan for an all-ignored column)
 *   d_logits[r, c] = (softmax - onehot) * (*d_loss) / (2 n_c)   (0 on an ignored column and on rows of no sequence)
 * with n_c the sequences whose column-c target is not ignored.  d_loss NULL: 1; d_logits / loss NULL: not written;
 * seq_loss: fp32 scratch [2 * num_seqs].  Every sum is in a fixed order without atomics: bitwise repeatable.  A
 * target inside [0, ignored_index) but past its sequence's rows traps.                                          */
int32_t b2_qa_span_loss(const float* logits, int64_t rows, const int64_t* start_positions,
                        const int64_t* end_positions, int64_t num_seqs, int64_t ignored_index, const int64_t* seq_first,
                        const int64_t* seq_len, const float* d_loss, float* seq_loss, float* d_logits, float* loss,
                        void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* optimizer + gradient exchange                                                                          */
/*   replaces: HF AdamW.step (transformers 4.28.1 optimization.py, built at multi-gpu-distributed-cls.py    */
/*   :100-111, stepped :174), optimizer.zero_grad (:172), and the DDP Reducer's bucket all-reduce            */
/*   (SP/torch/nn/parallel/distributed.py:1255-1280, reducer.hpp:276-286) for world > 1.                     */
/* ------------------------------------------------------------------------------------------------------ */
typedef struct b2_adamw_hparams {
  double lr, beta1, beta2, eps, weight_decay; /* python doubles, rounded to fp32 the way torch rounds them */
  int32_t correct_bias;
  /* optional DEVICE pointer to the fp32 loss scale of a torch.cuda.amp.GradScaler (the reference's -amp scripts,
   * multi-gpu-distributed-mp-amp-cls.py:160-171): gradients are divided by *grad_scale before the update.
   * NULL = unscaled gradients.                                                                                */
  const float* grad_scale;
  /* optional DEVICE pointer to the GradScaler's fp32 inf/nan indicator: a non-zero value skips the update (and the
   * step count), as GradScaler.step() skips optimizer.step().  NULL = always update.                            */
  const float* found_inf;
  /* gradient-norm clipping (torch.nn.utils.clip_grad_norm_, HF TrainingArguments.max_grad_norm) as optional fields
   * rather than separate entry points.  clip_coef: optional DEVICE fp32 scalar from b2_grad_norm_finalize; the
   * gradient is multiplied by it before the moments.  grad_f32 (b2_bucket_reduce_adamw only): optional DEVICE fp32
   * mean gradient of the slice [begin, end), indexed from begin (the stash of b2_grad_reduce_sumsq), read instead of
   * the peers' bf16 gradients.  NULL = today's update, bit for bit.                                                */
  const float* clip_coef;
  const float* grad_f32;
  /* optional DEVICE fp64 learning rate, read in place of `lr` by all three AdamW entry points: a captured training
   * step refreshes it before every replay from the host's param_groups[0]["lr"], so a torch LR scheduler keeps
   * working there.  lr * weight_decay is formed in double from it, as the host forms it from `lr`: a device value
   * equal to `lr` gives the same bits.  NULL = `lr` by value.                                                  */
  const double* lr_dev;
} b2_adamw_hparams_t;

/* Fused update of one contiguous slice [begin, end) (element indices, multiples of 8) of the flat parameter
 * space.  world == 1: grads read from `grad_local`.  world > 1: element-wise mean over `peer_grads[0..world)`
 * (peer-mapped bf16 buffers, fixed rank order => bit-identical on every rank), then the HF AdamW update on the
 * fp32 master / moments, then the bf16 shadow weights are stored to every non-NULL `peer_shadow[r]`
 * (peer_shadow[rank] must be set; NULL elsewhere = that peer's copy travels by b2_copy_async).
 * decay_flags: uint8 per 8-element vector (1 = apply weight decay).  step_counter: device int64, read here
 * (t = *step_counter + 1 for the bias correction); bumped separately by b2_step_advance.                     */
int32_t b2_bucket_reduce_adamw(const void* const* peer_grads, void* const* peer_shadow, int32_t world,
                               int32_t rank, float* master, float* exp_avg, float* exp_avg_sq,
                               const uint8_t* decay_flags, int64_t begin, int64_t end,
                               const b2_adamw_hparams_t* hp, const int64_t* step_counter, void* stream);

/* Single-GPU background form of the same update (world == 1, no GradScaler state): blocks of 128 threads x 32
 * registers and no shared memory, i.e. shaped to become resident BESIDE a 640-thread GEMM CTA instead of waiting for the
 * gaps between GEMM kernels; launched per bucket on the optimizer stream while the backward pass is still running.
 * `step_size` = the bias-corrected step of this update, a device float written by b2_adamw_prepare (lr * sqrt(1 - b2^t)
 * / (1 - b1^t), t = *step_counter + 1, in double like the host would); call b2_adamw_prepare once per step, after
 * b2_step_advance.  Same arithmetic as b2_bucket_reduce_adamw.                                                  */
int32_t b2_adamw_prepare(const b2_adamw_hparams_t* hp, const int64_t* step_counter, float* step_size, void* stream);
int32_t b2_adamw_background(const void* grads, void* shadow, float* master, float* exp_avg, float* exp_avg_sq,
                            const uint8_t* decay_flags, int64_t begin, int64_t end, const b2_adamw_hparams_t* hp,
                            const float* step_size, void* stream);

/* SGD with momentum: torch.optim.SGD (torch 2.11 sgd.py::_single_tensor_sgd) as the same two fused forms.  The optional
 * device fields mean exactly what they mean in b2_adamw_hparams_t.  Per element, with g the gradient AdamW would use
 * (mean over ranks / grad_scale * clip_coef):
 *   if maximize:     g = -g
 *   if decay flag:   g = g + weight_decay * w                      (coupled L2, on the master before the update)
 *   if momentum:     buf = g on the first applied step, else buf = momentum * buf + (1 - dampening) * g
 *                    g = nesterov ? g + momentum * buf : buf
 *   w = w + (-lr) * g;  shadow = bf16_rne(w)
 * Each `a + alpha * b` is one fma, as torch's CUDA add is; `momentum * buf` is rounded on its own.  weight_decay,
 * momentum, 1 - dampening and -lr are rounded to fp32 from the doubles (and -lr from *lr_dev the same way).
 * `momentum_buffer` (fp32, indexed like master) is given exactly when momentum != 0; with momentum 0 it is neither
 * read nor written.  `step_counter` (device int64, required with momentum) counts the applied steps since the buffer
 * came into use: 0 = the buffer is initialised from g (torch's `momentum_buffer is None`).  b2_step_advance bumps it
 * and leaves it alone on a skipped step.  A non-zero *found_inf leaves master, buffer and shadow untouched.
 * bytes / parameter at world 1: 12 without momentum (2 gradient, 4 + 4 master, 2 shadow), 20 with it.        */
typedef struct b2_sgd_hparams {
  double lr, momentum, dampening, weight_decay; /* python doubles, rounded to fp32 the way torch rounds them */
  int32_t nesterov, maximize;
  const float* grad_scale;
  const float* found_inf;
  const float* clip_coef;
  const float* grad_f32;
  const double* lr_dev;
} b2_sgd_hparams_t;

/* Any world: the form of b2_bucket_reduce_adamw (mean over peer_grads, or grad_f32; shadow stores to every non-NULL
 * peer_shadow[r]).                                                                                               */
int32_t b2_bucket_reduce_sgd(const void* const* peer_grads, void* const* peer_shadow, int32_t world, int32_t rank,
                             float* master, float* momentum_buffer, const uint8_t* decay_flags, int64_t begin,
                             int64_t end, const b2_sgd_hparams_t* hp, const int64_t* step_counter, void* stream);
/* world 1, no GradScaler state and no grad_f32: the form of b2_adamw_background (128 threads x <= 32 registers, no
 * shared memory), to run per bucket beside the backward's GEMM CTAs.  Needs no prepare step.                    */
int32_t b2_sgd_background(const void* grads, void* shadow, float* master, float* momentum_buffer,
                          const uint8_t* decay_flags, int64_t begin, int64_t end, const b2_sgd_hparams_t* hp,
                          const int64_t* step_counter, void* stream);

/* torch.optim.Adam / torch.optim.AdamW with fused=True (torch 2.11 ATen/native/cuda/fused_adam_utils.cuh, the
 * default optimizer of HF transformers 5.5's Trainer) as the same two fused forms.  The optional device fields mean
 * exactly what they mean in b2_adamw_hparams_t.  Everything is fp32: lr (or *lr_dev), betas, eps and weight_decay are
 * the doubles cast to float, t = (float)(*step_counter + 1).  Per element, with g the gradient AdamW would use:
 *   if maximize:     g = -g
 *   if decay flag:   decoupled (AdamW): w = w - (lr * weight_decay) * w;  else (Adam): g = g + w * weight_decay
 *   m = b1 * m + (g - b1 * g);  v = b2 * v + (g*g - b2 * g*g)        (torch's nested fmas)
 *   if amsgrad:      vmax = max(vmax, v), used in place of v below
 *   denom = sqrt(v) / sqrt(1 - b2^t) + eps;  w = w - (lr / (1 - b1^t)) * m / denom;  shadow = bf16_rne(w)
 * Each `a * b + c` is one fma and every other operation is rounded on its own, as in torch's build, so the result is
 * bitwise torch's fused kernel.  The one place that build varies is Adam's `g + w * weight_decay`: one fma with amsgrad
 * or a grad_scale; otherwise a product and a sum when maximizing and in lane 0 of torch's loop, one fma in lanes 1-3.
 * Lane 0 is an element whose index in its tensor is a multiple of 4; for a tensor whose size is not a multiple of 4
 * the decay flags of its vectors say it: B2_ADAM_DECAY_UNALIGNED, plus B2_ADAM_DECAY_LANE0 where (index % 2048) < 512.
 * `max_exp_avg_sq` (fp32, indexed like master) is given exactly when amsgrad is set.  A non-zero *found_inf leaves
 * master, moments and shadow untouched (and b2_step_advance leaves the step count).
 * bytes / parameter at world 1: 28 (2 gradient, 4 + 4 master, 8 + 8 moments, 2 shadow), 36 with amsgrad.       */
#define B2_ADAM_DECAY_UNALIGNED 2   /* decay flag bits (with bit 0 set) read by the Adam entry points only */
#define B2_ADAM_DECAY_LANE0 4
typedef struct b2_adam_hparams {
  double lr, beta1, beta2, eps, weight_decay; /* python doubles; the kernels cast them to float, as torch does */
  int32_t amsgrad, maximize, decoupled;
  const float* grad_scale;
  const float* found_inf;
  const float* clip_coef;
  const float* grad_f32;
  const double* lr_dev;
} b2_adam_hparams_t;

/* Any world: the form of b2_bucket_reduce_adamw.                                                                  */
int32_t b2_bucket_reduce_adam(const void* const* peer_grads, void* const* peer_shadow, int32_t world, int32_t rank,
                              float* master, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                              const uint8_t* decay_flags, int64_t begin, int64_t end, const b2_adam_hparams_t* hp,
                              const int64_t* step_counter, void* stream);
/* `prepared` = device float[2] {lr / (1 - b1^t), sqrt(1 - b2^t)} of the next update, written by b2_adam_prepare (t =
 * *step_counter + 1, lr from *lr_dev when set); call it once per step, after b2_step_advance.  b2_adam_background is
 * world 1 with no GradScaler state and no grad_f32: the form of b2_adamw_background (128 threads x <= 32 registers,
 * no shared memory, with and without amsgrad), to run per bucket beside the backward's GEMM CTAs.               */
int32_t b2_adam_prepare(const b2_adam_hparams_t* hp, const int64_t* step_counter, float* prepared, void* stream);
int32_t b2_adam_background(const void* grads, void* shadow, float* master, float* exp_avg, float* exp_avg_sq,
                           float* max_exp_avg_sq, const uint8_t* decay_flags, int64_t begin, int64_t end,
                           const b2_adam_hparams_t* hp, const float* prepared, void* stream);

/* Gradient accumulation over the slice [begin, end) (element indices, multiples of 8) of the bf16 gradient space
 * `grads` and its fp32 accumulator `accum` (both indexed from their base, 16-byte aligned).
 *   replaces: torch's accumulation into `.grad` across backwards, and DDP's no_sync() skipping the Reducer
 *   (SP/torch/nn/parallel/distributed.py `no_sync`, `require_backward_grad_sync`) for the micro-batches of a window.
 *   mode   operation                               bytes / parameter
 *   STORE  accum = f32(grads)                      6   (first pass of a window: the accumulator is never zeroed)
 *   ADD    accum += f32(grads)                     10
 *   FOLD   grads = bf16_rne(accum + f32(grads))    8   (the final pass: exchange / AdamW then read `grads`)
 *   FLUSH  grads = bf16_rne(accum)                 6   (optimizer step with no final pass)
 * inf / nan propagate.  Blocks of 128 threads x <= 32 registers, no shared memory: shaped like
 * b2_adamw_background, to run per bucket beside the backward's GEMM CTAs.                                      */
#define B2_ACCUM_STORE 0
#define B2_ACCUM_ADD 1
#define B2_ACCUM_FOLD 2
#define B2_ACCUM_FLUSH 3
int32_t b2_grad_accumulate(void* grads, float* accum, int64_t begin, int64_t end, int32_t mode, void* stream);

/* Gradient-norm clipping (torch.nn.utils.clip_grad_norm_ with norm_type 2, torch 2.11 `clip_grads_with_norm_`).  No
 * parameter may move until the norm of the whole (DDP-mean) gradient is known, so a clipped step runs in three phases:
 * reduce (+ partial sums of squares) per bucket slice, one finalize, then the update with hparams.clip_coef.
 *
 * Reduce phase over [begin, end) (multiples of 8).  world > 1: rank-order fp32 sum of the slice over
 * `peer_grads[0..world)` times 1/world -- the gradient b2_bucket_reduce_adamw would use -- stored into `stash`
 * (fp32 [end - begin], indexed from begin, 16-byte aligned).  world 1: reads peer_grads[0], stash must be NULL.
 * Each warp writes the sum of squares of the gradients it saw to its own fp64 slot of `partials`:
 * B2_SUMSQ_SLOTS(end - begin) slots, every one written.  No atomics: bit-reproducible.  Blocks of 128 threads x
 * <= 32 registers, no shared memory: shaped to run per bucket beside the backward's GEMM CTAs.
 * bytes / parameter: 2 * world in, 4 out (world 1: 2 in).                                                          */
#define B2_SUMSQ_SLOTS(n) (4 * (((n) + 8191) / 8192))
int32_t b2_grad_reduce_sumsq(const void* const* peer_grads, int32_t world, float* stash, int64_t begin, int64_t end,
                             double* partials, void* stream);
/* Norm finalize: sums partials[0..nslots) in a fixed order (fp64).  world > 1: the ranks' totals are then added in rank
 * order through peer memory (b2_scalar_allreduce_mean on `slot`, x world): bit-identical on every rank.  Writes
 *   *total_norm = sqrt(sum) / *grad_scale (grad_scale optional: the norm of the unscaled gradients)
 *   *clip_coef  = min(1, max_norm / (*total_norm + 1e-6)); a non-finite norm propagates as in torch (NaN stays NaN)
 *   *skip       (optional) = 1 if *found_inf (optional) is non-zero, or a grad_scale is given and the norm is not
 *                 finite (GradScaler's inf check over every gradient); else 0.  Use it as the update's found_inf.
 * world 1: one launch; peer_scratch / peer_flags / epoch may be NULL.                                            */
int32_t b2_grad_norm_finalize(const double* partials, int64_t nslots, float* const* peer_scratch,
                              void* const* peer_flags, int32_t world, int32_t rank, int32_t slot, uint32_t* epoch,
                              float max_norm, const float* grad_scale, const float* found_inf, float* total_norm,
                              float* clip_coef, float* skip, void* stream);

/* ++step (AdamW t, SGD's applied-step count) and ++rng step (dropout stream) on the device: keeps CUDA-graph replays
 * stateful.  found_inf (optional device fp32, see b2_adamw_hparams_t): non-zero leaves the step count untouched.  */
int32_t b2_step_advance(int64_t* step_counter, void* rng_state, const float* found_inf, void* stream);
int32_t b2_rng_seed(void* rng_state, uint64_t seed, uint64_t step, void* stream);

/* segments[i] = {src element offset in `src` (fp32), dst element offset in `dst` (bf16), count}: dst <- bf16(src), then
 * src <- 0.  One launch turns the per-step fp32 bias-gradient accumulators (filled by atomics from the GEMM and
 * attention-backward epilogues) into bf16 gradients and re-arms them.                                           */
int32_t b2_accum_finish(float* src, void* dst, const int64_t* segments /* device [n][3] */, int64_t n_segments,
                        int64_t max_count, void* stream);

/* bf16 <- fp32 cast of a flat range (initial shadow weights, load_state_dict) and zero fill                 */
int32_t b2_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
int32_t b2_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream);
int32_t b2_zero(void* dst, int64_t bytes, void* stream);
/* stream-ordered device-to-device copy; with an IPC-mapped peer pointer on one side it is a copy-engine transfer
 * over NVLink (the DMA form of the gradient exchange: peers' slices in, updated bf16 weights out)             */
int32_t b2_copy_async(void* dst, const void* src, int64_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------ */
/* peer memory over NVLink / NVSwitch (one process per GPU; handles exchanged by the host through           */
/* torch.distributed).  replaces dist.all_reduce / all_gather / barrier call sites                          */
/* (multi-gpu-distributed-cls.py:141,148,153,171) on the step path.                                          */
/* ------------------------------------------------------------------------------------------------------ */
#define B2_IPC_HANDLE_BYTES 64
int32_t b2_comm_alloc(int64_t bytes, void** ptr);                       /* cudaMalloc'ed, IPC-exportable     */
int32_t b2_comm_free(void* ptr);
int32_t b2_comm_export(void* ptr, uint8_t handle[B2_IPC_HANDLE_BYTES]);
int32_t b2_comm_import(const uint8_t handle[B2_IPC_HANDLE_BYTES], void** ptr);
int32_t b2_comm_unimport(void* ptr);

/* Device-side barrier across ranks through flag words in each rank's signal pad.
 * peer_flags[r] points at rank r's pad (uint32[world * B2_FLAG_SLOTS]); `slot` selects the flag family; `epoch` is a
 * device counter incremented by the kernel so graph replays stay in lock-step.  Bounded spin -> trap.       */
#define B2_FLAG_SLOTS 64
int32_t b2_peer_barrier(void* const* peer_flags, int32_t world, int32_t rank, int32_t slot, uint32_t* epoch,
                        void* stream);

/* Trainer.output_reduce (multi-gpu-distributed-cls.py:145-155): every rank stores its [rows, row_bytes] block
 * into slot `rank` of every peer's gather buffer, then a barrier.                                           */
int32_t b2_allgather_rows(const void* src, int64_t bytes, void* const* peer_dst, void* const* peer_flags,
                          int32_t world, int32_t rank, int32_t slot, uint32_t* epoch, void* stream);
/* Trainer.loss_reduce (:139-143): mean of one fp32 scalar over ranks                                        */
int32_t b2_scalar_allreduce_mean(const float* src, float* dst, float* const* peer_scratch,
                                 void* const* peer_flags, int32_t world, int32_t rank, int32_t slot,
                                 uint32_t* epoch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2_DDP_BERT_H_ */
