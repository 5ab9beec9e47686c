/* dprb.h — C ABI of libdprb.so: the H100 (sm_90a) drop-in for the arithmetic of dpr-scale's
 * bi-encoder contrastive training step.
 *
 * The reference (facebookresearch/dpr-scale) is pure Python and has no FFI of its own; every FLOP on
 * the path is delegated to torch / HuggingFace modules.  Each entry point below therefore cites the
 * reference call site (file:line under /root/reference, or site-packages/transformers for the
 * third-party code the reference calls) whose arithmetic it replaces.  INTEGRATION.md shows the
 * ctypes binding a dpr-scale maintainer would add.
 *
 * Conventions
 *  - Every function returns 0 on success; non-zero = error, text via dprb_last_error() (thread-local).
 *  - All pointers are DEVICE pointers owned by the caller (PyTorch caching allocator); the library
 *    allocates nothing persistent and keeps no global mutable state besides cached device attributes.
 *  - `stream` is a cudaStream_t; all work is enqueued on it and no call synchronises the device.
 *  - bf16 tensors are row-major with 16-byte aligned rows; H, I multiples of 8; head_dim == 64.
 *  - One process per GPU; collectives are NOT issued here (torch.distributed/NCCL does that).
 */
#ifndef DPRB_H_
#define DPRB_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dprb_stream_t; /* cudaStream_t */

#define DPRB_VERSION 101

int dprb_version(void);
const char* dprb_last_error(void);
/* SM count of the current device (cached); <=0 when no device. */
int dprb_num_sms(void);
/* Number of kernels this library has launched in this process since load (every <<<>>> / cudaLaunchKernelEx site
 * increments it).  bench.py reports the difference over its timed region as `gpu_launches` - a count, not an estimate.
 * No reference counterpart (the reference launches through PyTorch). */
int64_t dprb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * GEMM (TMA / wgmma):  D[M,N] = epilogue( alpha * sum_k A(m,k) * B(n,k) )
 * Replaces torch.nn.Linear forward/backward inside HF BertLayer:
 *   site-packages/transformers/models/bert/modeling_bert.py:179-181 (Q,K,V — fused here into one
 *   [3H,H] weight), :295 (attention output dense), :340 (intermediate dense), :353 (output dense).
 * colsum (optional, bf16 epilogues except BIAS_GELU): colsum[n] += sum_m D(m,n) — the bias gradient of the
 * Linear whose output gradient this GEMM produces, fused into the epilogue instead of a separate pass.
 * dropout_p / dropout_site_seed (BIAS_RESIDUAL only): D = dropout(acc + bias) + aux — HF's hidden dropout between the
 * dense layer and the residual add (modeling_bert.py:296-297, :354-355); the mask is a counter-based hash of the
 * element index (never stored; dprb_ln_bwd re-derives it, dprb_dropout_mask exports it for tests).
 * a_mn_major/b_mn_major = 0: operand stored [MN, K] (K contiguous, leading dim ld);
 *                       = 1: operand stored [K, MN] (MN contiguous, leading dim ld).
 * ------------------------------------------------------------------------------------------- */
enum {
  DPRB_EPI_BIAS = 0,           /* D(bf16) = acc + bias                      (bias may be NULL)        */
  DPRB_EPI_BIAS_GELU = 1,      /* D(bf16) = gelu(acc + bias) ; out2(bf16, optional) = gelu'(acc + bias) */
  DPRB_EPI_BIAS_RESIDUAL = 2,  /* D(bf16) = acc + bias + aux(bf16)                                     */
  DPRB_EPI_DGELU = 3,          /* D(bf16) = acc * aux(bf16), aux = the gelu' saved by BIAS_GELU          */
  DPRB_EPI_F32_ATOMIC_ADD = 4, /* D(fp32) += acc  (split-K over `splits` CTAs; 0 = choose)            */
  DPRB_EPI_F32_STORE = 5,      /* D(fp32) = acc + bias                                                 */
  DPRB_EPI_DGELU_PRE = 6,      /* D(bf16) = acc * gelu'(aux), aux(bf16) = the PRE-activation saved by BIAS_GELU|SAVE_PRE */
  DPRB_EPI_COUNT = 7
};
/* OR-ed into `epilogue`: the named 16-bit operand holds IEEE fp16 instead of bf16 (wgmma takes one
 * format for both operands: give DPRB_GEMM_A_F16 and DPRB_GEMM_B_F16 together or not at all).  The encoder keeps its residual stream - LayerNorm inputs and outputs - in fp16 (11 significand
 * bits in the same 2 bytes): these are the tensors HF's autocast keeps in fp32 (modeling_bert.py:296-298, :354-356
 * run LayerNorm and the residual add outside the 16-bit region).  AUX / OUT apply to the BIAS and BIAS_RESIDUAL
 * epilogues. */
enum { DPRB_GEMM_A_F16 = 0x100, DPRB_GEMM_B_F16 = 0x200, DPRB_GEMM_AUX_F16 = 0x400, DPRB_GEMM_OUT_F16 = 0x800,
       /* BIAS_GELU: out2 receives the pre-activation instead of gelu'(pre) - the "lean activations" mode of the encoder,
        * which saves ONE [T, I] tensor per layer (pre) instead of two (gelu', gelu) and rebuilds both in backward. */
       DPRB_GEMM_SAVE_PRE = 0x1000 };
/* (A_F16 and B_F16 must be given together: the hardware rejects an fp16 x bf16 operand pair.) */
int dprb_gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int64_t lda, int64_t ldb,
                   int64_t ldd, int a_mn_major, int b_mn_major, int epilogue, const float* bias,
                   const void* aux, int64_t ld_aux, void* out2, float alpha, int splits, float* colsum,
                   float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream);

/* Measurement aid (bench.py roofline leg): when enabled, every GEMM launch is bracketed by CUDA events on
 * its launch stream; dprb_gemm_profile_read sums the per-launch durations and algorithmic FLOPs (2*M*N*K). */
int dprb_gemm_profile_enable(int enable, int max_launches);
int dprb_gemm_profile_read(double* total_ms, double* total_flops, int64_t* launches);

/* ---------------------------------------------------------------------------------------------
 * Embeddings + LayerNorm.  Replaces BertEmbeddings.forward (modeling_bert.py:72-112):
 *   z = word[ids] + type[type_ids] + pos[pos_ids];  y = LN(z) (eps, gamma, beta).
 * Tables and LN parameters are the fp32 master weights.  stats[t] = (mean, rstd).
 * ------------------------------------------------------------------------------------------- */
int dprb_embed_ln_fwd(const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids, const float* word,
                      const float* pos, const float* type, const float* gamma, const float* beta, void* y_bf16,
                      float* stats, int T, int H, int vocab, int max_pos, int type_vocab, float eps,
                      float dropout_p, uint64_t dropout_seed, void* y_res_f16, dprb_stream_t stream);
/* The residual stream in fp16.  y_res_f16 (here and in dprb_ln_fwd, optional): a second copy of the LayerNorm output
 * in IEEE fp16, read by the NEXT residual add (DPRB_GEMM_AUX_F16) while the bf16 copy y feeds the next GEMM - kind::f16
 * cannot mix fp16 activations with bf16 weights, and HF's autocast keeps exactly this path (LayerNorm output ->
 * residual add -> LayerNorm input) out of 16-bit bf16.  z_f16 (dprb_ln_fwd / dprb_ln_bwd): the pre-LayerNorm sum z,
 * written by a DPRB_GEMM_OUT_F16 epilogue, holds fp16. */
/* Backward: dz = LN'(dy); dgamma/dbeta accumulated; scatter-add of dz into the three table grads. */
int dprb_embed_ln_bwd(const void* dy_bf16, const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids,
                      const float* word, const float* pos, const float* type, const float* gamma,
                      const float* stats, float* dword, float* dpos, float* dtype, float* dgamma, float* dbeta,
                      int T, int H, float dropout_p, uint64_t dropout_seed, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * LayerNorm over rows of z (the residual sum is produced by the preceding GEMM epilogue).
 * Replaces BertSelfOutput / BertOutput LayerNorm (modeling_bert.py:294-298, :352-356).
 * If cls_out != NULL, rows t with t % cls_stride == 0 are also written in fp32 to
 * cls_out[t / cls_stride, :] — the CLS pooling + .clone() of hf_model.py:39-41.
 * ------------------------------------------------------------------------------------------- */
int dprb_ln_fwd(const void* z_bf16, const float* gamma, const float* beta, void* y_bf16, float* stats,
                float* cls_out, int cls_stride, int T, int H, float eps, int z_f16, void* y_res_f16,
                dprb_stream_t stream);
/* dz = LN'(dy; z, stats); dgamma += sum dy*xhat; dbeta += sum dy; if dbias != NULL: dbias += sum_t dz
 * (the bias gradient of the Linear that produced z).  If dy_cls != NULL, dy is implicit: zero
 * everywhere except rows t % cls_stride == 0 which take dy_cls[t / cls_stride, :] (fp32). */
/* With hidden dropout (dropout_p > 0): dzm_bf16 receives dz * mask/(1-p) — the gradient of the Linear output that was
 * dropped before the residual add — and dbias sums dzm instead of dz. */
int dprb_ln_bwd(const void* dy_bf16, const float* dy_cls, int cls_stride, const void* z_bf16,
                const float* stats, const float* gamma, void* dz_bf16, float* dgamma, float* dbeta,
                float* dbias, int T, int H, void* dzm_bf16, float dropout_p, uint64_t dropout_site_seed,
                int z_f16, dprb_stream_t stream);
/* Dropout sites: 0 embeddings [T,H], 1 attention probabilities [nseq*heads*S, S], 2 attention-output dense [T,H],
 * 3 FFN-output dense [T,H]; with layer 0, the cross-encoder head's 4 after tanh [N,H] (dprb_seqcls_group_ce) and 5 on
 * RoBERTa's CLS rows before the head's dense layer [N,H].  Element (r, c) of a site is kept iff its 16-bit lane of h(r, c/8, (c/2)%4, site seed)
 * is >= round(p * 65536) - one hash chain per group of 8 columns, one multiply-xorshift finaliser per column pair
 * (csrc/common.cuh: Drop); site seed = fold32(dropout_seed + (layer*8 + site + 1) * 0x9E3779B97F4A7C15).
 * dprb_ln_bwd: dbias accumulates the column sums of the Linear's own output gradient (dzm when dropout is on).
 * dprb_dropout_mask materialises keep[r * cols + c] of one site (test aid). */
uint64_t dprb_dropout_site_seed(uint64_t dropout_seed, int layer, int site);
int dprb_dropout_mask(uint8_t* keep, int64_t rows, int cols, float dropout_p, uint64_t dropout_seed, int layer,
                      int site, dprb_stream_t stream);

/* out(bf16) = gelu(pre(bf16)), elementwise over n (multiple of 8) values: rebuilds BertIntermediate's activation
 * (modeling_bert.py:339-342) in backward when the encoder ran with lean activations (save_for_backward = 2). */
int dprb_gelu_from_pre(const void* pre_bf16, void* out_bf16, int64_t n, dprb_stream_t stream);
/* Column sums: out[n] += sum_t x[t, n]  (bias gradients; x bf16 [T, N] with leading dim ld). */
int dprb_colsum_bf16(const void* x_bf16, int64_t ld, float* out, int T, int N, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Self-attention core for head_dim 64, S <= 512.  Replaces BertSelfAttention.forward's
 * scaled_dot_product_attention (modeling_bert.py:168-207, integrations/sdpa_attention.py:92-101):
 *   ctx = softmax(Q K^T / 8 + key_mask) V      per (sequence, head).
 * qkv: bf16 [nseq*S, 3H] = [Q | K | V] column blocks, head h at columns h*64.
 * attn_mask: int32 [nseq, S], 1 = real token, 0 = padding (HF attention_mask); may be NULL.
 * lse: fp32 [nseq, heads, S] natural-log row log-sum-exp, written by fwd (may be NULL for
 *      forward-only use) and consumed by bwd together with the forward output ctx.
 * Kernels: S <= 256 keeps every key of a row in one block; 256 < S <= 512 streams 128-key blocks with an online
 * softmax, and its backward (one dK/dV and one dQ kernel, deterministic) takes D = rowsum(dctx * ctx) from ctx.
 * ------------------------------------------------------------------------------------------- */
int dprb_attn_fwd(const void* qkv_bf16, const int32_t* attn_mask, void* ctx_bf16, float* lse, int nseq, int S,
                  int heads, float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream);
/* dbias (optional, fp32 [3H]): dbias[n] += sum_t dqkv[t, n] — the bias gradient of the fused QKV projection. */
int dprb_attn_bwd(const void* qkv_bf16, const int32_t* attn_mask, const void* ctx_bf16, const float* lse,
                  const void* dctx_bf16, void* dqkv_bf16, float* dbias, int nseq, int S, int heads,
                  float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream);
/* Single-query (CLS row) attention of the encoder's pruned last layer, where only query 0 of each sequence attends
 * (test hooks: the encoder calls these kernels internally).  Same qkv / attn_mask layout and dropout site as
 * dprb_attn_fwd; the probability dropout of query 0 of problem (seq, h) uses row (seq*heads + h)*S of site 1.
 *   ctx_cls: bf16 [nseq, H]  = softmax(q_0 K^T / 8 + key_mask) V per head;
 *   probs:   fp32 [nseq, heads, S] the (undropped) probabilities of query 0, written by fwd and read by bwd;
 *   dqkv:    bf16 [nseq*S, 3H] fully written by bwd: dQ on row 0 of each sequence (zeros on rows 1..S-1), dK / dV on
 *            every row (zeros for masked keys). */
int dprb_attn_cls_fwd(const void* qkv_bf16, const int32_t* attn_mask, void* ctx_cls_bf16, float* probs, int nseq, int S,
                      int heads, float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream);
int dprb_attn_cls_bwd(const void* qkv_bf16, const float* probs, const void* dctx_cls_bf16, void* dqkv_bf16, int nseq,
                      int S, int heads, float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Fused in-batch-negative scoring + softmax cross-entropy.
 * Replaces dpr_scale/task/dpr_task.py:98-105 (sim_score: q @ c.T, scores[mask] = -inf),
 * :197 (mask.repeat), :211 (scores /= T), :212 (nn.CrossEntropyLoss, mean over Q).
 *   q fp32 [Q,d], c fp32 [C,d] (16-byte aligned), col_mask u8 [C] (1 = dummy ctx -> -inf), labels i64 [Q];
 *   pair_mask u8 [Q,C] (optional, 1 -> -inf): the per-query block mask of the non-in-batch branch (:199-207).
 *   d % 8 == 0 (pad q and c with zero columns otherwise: they add exactly 0 to every product); Q == 0 is a no-op.
 * Outputs: lse[Q], loss_sum (caller-zeroed; += sum over rows of lse - logit[label]; caller divides by Q),
 *          logits fp32 [Q,C] (masked columns = -inf) only if non-NULL.
 * Backward of mean-over-Q loss (grad_scale = upstream dL, normally 1):
 *   dq[q0:q0+nq, :]  (rows owned by this rank)  and  dc[c0:c0+nc, :] (columns owned by this rank),
 *   reproducing dpr_task.py:163-195 where remote slices are detached constants.
 * ONE tensor-core pass (the form BASELINE.json's north_star names): similarity tile via wgmma tiles staged in shared
 * memory, online row max / sum-exp / label pick per row, loss accumulated by the last tile of each row block.
 * fp32 fidelity comes from a 2-part bf16 split of q and c (x ~ h + m; the three products h.m, m.h, h.h per k-block,
 * fp32 accumulate): logits agree with the fp32 product of dpr_task.py:99 to a few 1e-6 of max|logit|.  Backward
 * RECOMPUTES the tiles of the rank-local row block and column block (no stored logits) and runs dq = W_rows c,
 * dc = W_cols^T q on the library's GEMM.
 * The softmax is taken relative to each row's max: the forward leaves the row max and log-sum in the workspace and
 * the backward builds W = softmax - onehot from them, so every row of W sums to 0 within a few ulp of 1, and the loss
 * of a row whose label wins by a margin keeps fp32 relative accuracy, at any |logit| (raw dot products in the
 * hundreds).  The backward's `lse` argument is not read; it is the forward's output, kept for the ABI.
 *   nq / nc: the local row / column counts backward will ask for (sizes the workspace; -1 = all).
 *   workspace: caller-owned, 256-byte aligned, >= dprb_score_tc_workspace_bytes(...); it carries the operand splits
 *   from the forward call to the backward call of the same step.
 * ------------------------------------------------------------------------------------------- */
int64_t dprb_score_tc_workspace_bytes(int Q, int C, int d, int nq, int nc);
int dprb_score_tc_fwd(const float* q, const float* c, const uint8_t* col_mask, const uint8_t* pair_mask,
                      const int64_t* labels, float inv_temperature, float* lse, float* loss_sum, float* logits, int Q,
                      int C, int d, int nq, int nc, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);
int dprb_score_tc_bwd(const uint8_t* col_mask, const uint8_t* pair_mask, const int64_t* labels, const float* lse,
                      float grad_scale, float inv_temperature, float* dq, float* dc, int Q, int C, int d, int q0, int nq,
                      int c0, int nc, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Optimizer step over a flat fp32 parameter arena.  Replaces torch.optim.AdamW
 * (conf/task/optim/adamw.yaml via dpr_task.py:124) + clip_grad_norm_(2.0)
 * (conf/trainer/gpu_1_host.yaml:8) + the bf16 weight shadow refresh.
 *   dprb_sumsq: out[0] += sum g^2.
 *   dprb_adamw_step: coef = min(1, max_norm / (sqrt(*sumsq) * grad_scale) + 1e-6) multiplies grad_scale * g
 *   before the moments are updated (optim.cu).
 * ------------------------------------------------------------------------------------------- */
int dprb_sumsq_f32(const float* g, int64_t n, float* out, dprb_stream_t stream);
int dprb_adamw_step(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t n, float lr,
                    float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                    const float* sumsq, float max_norm, dprb_stream_t stream);
/* LAMB (torch_optimizer.Lamb 0.3.x, conf/task/optim/lamb.yaml) with the same clip coefficient, per parameter tensor.
 * With g = coef * grad_scale * grad:  m, v as Adam (no bias correction);  u = m / (sqrt(v) + eps) + weight_decay * p;
 * trust = min(||p||, clamp_value) / ||u|| per segment (1 if either norm is 0 or adam != 0);
 * p -= lr * (debias ? sqrt(1 - beta2^step) / (1 - beta1^step) : 1) * trust * u.  grads are read only.
 * plan (device, int64): chunk_off[nchunks+1] | chunk_seg[nchunks] | seg_chunk[nseg+1] - chunks are contiguous ranges of
 * the arena, every offset a multiple of 4, none straddling a segment; chunk_off[0] = 0, chunk_off[nchunks] = n.
 * Norms are reduced per chunk and then per segment in a fixed order (no atomics): the update is bitwise repeatable.
 * workspace: at least dprb_lamb_workspace_bytes(nchunks, nseg) bytes, 16-byte aligned (partial sums, trust ratios). */
int64_t dprb_lamb_workspace_bytes(int nchunks, int nseg);
int dprb_lamb_step(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t n, const int64_t* plan,
                   int nchunks, int nseg, float lr, float beta1, float beta2, float eps, float weight_decay,
                   float clamp_value, int adam, int debias, int step, float grad_scale, const float* sumsq,
                   float max_norm, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);
/* MADGRAD, the dense branch of dpr_scale/optim/madgrad.py (conf/task/optim/madgrad.yaml), same clip coefficient.
 * lamb = (lr + eps) * sqrt(k + 1), k counting steps from 0;  g = coef * grad_scale * grad + weight_decay * p;
 * momentum == 0: x0 = p + s / (cbrt(grad_sum_sq) + eps) before the update (x0 must be NULL);
 * momentum != 0: x0 is the caller's copy of the parameters taken when the optimizer was built;
 * grad_sum_sq += lamb * g^2;  s += lamb * g;  z = x0 - s / (cbrt(grad_sum_sq) + eps);
 * p = momentum == 0 ? z : momentum * p + (1 - momentum) * z.  grads are read only. */
int dprb_madgrad_step(float* p, const float* g, float* grad_sum_sq, float* s, const float* x0, void* shadow_bf16,
                      int64_t n, float lr, float momentum, float weight_decay, float eps, int k, float grad_scale,
                      const float* sumsq, float max_norm, dprb_stream_t stream);
/* fp32 -> bf16 shadow refresh (after a state_dict load). */
int dprb_cast_f32_bf16(const float* src, void* dst_bf16, int64_t n, dprb_stream_t stream);
/* bf16 -> fp32: unpacks a bf16-compressed gradient slice after its all-reduce (the `fp16_grads` path:
 * torch's fp16_compress_hook registered at dpr_scale/task/dpr_task.py:90-92 casts, all-reduces and casts back). */
int dprb_cast_bf16_f32(const void* src_bf16, float* dst, int64_t n, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Whole-encoder forward / backward: the BertModel stack of modeling_bert.py:628-691 as called from
 * dpr_scale/models/hf_model.py:36-41, minus the unused pooler.  See dprb_encoder.h-style struct below.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  /* dims */
  int32_t hidden, inter, layers, heads, vocab, max_pos, type_vocab;
  float ln_eps;
  /* flat arenas (see dprb_param_offsets): fp32 master, bf16 shadow, fp32 grads */
  const float* master;
  const void* shadow;
  float* grads;
  /* offsets (in elements) into the arenas */
  int64_t off_word, off_pos, off_type, off_emb_ln_g, off_emb_ln_b;
  int64_t off_layer0;     /* first layer block */
  int64_t layer_stride;   /* elements per layer block */
  /* per-layer relative offsets */
  int64_t rel_wqkv, rel_bqkv, rel_wo, rel_bo, rel_ln1_g, rel_ln1_b, rel_w1, rel_b1, rel_w2, rel_b2, rel_ln2_g,
      rel_ln2_b;
} dprb_encoder_weights;

typedef struct {
  int32_t nseq, S;
  const int64_t* ids;      /* [nseq*S] */
  const int64_t* type_ids; /* [nseq*S] */
  const int64_t* pos_ids;  /* [nseq*S] */
  const int32_t* attn_mask;/* [nseq*S] or NULL */
  /* activation workspace, caller-allocated: see dprb_encoder_workspace_bytes */
  void* workspace;
  int64_t workspace_bytes;
  int32_t save_for_backward; /* 0: forward-only (generate_embeddings path) reuses per-layer buffers; 1: keep every
                              * activation backward reads; 2: "lean" - per layer keep qkv, the two pre-LayerNorm sums,
                              * x1, the FFN pre-activation and the layer output, and REBUILD the attention output
                              * (one more attention forward) and gelu / gelu' (from the pre-activation) in backward:
                              * 22 KB instead of 32 KB per token and layer at RoBERTa-large, which is what lets
                              * RoBERTa-large at S = 256 train on an 80 GB H100 without recomputing the whole
                              * forward. */
  float dropout_p;           /* hidden + attention-probability dropout (HFEncoder's `dropout`); 0 in eval mode */
  uint64_t dropout_seed;     /* per-forward seed; backward must be given the same value */
} dprb_encoder_batch;

int64_t dprb_encoder_workspace_bytes(const dprb_encoder_weights* w, int nseq, int S, int save_for_backward);
/* pooled fp32 [nseq, hidden] = last-layer hidden state of token 0 of each sequence.
 * Requires S <= 512 and S <= max_pos; every pos_ids entry must be < max_pos (RoBERTa's pad-derived ids reach
 * S + pad_token_id, so there max_pos >= S + pad_token_id + 1). */
int dprb_encoder_fwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, float* pooled,
                     dprb_stream_t stream);
/* Accumulates parameter gradients into w->grads given dpooled fp32 [nseq, hidden].
 * Layers [layer_hi-1 .. layer_lo] are processed (layer_lo == 0 also runs the embedding backward), so
 * the host can interleave gradient all-reduce buckets between calls. */
int dprb_encoder_bwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, const float* dpooled,
                     int layer_lo, int layer_hi, dprb_stream_t stream);

/* Token-level forward (ColBERT / late-interaction encoders: dpr_scale/models/citadel_models/colbert_model.py:39-44
 * reads hidden_states[-1]).  Writes the final LayerNorm output of EVERY token, bf16 [nseq*S, hidden] row-major, straight
 * into `tokens`; the last layer is never CLS-pruned, whatever DPRB_NO_CLS_PRUNE says.  Forward only: returns 1 unless
 * b->save_for_backward == 0.  Workspace: dprb_encoder_workspace_bytes(w, nseq, S, 0).  Row s*S of `tokens` equals
 * bf16(pooled[s]) of dprb_encoder_fwd run with DPRB_NO_CLS_PRUNE=1 on the same batch, bit for bit. */
int dprb_encoder_fwd_tokens(const dprb_encoder_weights* w, const dprb_encoder_batch* b, void* tokens,
                            dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Late-interaction (ColBERT MaxSim) scores of reranking pairs, forward only.  Replaces expert_sim_score of
 * dpr_scale/task/citadel_eval_task.py:236-265 (no expert ids): for pair b with query qi = q_index[b],
 *   s[i][j] = q[qi][i] . d[b][j]            over tokens i = 1 .. SQ-1, j = 1 .. SD-1 (token 0 is skipped)
 *   score[b] = sum_i max_j s[i][j]          (pool DPRB_MAXSIM_SUM)   or   max_i max_j s[i][j]   (DPRB_MAXSIM_MAX)
 * with the reference's zero-vector padding: a masked passage token (d_mask 0) scores exactly 0 and takes part in the
 * max; a masked query token contributes exactly 0 (sum) or offers 0 (max).  Masks may be NULL (every token real).
 *   q bf16 [nq, SQ, P], d bf16 [B, SD, P] row-major, 16-byte aligned; q_mask int32 [nq, SQ], d_mask int32 [B, SD];
 *   q_index int32 [B] (device), each in [0, nq): the caller checks this (an index out of range gives a NaN score);
 *   score fp32 [B].  bf16 products, fp32 accumulation; scores are bitwise repeatable (fixed reduction order).
 * Requires P % 8 == 0, P <= 1024, 2 <= SQ, SD <= 512 (checked before any launch, return code 1). */
#define DPRB_MAXSIM_SUM 0
#define DPRB_MAXSIM_MAX 1
int dprb_maxsim_fwd(const void* q, const void* d, const int32_t* q_mask, const int32_t* d_mask, const int32_t* q_index,
                    int nq, int SQ, int B, int SD, int P, int pool, float* score, dprb_stream_t stream);

/* Expert-matched late interaction (COIL / CITADEL rerankers): the expert-id branch of expert_sim_score,
 * dpr_scale/task/citadel_eval_task.py:240-258, plus the CLS term of _eval_step (:282-283).  Query token i (1 .. SQ-1) has
 * KQ (expert id, weight) pairs, passage token j (1 .. SD-1) has KD; with s[i][j] = q[qi][i] . d[b][j],
 *   e[(i,a)][(j,b)] = s[i][j] * (wq[i][a] * wd[j][b])   where q_ids[i][a] == d_ids[j][b], exactly 0 where they differ
 *   score[b] = sum over rows (i,a) of max over columns (j,b) of e   (DPRB_MAXSIM_SUM; max over rows for DPRB_MAXSIM_MAX)
 *            + sum_k q_cls[qi][k] * d_cls[b][k]                      (fp32; only when q_cls / d_cls are given)
 * The zeros of unmatched entries take part in the max, as in the reference.  Masks enter through the weights: give a
 * masked token weight 0 on its side (its ids are then irrelevant), which reproduces the reference's zero-vector padding.
 *   q / d / q_index / score as in dprb_maxsim_fwd (q and d are the unmasked tokens);
 *   q_ids int32 / q_w fp32 [nq, SQ, KQ], d_ids int32 / d_w fp32 [B, SD, KD] (entries of token 0 are not read);
 *   q_cls bf16 [nq, Pc], d_cls bf16 [B, Pc], 16-byte aligned, or both NULL (Pc is then ignored).
 * With KQ = KD = 1, equal ids and the 0/1 masks as weights, the scores equal dprb_maxsim_fwd's bit for bit.  Bitwise
 * repeatable.  Requires P % 8 == 0, P <= 1024, 2 <= SQ, SD <= 512, 1 <= KQ, KD <= 8 and, with CLS operands,
 * Pc % 8 == 0, Pc <= 1024 (checked before any launch, return code 1). */
int dprb_maxsim_expert_fwd(const void* q, const void* d, const int32_t* q_ids, const float* q_w, const int32_t* d_ids,
                           const float* d_w, const void* q_cls, const void* d_cls, const int32_t* q_index, int nq,
                           int SQ, int B, int SD, int P, int KQ, int KD, int Pc, int pool, float* score,
                           dprb_stream_t stream);

/* SPLADE vocabulary max-pool (SPLADEEncoder.forward of dpr_scale/models/citadel_models/splade_model.py after the
 * masked-LM head's transform): the decoder GEMM with the pooling in its epilogue; the [rows, V] logits are never written.
 *   out[n, v] = log1p( max(0, max_{r in [off[n], off[n+1])} ( x[r, :K] . W[v, :K] + bias[v] ) ) )   (0: empty range)
 * This equals the reference's max over tokens 1.. of log(1 + relu(logit)) * attention_mask when the rows of sequence n
 * are its valid tokens (token 0 and masked tokens dropped): every valid token contributes log(1 + relu(l)) >= 0 and
 * every masked token exactly 0, so the masked max is log1p(relu(max over the valid tokens)), or 0 without one.
 *   x fp16 [T, ldx], W fp16 [V, ldw], row-major, 16-byte aligned; only the first K columns are read (so the CITADEL
 *   router's [T, H + 8] / [V, H + 8] operands serve with K = H);
 *   bias fp32 [V], added in fp32 in the epilogue, or NULL;
 *   off int32 [N + 1] (device), non-decreasing, off[N] <= T: the rows of sequence n are off[n] .. off[n+1] - 1; rows
 *   before off[0] are never loaded and rows from off[N] on never enter a maximum;
 *   out fp32 [N, ldo], ldo >= V: elements [N, V] are written (every one of them), columns >= V and rows >= N never.
 * fp16 products, fp32 accumulation; out is bitwise repeatable and does not depend on how the sequences are grouped into
 * calls or ordered.  Non-finite logits are out of contract.  Requires K % 8 == 0, 8 <= K <= 1024, ldx and ldw multiples
 * of 8 and at least K, V >= 1, N >= 1, ldo >= V, 0 <= T < 2^31 (checked before any launch, return code 1).  Three
 * launches: zero-fill, the pool, log1p. */
int dprb_splade_pool_fwd(const void* x, int64_t ldx, const void* W, int64_t ldw, const float* bias, const int32_t* off,
                         int64_t T, int N, int V, int K, float* out, int64_t ldo, dprb_stream_t stream);

/* COIL / CITADEL expert-index generation: the kept (token, expert) entries of one encoded batch, grouped by expert.
 * Replaces the per-entry loops of GenerateMultiVecEmbeddingsTask / GenerateMultiVecQueryEmbeddingsTask
 * (dpr_scale/task/citadel_eval_task.py:43-70, :95-102, :143-171).  Entry i = (n, s, k), i = (n*S + s)*K + k, is kept when
 *   s >= 1 and mask[n, s] != 0 and w[i] > threshold        (DPRB_EXPERT_GROUP_CONTEXT_ID: the weight test is skipped)
 * The E kept entries are written sorted by expert id (DPRB_EXPERT_GROUP_PER_SEQUENCE: by (n, expert id)), ties in
 * (n, s, k) order, which is the reference's iteration order:
 *   out_expert / out_seq / out_tok int32 [E] = ids[i], n, s;   out_w fp32 [E] = w[i];
 *   out_payload fp32 [E, P] = w[i] * float(reps[n, s, :P])   (one rounding)   or, in context-id mode, fp32 [E] =
 *   float(tokens[n, s]);   count int32 [1] = E (device).
 * Outputs must hold the worst case N*(S-1)*K entries.  ids int32 / w fp32 [N, S, K], mask int32 [N, S], tokens int32
 * [N, S] (context-id mode only, else may be NULL), reps bf16 [N, S, ldr] (not read in context-id mode), 16-byte aligned.
 * ids must lie in [0, V).  workspace: >= dprb_expert_group_workspace_bytes(N, S, K) bytes, 256-byte aligned.
 * Integer counting only: bitwise repeatable.  Requires N >= 1, N*S*K < 2^31, 1 <= K <= 8, 2 <= S <= 512, 1 <= V < 2^24
 * and, outside context-id mode, P % 8 == 0, 8 <= P <= 1024, ldr >= P, ldr % 8 == 0 (checked before any launch, return
 * code 1).  Enqueues a memset and 3 launches per radix pass (ceil(log2 V / 8) passes, plus ceil(log2 N / 8) per
 * sequence) and one gather; never synchronises. */
#define DPRB_EXPERT_GROUP_CONTEXT_ID 1
#define DPRB_EXPERT_GROUP_PER_SEQUENCE 2
int64_t dprb_expert_group_workspace_bytes(int N, int S, int K);
int dprb_expert_group(const int32_t* ids, const float* w, const int32_t* mask, const int32_t* tokens, const void* reps,
                      int64_t ldr, int N, int S, int K, int P, int V, float threshold, int flags, int32_t* count,
                      int32_t* out_expert, int32_t* out_seq, int32_t* out_tok, float* out_w, float* out_payload,
                      void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Cross-encoder sequence-classification head (reranking: dpr_scale/models/citadel_models/cross_encoder.py:21-26,
 * AutoModelForSequenceClassification under no_grad).  The caller runs the head's dense layer first, on the CLS rows
 * that dprb_encoder_fwd returns: dprb_gemm_bf16 with DPRB_EPI_F32_STORE (bf16 operands, fp32 accumulate + bias) gives
 * pre fp32 [N, H].  This entry point does the rest in fp32:
 *   logits[n, l] = tanh(pre[n, :]) . weight[l, :] + bias[l]      (bias may be NULL)
 *   score[n]     = max_l logits[n, l]                             (optional: score may be NULL)
 * It replaces, in site-packages/transformers:
 *   BERT: BertPooler.forward (models/bert/modeling_bert.py: dense -> tanh on token 0) and the dropout + classifier
 *         Linear of BertForSequenceClassification.forward (dropout is the identity in eval);
 *   RoBERTa / XLM-R: RobertaClassificationHead.forward (models/roberta/modeling_roberta.py: token 0 -> dense -> tanh
 *         -> out_proj).
 * pre and weight fp32 row-major, 16-byte aligned; requires H % 8 == 0, H <= 1024, 1 <= L <= DPRB_SEQCLS_MAX_LABELS
 * (checked before any launch, return code 1). */
#define DPRB_SEQCLS_MAX_LABELS 16
int dprb_seqcls_head_fwd(const float* pre, const float* weight, const float* bias, float* logits, float* score, int N,
                         int H, int L, dprb_stream_t stream);
/* Training the same head with one relevance label: the grouped softmax cross-entropy of a reranker trained on (question,
 * passage) groups - candidate 0 .. G-1 of group g are rows g*G .. g*G + G-1, and labels[g] names the relevant one.  With
 * t = tanh(pre), mask the dropout multiplier (keep / (1 - p), or 0) of site 4, layer 0 under dropout_seed - element
 * (n, h) of dprb_dropout_mask(keep, B*G, H, p, dropout_seed, 0, 4) - and q_g = softmax over the group's logits:
 *   logits[n]    = weight . (t[n] * mask[n]) + bias[0]           (BertForSequenceClassification's dropout + classifier,
 *                                                                 RobertaClassificationHead's dropout + out_proj)
 *   loss[0]      = mean over groups of (logsumexp_g - logits[g*G + labels[g]])
 *   dlogit[n]    = (q_g[n] - [n is the label row]) / B
 *   dpre[n, h]   = bf16(dlogit[n] * weight[h] * mask[n, h] * (1 - t[n, h]^2))      (bf16 [B*G, H], for the GEMMs)
 *   dweight[h]   = sum_n dlogit[n] * t[n, h] * mask[n, h],   dbias[0] = sum_n dlogit[n]
 * The caller back-propagates dpre through the dense layer with dprb_gemm_bf16 / dprb_colsum_bf16.  dweight, dbias and
 * loss are summed per group and then over the groups in a fixed order (no atomics): every output is bitwise repeatable.
 * A label outside [0, G) gives a NaN loss.  pre and weight fp32 row-major ([B*G, H] and [1, H]), labels int64 [B];
 * pre, weight, dpre and workspace 16-byte aligned; workspace >= dprb_seqcls_group_ce_workspace_bytes(B, H).  Requires
 * B >= 1, 2 <= G <= DPRB_SEQCLS_GROUP_MAX, H % 8 == 0, H <= 1024, 0 <= dropout_p < 1 (checked before any launch,
 * return code 1).  Two launches; never synchronises. */
#define DPRB_SEQCLS_GROUP_MAX 64
int64_t dprb_seqcls_group_ce_workspace_bytes(int B, int H);
int dprb_seqcls_group_ce(const float* pre, const float* weight, const float* bias, const int64_t* labels, int B, int G,
                         int H, float dropout_p, uint64_t dropout_seed, float* loss, float* logits, void* dpre_bf16,
                         float* dweight, float* dbias, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Brute-force retrieval : replaces search_index() of
 * dpr_scale/run_retrieval_pytorch.py:141-176 -- einsum('ik,jk->ij') in fp16 followed by torch.topk over the
 * materialised [Q, N] score matrix -- with one fused pass: the corpus is streamed once per block of 128 queries
 * through wgmma and a running top-k is kept per query; no score matrix is written.
 *   queries [Q, d], corpus [N, d]: row-major 16-bit (dtype 0 = fp16 as in build_index() :178-190, 1 = bf16),
 *   d % 8 == 0, 16-byte aligned, N < 2^31 - 256, 1 <= k <= min(N, 1024).
 *   out_scores [Q, k] fp32 (fp32-accumulated inner products, descending; equal scores, -0 and +0 included, go to
 *   the lower row id),
 *   out_index  [Q, k] int64 = corpus row id + index_offset (the shard offset of :225-227).
 *   workspace: >= dprb_search_workspace_bytes(Q, k) bytes of device memory, caller-owned.
 *   dtype | DPRB_SEARCH_RANK_FP16: rank by (and return) the score ROUNDED TO fp16 - what the reference's topk sees,
 *   because its einsum on fp16 tensors returns fp16 (:150-151).  Ids then equal the reference's wherever its fp16
 *   scores are distinct; the default ranks by the exact fp32-accumulated score (a finer, deterministic order).
 * dprb_topk_merge replaces the per-shard merge of :272-277 (topk over the concatenated shard results + gather):
 *   scores / index [Q, total] -> the k best per row (equal scores, -0 and +0 included, go to the earlier
 *   position), workspace
 *   >= dprb_topk_merge_workspace_bytes(Q, total).
 * ------------------------------------------------------------------------------------------- */
enum { DPRB_SEARCH_RANK_FP16 = 0x100 };
int64_t dprb_search_workspace_bytes(int64_t Q, int k);
int dprb_search_topk(const void* queries, const void* corpus, int dtype, int64_t Q, int64_t N, int d, int k,
                     int64_t index_offset, float* out_scores, int64_t* out_index, void* workspace,
                     int64_t workspace_bytes, dprb_stream_t stream);
int64_t dprb_topk_merge_workspace_bytes(int64_t Q, int total);
int dprb_topk_merge(const float* scores, const int64_t* index, int64_t Q, int total, int k, float* out_scores,
                    int64_t* out_index, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * COIL / CITADEL retrieval from an expert index (the search the reference's CITADELRetrievalTask delegates to its
 * inverted vector index, dpr_scale/task/citadel_retrieval_task.py:114).  For every query q of a block of Qb queries and
 * every passage row d in [0, N):
 *   score(q, d) = q_cls[q] . cls[d]                                            (only with the CLS operands)
 *               + sum over q's entries (x, u) of max(0, max over d's entries (x, v) of u . v)    (max over {} = 0)
 * and the k best rows per query, descending, ties towards the lower row; out_ids [Qb, k] int64 = row_ids[row] (or the
 * row when row_ids is NULL), out_scores [Qb, k] fp32.
 * Index: payload fp16 [E, ldp] (width P) with row int32 [E], entries sorted by expert and, within an expert, by row;
 *   tile_bounds int32 [T + 1]: the index tiles [tile_bounds[t], tile_bounds[t+1]) partition [0, E) and never split one
 *   row's entries of one expert; cls fp16 [N, ldc] (width Pc) or NULL.
 * Queries: q_payload fp16 [Eq, ldp] sorted by expert, q_seq int32 [Eq] in [0, Qb); q_cls fp16 [Qb, ldc] or NULL.
 * groups int32 [G, 4] = (section, first row, rows <= 64, first tile): section 0 = query entries [first, first + rows)
 *   of one expert paired with that expert's tiles [first tile, first tile + n); section 1 = query CLS rows with the
 *   ceil(N / 128) CLS tiles.  item_end int32 [G]: inclusive prefix sums of the n; items = item_end[G - 1].
 * Products are fp32-accumulated; every term is added as int64 fixed point at 2^-32 (the caller keeps each query's sum
 * of |terms| below 2^30), so the result is bitwise repeatable and a query's result does not depend on its block.
 * Requires P % 8 == 0, 8 <= P <= 1024 (Pc likewise), ldp >= P and ldc >= Pc multiples of 8, 1 <= N < 2^31,
 * E, Eq < 2^31, 1 <= k <= min(1024, N), 1 <= Qb <= dprb_expert_search_block_queries(N) (a fixed accumulator budget of
 * 2 GiB); checked before any launch (return code 1).  workspace: >= dprb_expert_search_workspace_bytes(N, Qb) bytes,
 * 256-byte aligned.  Enqueues two memsets and two launches; never synchronises.
 * ------------------------------------------------------------------------------------------- */
int dprb_expert_search_block_queries(int64_t N);
int64_t dprb_expert_search_workspace_bytes(int64_t N, int Qb);
int dprb_expert_search(const void* payload, const int32_t* row, const int32_t* tile_bounds, int64_t E, int T, int P,
                       int ldp, const void* cls, int Pc, int ldc, const int64_t* row_ids, int64_t N,
                       const void* q_payload, const int32_t* q_seq, int64_t Eq, const void* q_cls, int Qb,
                       const int32_t* groups, const int32_t* item_end, int G, int items, int k, float* out_scores,
                       int64_t* out_ids, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Retrieval from a sparse vocabulary index (SPLADE first-stage retrieval).  For every query q of a block of Qb queries
 * and every passage row d in [0, N):
 *   score(q, d) = sum over q's entries (t, w_q) of sum over d's postings (t, w_p) of w_q * w_p
 * and the k best rows per query, descending, ties towards the lower row; out_ids [Qb, k] int64 = row_ids[row] (or the
 * row when row_ids is NULL), out_scores [Qb, k] fp32.
 * Index: postings sorted by term and, within a term, by row: row int32 [nnz] in [0, N), weight fp16 [nnz]; both
 *   16-byte aligned and allocated for nnz rounded up to a multiple of 8 entries (the padding is read, never used);
 *   term_ptr int64 [V + 1]: term t's postings are [term_ptr[t], term_ptr[t + 1]).
 * Queries: q_term int32 [Eq] in [0, V), q_weight fp32 [Eq], q_seq int32 [Eq] in [0, Qb) (entries in any order; a
 *   term may repeat).  Each entry's postings are cut into ceil(len / DPRB_SPARSE_SEARCH_TILE) tiles; item_end int32
 *   [Eq]: inclusive prefix sums of the entries' tile counts; items = item_end[Eq - 1].
 * Every product w_q * w_p is formed in fp32 and added as int64 fixed point at 2^-32 (the caller keeps each query's sum
 * of |products| below 2^30), so the result is bitwise repeatable and a query's result does not depend on its block.
 * Requires 1 <= N < 2^31, V >= 1, 0 <= nnz < 2^40, Eq >= 0, 1 <= k <= min(1024, N),
 * 1 <= Qb <= dprb_sparse_search_block_queries(N) (a fixed accumulator budget of 2 GiB); checked before any launch
 * (return code 1).  workspace: >= dprb_sparse_search_workspace_bytes(N, Qb) bytes, 256-byte aligned.  Enqueues two
 * memsets and two launches; never synchronises.
 * ------------------------------------------------------------------------------------------- */
enum { DPRB_SPARSE_SEARCH_TILE = 2048 };
int dprb_sparse_search_block_queries(int64_t N);
int64_t dprb_sparse_search_workspace_bytes(int64_t N, int Qb);
int dprb_sparse_search(const int32_t* row, const void* weight, const int64_t* term_ptr, int64_t nnz, int V,
                       const int64_t* row_ids, int64_t N, const int32_t* q_term, const float* q_weight,
                       const int32_t* q_seq, const int32_t* item_end, int Eq, int items, int Qb, int k,
                       float* out_scores, int64_t* out_ids, void* workspace, int64_t workspace_bytes,
                       dprb_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Squared-error sum for query-encoder distillation (MSELoss(reduction="sum") of the reference's DPRDistillTask,
 * dpr_scale/task/dpr_distill_task.py:43, :167, :186, and the gradient autograd takes through it):
 *   loss_sum[0] = sum_{r < rows, c < d} (x[r, c] - t[r, c])^2
 *   dx[r, c]    = 2 (x[r, c] - t[r, c])            (only when dx is not NULL; evaluation passes NULL)
 * x, t, dx fp32 row-major with row strides ldx, ldt, lddx (elements).  dx equals fp32 2 * (x - t) bit for bit; the
 * squares are rounded to fp32 and summed in double, per block and then over the blocks' partials in a fixed order
 * (no atomics), so loss_sum is bitwise repeatable.  16-byte loads when d, the strides and the pointers allow them.
 * workspace: >= dprb_sqerr_workspace_bytes(rows, d) bytes, 8-byte aligned.  Requires rows >= 0, d >= 1, strides at
 * least d (checked before any launch, return code 1).  Enqueues two launches (one when rows == 0, which writes 0);
 * never synchronises.
 * ------------------------------------------------------------------------------------------- */
int64_t dprb_sqerr_workspace_bytes(int rows, int d);
int dprb_sqerr_fwd(const float* x, int64_t ldx, const float* t, int64_t ldt, int rows, int d, float* loss_sum, float* dx,
                   int64_t lddx, void* workspace, int64_t workspace_bytes, dprb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DPRB_H_ */
