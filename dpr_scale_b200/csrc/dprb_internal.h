// Internal C++ declarations shared by the kernel translation units of libdprb.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/dprb.h"

namespace dprb {

// host.cu: a tiled tensor map of rank 2 or 3 (dims, box: innermost first; strides: bytes, rank - 1 of them), always
// 128B-swizzled, non-interleaved, out-of-bounds elements read as zero.  Binds the primary context to the calling
// thread first.  Returns 0, or an error code with the message set (`what` names the caller in it).
int encode_tmap(CUtensorMap* out, const char* what, CUtensorMapDataType dtype, int rank, const void* base,
                const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                CUtensorMapL2promotion l2);

// Bump allocator over a caller-owned workspace: every buffer starts 256-byte aligned.  With a null base it only
// measures (take returns null, off still grows), which is how the *_workspace_bytes functions size a workspace.
struct Carve {
  uint8_t* base;
  long long off;
  explicit Carve(void* b) : base(reinterpret_cast<uint8_t*>(b)), off(0) {}
  void* take(long long bytes) {
    void* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~255LL;
    return p;
  }
};

int gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, long long lda, long long ldb,
              long long ldd, int a_mn_major, int b_mn_major, int epilogue, const float* bias, const void* aux,
              long long ld_aux, void* out2, float alpha, int splits, float* colsum, float dropout_p,
              unsigned long long drop_site_seed, cudaStream_t stream);

int gemm_profile_enable(int enable, int max_launches);
int gemm_profile_read(double* total_ms, double* total_flops, long long* launches);

int embed_ln_fwd(const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids, const float* word,
                 const float* pos, const float* type, const float* gamma, const float* beta, void* y, float* stats,
                 int T, int H, int vocab, int max_pos, int type_vocab, float eps, float dropout_p,
                 unsigned long long seed, void* y_res, cudaStream_t stream);
int embed_ln_bwd(const void* dy, const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids,
                 const float* word, const float* pos, const float* type, const float* gamma, const float* stats,
                 float* dword, float* dpos, float* dtype, float* dgamma, float* dbeta, int T, int H,
                 float dropout_p, unsigned long long seed, cudaStream_t stream);
int ln_fwd(const void* z, const float* gamma, const float* beta, void* y, float* stats, float* cls_out,
           int cls_stride, int T, int H, float eps, int z_f16, void* y_res, cudaStream_t stream);
int ln_bwd(const void* dy, const float* dy_cls, int cls_stride, const void* z, const float* stats,
           const float* gamma, void* dz, float* dgamma, float* dbeta, float* dbias, int T, int H, void* dzm,
           float dropout_p, unsigned long long site_seed, int z_f16, cudaStream_t stream);
int dropout_mask(uint8_t* out, long long rows, int cols, float p, unsigned long long seed, int layer, int site,
                 cudaStream_t stream);
unsigned long long drop_site_seed(unsigned long long seed, int layer, int site);
int gelu_from_pre(const void* pre, void* out, long long n, cudaStream_t stream);
int colsum_bf16(const void* x, long long ld, float* out, int T, int N, cudaStream_t stream);

int attn_fwd_lse(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                 float dropout_p, unsigned long long site_seed, cudaStream_t stream);
int attn_bwd_lse(const void* qkv, const int32_t* attn_mask, const void* ctx, const float* lse, const void* dctx,
                 void* dqkv, float* dbias, int nseq, int S, int heads, float dropout_p,
                 unsigned long long site_seed, cudaStream_t stream);

int attn_fwd_wg(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                float dropout_p, unsigned long long site_seed, cudaStream_t stream);
// adds the QKV bias gradient into dbias when it is given
int attn_bwd_wg(const void* qkv, const int32_t* attn_mask, const float* lse, const void* dctx,
                void* dqkv, float* dbias, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                cudaStream_t stream);

int attn_cls_fwd(const void* qkv, const int32_t* attn_mask, void* ctx_cls, float* probs, int nseq, int S, int heads,
                 float dropout_p, unsigned long long site_seed, cudaStream_t stream);
int attn_cls_bwd(const void* qkv, const float* probs, const void* dctx_cls, void* dqkv, int nseq, int S, int heads,
                 float dropout_p, unsigned long long site_seed, cudaStream_t stream);
int add_rows_bf16(void* dst, const void* src, int nrows, int H, long long stride_rows, cudaStream_t stream);

long long score_tc_workspace_bytes(int Q, int C, int d, int nq, int nc);
int score_tc_fwd(const float* q, const float* c, const uint8_t* col_mask, const uint8_t* pair_mask,
                 const int64_t* labels, float inv_t, float* lse, float* loss_sum, float* logits, int Q, int C, int d,
                 int nq, int nc, void* workspace, long long workspace_bytes, cudaStream_t stream);
int score_tc_bwd(const uint8_t* col_mask, const uint8_t* pair_mask, const int64_t* labels, const float* lse,
                 float grad_scale, float inv_t, float* dq, float* dc, int Q, int C, int d, int q0, int nq, int c0, int nc,
                 void* workspace, long long workspace_bytes, cudaStream_t stream);

int sumsq_f32(const float* g, long long n, float* out, cudaStream_t stream);
int adamw_step(float* p, const float* g, float* m, float* v, void* shadow, long long n, float lr, float beta1,
               float beta2, float eps, float wd, int step, float grad_scale, const float* sumsq, float max_norm,
               cudaStream_t stream);
long long lamb_workspace_bytes(int nchunks, int nseg);
int lamb_step(float* p, const float* g, float* m, float* v, void* shadow, long long n, const long long* plan,
              int nchunks, int nseg, float lr, float beta1, float beta2, float eps, float wd, float clamp_value,
              int adam, int debias, int step, float grad_scale, const float* sumsq, float max_norm, void* workspace,
              long long workspace_bytes, cudaStream_t stream);
int madgrad_step(float* p, const float* g, float* nu, float* s, const float* x0, void* shadow, long long n, float lr,
                 float momentum, float wd, float eps, int k, float grad_scale, const float* sumsq, float max_norm,
                 cudaStream_t stream);
int cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t stream);
int cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t stream);

long long search_workspace_bytes(long long Q, int k);
int search_topk(const void* queries, const void* corpus, int dtype, long long Q, long long N, int d, int k,
                long long index_offset, float* out_scores, long long* out_index, void* workspace,
                long long workspace_bytes, cudaStream_t stream);
long long topk_merge_workspace_bytes(long long Q, int total);
int topk_merge(const float* scores, const long long* index, long long Q, int total, int k, float* out_scores,
               long long* out_index, void* workspace, long long workspace_bytes, cudaStream_t stream);

int seqcls_head_fwd(const float* pre, const float* weight, const float* bias, float* logits, float* score, int N,
                    int H, int L, cudaStream_t stream);
long long seqcls_group_ce_workspace_bytes(int B, int H);
int seqcls_group_ce(const float* pre, const float* weight, const float* bias, const long long* labels, int B, int G,
                    int H, float dropout_p, unsigned long long dropout_seed, float* loss, float* logits, void* dpre,
                    float* dweight, float* dbias, void* workspace, long long workspace_bytes, cudaStream_t stream);

long long encoder_workspace_bytes(const dprb_encoder_weights* w, int nseq, int S, int save);
int encoder_fwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, float* pooled, cudaStream_t stream);
int encoder_bwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, const float* dpooled, int layer_lo,
                int layer_hi, cudaStream_t stream);
int encoder_fwd_tokens(const dprb_encoder_weights* w, const dprb_encoder_batch* b, void* tokens, cudaStream_t stream);

int maxsim_fwd(const void* q, const void* d, const int32_t* q_mask, const int32_t* d_mask, const int32_t* q_index,
               int nq, int SQ, int B, int SD, int P, int pool, float* score, cudaStream_t stream);
int maxsim_expert_fwd(const void* q, const void* d, const int32_t* q_ids, const float* q_w, const int32_t* d_ids,
                      const float* d_w, const void* q_cls, const void* d_cls, const int32_t* q_index, int nq, int SQ,
                      int B, int SD, int P, int KQ, int KD, int Pc, int pool, float* score, cudaStream_t stream);

int splade_pool_fwd(const void* x, long long ldx, const void* W, long long ldw, const float* bias, const int32_t* off,
                    long long T, int N, int V, int K, float* out, long long ldo, cudaStream_t stream);

long long expert_group_workspace_bytes(int N, int S, int K);
int expert_group(const int32_t* ids, const float* w, const int32_t* mask, const int32_t* tokens, const void* reps,
                 long long ldr, int N, int S, int K, int P, int V, float threshold, int flags, int32_t* count,
                 int32_t* out_expert, int32_t* out_seq, int32_t* out_tok, float* out_w, float* out_payload,
                 void* workspace, long long workspace_bytes, cudaStream_t stream);

// fixed_select.cu: the int64 fixed-point accumulator [Qb, N] at 2^-32 of the index searches, and its per-query top-k.
// fixed_acc_init carves the accumulator and a work counter from the workspace and zeroes both on the stream;
// fixed_acc_select writes the k best rows of every query (descending, ties towards the lower row), as row_ids[row].
struct FixedAcc {
  unsigned long long* acc;
  int* counter;
};
int fixed_acc_block_queries(long long N);
long long fixed_acc_workspace_bytes(long long N, int Qb);
int fixed_acc_init(void* workspace, long long N, int Qb, FixedAcc* out, cudaStream_t stream);
int fixed_acc_select(const unsigned long long* acc, long long N, int Qb, int k, const long long* row_ids,
                     float* out_scores, long long* out_ids, cudaStream_t stream);

int expert_search_block_queries(long long N);
long long expert_search_workspace_bytes(long long N, int Qb);
int expert_search(const void* payload, const int32_t* row, const int32_t* tile_bounds, long long E, int T, int P,
                  int ldp, const void* cls, int Pc, int ldc, const long long* row_ids, long long N,
                  const void* q_payload, const int32_t* q_seq, long long Eq, const void* q_cls, int Qb,
                  const int32_t* groups, const int32_t* item_end, int G, int items, int k, float* out_scores,
                  long long* out_ids, void* workspace, long long workspace_bytes, cudaStream_t stream);

int sparse_search_block_queries(long long N);
long long sparse_search_workspace_bytes(long long N, int Qb);
int sparse_search(const int32_t* row, const void* weight, const long long* term_ptr, long long nnz, int V,
                  const long long* row_ids, long long N, const int32_t* q_term, const float* q_weight,
                  const int32_t* q_seq, const int32_t* item_end, int Eq, int items, int Qb, int k, float* out_scores,
                  long long* out_ids, void* workspace, long long workspace_bytes, cudaStream_t stream);

long long sqerr_workspace_bytes(int rows);
int sqerr_fwd(const float* x, long long ldx, const float* t, long long ldt, int rows, int d, float* loss_sum, float* dx,
              long long lddx, void* workspace, long long workspace_bytes, cudaStream_t stream);

}  // namespace dprb
