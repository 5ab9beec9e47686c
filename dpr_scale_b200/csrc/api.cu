// C-ABI surface of libdprb.so (declared in include/dprb.h): thin extern "C" shims over the C++
// launchers, plus the thread-local error string.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {

static thread_local char g_err[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

}  // namespace dprb

using namespace dprb;
#define S(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

int dprb_version(void) { return DPRB_VERSION; }
const char* dprb_last_error(void) { return g_err; }
int dprb_num_sms(void) { return num_sms(); }
int64_t dprb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int dprb_gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int64_t lda, int64_t ldb,
                   int64_t ldd, int a_mn_major, int b_mn_major, int epilogue, const float* bias, const void* aux,
                   int64_t ld_aux, void* out2, float alpha, int splits, float* colsum, float dropout_p,
                   uint64_t dropout_site_seed, dprb_stream_t stream) {
  return gemm_bf16(A, B, D, M, N, K, lda, ldb, ldd, a_mn_major, b_mn_major, epilogue, bias, aux, ld_aux, out2,
                   alpha, splits, colsum, dropout_p, dropout_site_seed, S(stream));
}

int dprb_gemm_profile_enable(int enable, int max_launches) { return gemm_profile_enable(enable, max_launches); }
int dprb_gemm_profile_read(double* total_ms, double* total_flops, int64_t* launches) {
  long long n = 0;
  int rc = gemm_profile_read(total_ms, total_flops, &n);
  if (launches) *launches = n;
  return rc;
}

int dprb_embed_ln_fwd(const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids, const float* word,
                      const float* pos, const float* type, const float* gamma, const float* beta, void* y,
                      float* stats, int T, int H, int vocab, int max_pos, int type_vocab, float eps,
                      float dropout_p, uint64_t dropout_seed, void* y_res, dprb_stream_t stream) {
  return embed_ln_fwd(ids, type_ids, pos_ids, word, pos, type, gamma, beta, y, stats, T, H, vocab, max_pos,
                      type_vocab, eps, dropout_p, dropout_seed, y_res, S(stream));
}
int dprb_embed_ln_bwd(const void* dy, const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids,
                      const float* word, const float* pos, const float* type, const float* gamma,
                      const float* stats, float* dword, float* dpos, float* dtype, float* dgamma, float* dbeta,
                      int T, int H, float dropout_p, uint64_t dropout_seed, dprb_stream_t stream) {
  return embed_ln_bwd(dy, ids, type_ids, pos_ids, word, pos, type, gamma, stats, dword, dpos, dtype, dgamma,
                      dbeta, T, H, dropout_p, dropout_seed, S(stream));
}
int dprb_ln_fwd(const void* z, const float* gamma, const float* beta, void* y, float* stats, float* cls_out,
                int cls_stride, int T, int H, float eps, int z_f16, void* y_res, dprb_stream_t stream) {
  return ln_fwd(z, gamma, beta, y, stats, cls_out, cls_stride, T, H, eps, z_f16, y_res, S(stream));
}
int dprb_ln_bwd(const void* dy, const float* dy_cls, int cls_stride, const void* z, const float* stats,
                const float* gamma, void* dz, float* dgamma, float* dbeta, float* dbias, int T, int H, void* dzm,
                float dropout_p, uint64_t dropout_site_seed, int z_f16, dprb_stream_t stream) {
  return ln_bwd(dy, dy_cls, cls_stride, z, stats, gamma, dz, dgamma, dbeta, dbias, T, H, dzm, dropout_p,
                dropout_site_seed, z_f16, S(stream));
}
uint64_t dprb_dropout_site_seed(uint64_t dropout_seed, int layer, int site) {
  return drop_site_seed64(dropout_seed, layer, site);
}
int dprb_dropout_mask(uint8_t* keep, int64_t rows, int cols, float dropout_p, uint64_t dropout_seed, int layer,
                      int site, dprb_stream_t stream) {
  return dropout_mask(keep, rows, cols, dropout_p, dropout_seed, layer, site, S(stream));
}
int dprb_gelu_from_pre(const void* pre, void* out, int64_t n, dprb_stream_t stream) {
  return gelu_from_pre(pre, out, n, S(stream));
}
int dprb_colsum_bf16(const void* x, int64_t ld, float* out, int T, int N, dprb_stream_t stream) {
  return colsum_bf16(x, ld, out, T, N, S(stream));
}
int dprb_attn_fwd(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int Sq, int heads,
                  float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream) {
  return attn_fwd_lse(qkv, attn_mask, ctx, lse, nseq, Sq, heads, dropout_p, dropout_site_seed, S(stream));
}
int dprb_attn_bwd(const void* qkv, const int32_t* attn_mask, const void* ctx, const float* lse, const void* dctx,
                  void* dqkv, float* dbias, int nseq, int Sq, int heads, float dropout_p,
                  uint64_t dropout_site_seed, dprb_stream_t stream) {
  return attn_bwd_lse(qkv, attn_mask, ctx, lse, dctx, dqkv, dbias, nseq, Sq, heads, dropout_p, dropout_site_seed,
                      S(stream));
}
int dprb_attn_cls_fwd(const void* qkv, const int32_t* attn_mask, void* ctx_cls, float* probs, int nseq, int Sq,
                      int heads, float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream) {
  return attn_cls_fwd(qkv, attn_mask, ctx_cls, probs, nseq, Sq, heads, dropout_p, dropout_site_seed, S(stream));
}
int dprb_attn_cls_bwd(const void* qkv, const float* probs, const void* dctx_cls, void* dqkv, int nseq, int Sq,
                      int heads, float dropout_p, uint64_t dropout_site_seed, dprb_stream_t stream) {
  return attn_cls_bwd(qkv, probs, dctx_cls, dqkv, nseq, Sq, heads, dropout_p, dropout_site_seed, S(stream));
}
int64_t dprb_score_tc_workspace_bytes(int Q, int C, int d, int nq, int nc) {
  return score_tc_workspace_bytes(Q, C, d, nq, nc);
}
int dprb_score_tc_fwd(const float* q, const float* c, const uint8_t* col_mask, const uint8_t* pair_mask,
                      const int64_t* labels, float inv_temperature, float* lse, float* loss_sum, float* logits, int Q,
                      int C, int d, int nq, int nc, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return score_tc_fwd(q, c, col_mask, pair_mask, labels, inv_temperature, lse, loss_sum, logits, Q, C, d, nq, nc,
                      workspace, workspace_bytes, S(stream));
}
int dprb_score_tc_bwd(const uint8_t* col_mask, const uint8_t* pair_mask, const int64_t* labels, const float* lse,
                      float grad_scale, float inv_temperature, float* dq, float* dc, int Q, int C, int d, int q0, int nq,
                      int c0, int nc, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return score_tc_bwd(col_mask, pair_mask, labels, lse, grad_scale, inv_temperature, dq, dc, Q, C, d, q0, nq, c0, nc,
                      workspace, workspace_bytes, S(stream));
}
int dprb_sumsq_f32(const float* g, int64_t n, float* out, dprb_stream_t stream) {
  return sumsq_f32(g, n, out, S(stream));
}
int dprb_adamw_step(float* p, const float* g, float* m, float* v, void* shadow, int64_t n, float lr, float beta1,
                    float beta2, float eps, float weight_decay, int step, float grad_scale, const float* sumsq,
                    float max_norm, dprb_stream_t stream) {
  return adamw_step(p, g, m, v, shadow, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale, sumsq,
                    max_norm, S(stream));
}
int64_t dprb_lamb_workspace_bytes(int nchunks, int nseg) { return lamb_workspace_bytes(nchunks, nseg); }
int dprb_lamb_step(float* p, const float* g, float* m, float* v, void* shadow, int64_t n, const int64_t* plan,
                   int nchunks, int nseg, float lr, float beta1, float beta2, float eps, float weight_decay,
                   float clamp_value, int adam, int debias, int step, float grad_scale, const float* sumsq,
                   float max_norm, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return lamb_step(p, g, m, v, shadow, n, reinterpret_cast<const long long*>(plan), nchunks, nseg, lr, beta1, beta2,
                   eps, weight_decay, clamp_value, adam, debias, step, grad_scale, sumsq, max_norm, workspace,
                   workspace_bytes, S(stream));
}
int dprb_madgrad_step(float* p, const float* g, float* grad_sum_sq, float* s, const float* x0, void* shadow, int64_t n,
                      float lr, float momentum, float weight_decay, float eps, int k, float grad_scale,
                      const float* sumsq, float max_norm, dprb_stream_t stream) {
  return madgrad_step(p, g, grad_sum_sq, s, x0, shadow, n, lr, momentum, weight_decay, eps, k, grad_scale, sumsq,
                      max_norm, S(stream));
}
int dprb_cast_f32_bf16(const float* src, void* dst, int64_t n, dprb_stream_t stream) {
  return cast_f32_bf16(src, dst, n, S(stream));
}
int dprb_cast_bf16_f32(const void* src, float* dst, int64_t n, dprb_stream_t stream) {
  return cast_bf16_f32(src, dst, n, S(stream));
}
int64_t dprb_encoder_workspace_bytes(const dprb_encoder_weights* w, int nseq, int Sq, int save) {
  return encoder_workspace_bytes(w, nseq, Sq, save);
}
int dprb_encoder_fwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, float* pooled,
                     dprb_stream_t stream) {
  return encoder_fwd(w, b, pooled, S(stream));
}
int dprb_encoder_bwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, const float* dpooled,
                     int layer_lo, int layer_hi, dprb_stream_t stream) {
  return encoder_bwd(w, b, dpooled, layer_lo, layer_hi, S(stream));
}
int dprb_encoder_fwd_tokens(const dprb_encoder_weights* w, const dprb_encoder_batch* b, void* tokens,
                            dprb_stream_t stream) {
  return encoder_fwd_tokens(w, b, tokens, S(stream));
}
int dprb_maxsim_fwd(const void* q, const void* d, const int32_t* q_mask, const int32_t* d_mask, const int32_t* q_index,
                    int nq, int SQ, int B, int SD, int P, int pool, float* score, dprb_stream_t stream) {
  return maxsim_fwd(q, d, q_mask, d_mask, q_index, nq, SQ, B, SD, P, pool, score, S(stream));
}
int dprb_maxsim_expert_fwd(const void* q, const void* d, const int32_t* q_ids, const float* q_w, const int32_t* d_ids,
                           const float* d_w, const void* q_cls, const void* d_cls, const int32_t* q_index, int nq,
                           int SQ, int B, int SD, int P, int KQ, int KD, int Pc, int pool, float* score,
                           dprb_stream_t stream) {
  return maxsim_expert_fwd(q, d, q_ids, q_w, d_ids, d_w, q_cls, d_cls, q_index, nq, SQ, B, SD, P, KQ, KD, Pc, pool,
                           score, S(stream));
}
int dprb_splade_pool_fwd(const void* x, int64_t ldx, const void* W, int64_t ldw, const float* bias, const int32_t* off,
                         int64_t T, int N, int V, int K, float* out, int64_t ldo, dprb_stream_t stream) {
  return splade_pool_fwd(x, ldx, W, ldw, bias, off, T, N, V, K, out, ldo, S(stream));
}
int64_t dprb_expert_group_workspace_bytes(int N, int S_, int K) { return expert_group_workspace_bytes(N, S_, K); }
int dprb_expert_group(const int32_t* ids, const float* w, const int32_t* mask, const int32_t* tokens, const void* reps,
                      int64_t ldr, int N, int S_, int K, int P, int V, float threshold, int flags, int32_t* count,
                      int32_t* out_expert, int32_t* out_seq, int32_t* out_tok, float* out_w, float* out_payload,
                      void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return expert_group(ids, w, mask, tokens, reps, ldr, N, S_, K, P, V, threshold, flags, count, out_expert, out_seq,
                      out_tok, out_w, out_payload, workspace, workspace_bytes, S(stream));
}
int dprb_seqcls_head_fwd(const float* pre, const float* weight, const float* bias, float* logits, float* score, int N,
                         int H, int L, dprb_stream_t stream) {
  return seqcls_head_fwd(pre, weight, bias, logits, score, N, H, L, S(stream));
}
int64_t dprb_seqcls_group_ce_workspace_bytes(int B, int H) { return seqcls_group_ce_workspace_bytes(B, H); }
int dprb_seqcls_group_ce(const float* pre, const float* weight, const float* bias, const int64_t* labels, int B, int G,
                         int H, float dropout_p, uint64_t dropout_seed, float* loss, float* logits, void* dpre_bf16,
                         float* dweight, float* dbias, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return seqcls_group_ce(pre, weight, bias, reinterpret_cast<const long long*>(labels), B, G, H, dropout_p,
                         dropout_seed, loss, logits, dpre_bf16, dweight, dbias, workspace, workspace_bytes, S(stream));
}
int64_t dprb_search_workspace_bytes(int64_t Q, int k) { return search_workspace_bytes(Q, k); }
int dprb_search_topk(const void* queries, const void* corpus, int dtype, int64_t Q, int64_t N, int d, int k,
                     int64_t index_offset, float* out_scores, int64_t* out_index, void* workspace,
                     int64_t workspace_bytes, dprb_stream_t stream) {
  return search_topk(queries, corpus, dtype, Q, N, d, k, index_offset, out_scores,
                     reinterpret_cast<long long*>(out_index), workspace, workspace_bytes, S(stream));
}
int64_t dprb_topk_merge_workspace_bytes(int64_t Q, int total) { return topk_merge_workspace_bytes(Q, total); }
int dprb_topk_merge(const float* scores, const int64_t* index, int64_t Q, int total, int k, float* out_scores,
                    int64_t* out_index, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return topk_merge(scores, reinterpret_cast<const long long*>(index), Q, total, k, out_scores,
                    reinterpret_cast<long long*>(out_index), workspace, workspace_bytes, S(stream));
}

int dprb_expert_search_block_queries(int64_t N) { return expert_search_block_queries(N); }
int64_t dprb_expert_search_workspace_bytes(int64_t N, int Qb) { return expert_search_workspace_bytes(N, Qb); }
int dprb_expert_search(const void* payload, const int32_t* row, const int32_t* tile_bounds, int64_t E, int T, int P,
                       int ldp, const void* cls, int Pc, int ldc, const int64_t* row_ids, int64_t N,
                       const void* q_payload, const int32_t* q_seq, int64_t Eq, const void* q_cls, int Qb,
                       const int32_t* groups, const int32_t* item_end, int G, int items, int k, float* out_scores,
                       int64_t* out_ids, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return expert_search(payload, row, tile_bounds, E, T, P, ldp, cls, Pc, ldc, reinterpret_cast<const long long*>(row_ids),
                       N, q_payload, q_seq, Eq, q_cls, Qb, groups, item_end, G, items, k, out_scores,
                       reinterpret_cast<long long*>(out_ids), workspace, workspace_bytes, S(stream));
}

int dprb_sparse_search_block_queries(int64_t N) { return sparse_search_block_queries(N); }
int64_t dprb_sparse_search_workspace_bytes(int64_t N, int Qb) { return sparse_search_workspace_bytes(N, Qb); }
int dprb_sparse_search(const int32_t* row, const void* weight, const int64_t* term_ptr, int64_t nnz, int V,
                       const int64_t* row_ids, int64_t N, const int32_t* q_term, const float* q_weight,
                       const int32_t* q_seq, const int32_t* item_end, int Eq, int items, int Qb, int k,
                       float* out_scores, int64_t* out_ids, void* workspace, int64_t workspace_bytes,
                       dprb_stream_t stream) {
  return sparse_search(row, weight, reinterpret_cast<const long long*>(term_ptr), nnz, V,
                       reinterpret_cast<const long long*>(row_ids), N, q_term, q_weight, q_seq, item_end, Eq, items,
                       Qb, k, out_scores, reinterpret_cast<long long*>(out_ids), workspace, workspace_bytes, S(stream));
}

int64_t dprb_sqerr_workspace_bytes(int rows, int d) {
  (void)d;
  return sqerr_workspace_bytes(rows);
}
int dprb_sqerr_fwd(const float* x, int64_t ldx, const float* t, int64_t ldt, int rows, int d, float* loss_sum, float* dx,
                   int64_t lddx, void* workspace, int64_t workspace_bytes, dprb_stream_t stream) {
  return sqerr_fwd(x, ldx, t, ldt, rows, d, loss_sum, dx, lddx, workspace, workspace_bytes, S(stream));
}

}  // extern "C"
