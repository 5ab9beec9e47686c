// Whole-encoder forward / backward orchestration: the BERT/RoBERTa layer stack as a fixed sequence of
// dprb kernels on one stream, no host synchronisation, activations saved in a caller-owned workspace.
//
// Replaces BertModel.forward (site-packages/transformers/models/bert/modeling_bert.py:628-691, layer
// loop :440-448, BertLayer :359-421) + CLS pooling of /root/reference/dpr_scale/models/hf_model.py:36-41
// and the autograd backward Lightning runs after dpr_scale/task/dpr_task.py:153-214.
// The HF pooler (modeling_bert.py:462-468) is not computed: hf_model.py:39 discards it.
#include <cstdlib>
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

struct LayerActs {
  bf16 *qkv, *ctx, *z1, *x1, *hpre, *hact, *z2, *out;
  float *lse, *stats1, *stats2;
};

struct Workspace {
  bf16 *rA, *rB;   // fp16 residual-stream copies of the LayerNorm outputs (forward only, not saved)
  bf16 *ctx_t, *hact_t;  // lean mode: ONE attention-output / GELU-output buffer shared by all layers (rebuilt in backward)
  int lean;
  bf16* x0;
  float* emb_stats;
  int n_layer_slots;
  LayerActs slot[64];
  // backward scratch
  bf16 *gA, *gB, *gB2, *gH, *gQKV;
  long long bytes;
};

int plan(const dprb_encoder_weights* w, int nseq, int S, int save, void* base, Workspace* ws) {
  DPRB_REQUIRE(w->layers >= 1 && w->layers <= 64, "encoder: layers=%d unsupported", w->layers);
  DPRB_REQUIRE(w->hidden % 8 == 0 && w->inter % 8 == 0 && w->hidden <= 1024, "encoder: H=%d I=%d unsupported", w->hidden, w->inter);
  DPRB_REQUIRE(w->heads * 64 == w->hidden, "encoder: head_dim must be 64 (H=%d heads=%d)", w->hidden, w->heads);
  DPRB_REQUIRE(S <= 512, "encoder: sequence length %d unsupported (at most 512)", S);
  const long long T = (long long)nseq * S, H = w->hidden, I = w->inter;
  Carve c(base);
  ws->rA = (bf16*)c.take(T * H * 2);
  ws->rB = (bf16*)c.take(T * H * 2);
  ws->x0 = (bf16*)c.take(T * H * 2);
  ws->emb_stats = (float*)c.take(T * 2 * 4);
  ws->n_layer_slots = save ? w->layers : 2;
  ws->lean = (save == 2);
  ws->ctx_t = ws->lean ? (bf16*)c.take(T * H * 2) : nullptr;
  ws->hact_t = ws->lean ? (bf16*)c.take(T * I * 2) : nullptr;
  for (int i = 0; i < ws->n_layer_slots; ++i) {
    LayerActs& a = ws->slot[i];
    a.qkv = (bf16*)c.take(T * 3 * H * 2);
    a.ctx = ws->lean ? ws->ctx_t : (bf16*)c.take(T * H * 2);
    a.lse = (float*)c.take((long long)nseq * w->heads * S * 4);
    a.z1 = (bf16*)c.take(T * H * 2);
    a.stats1 = (float*)c.take(T * 2 * 4);
    a.x1 = (bf16*)c.take(T * H * 2);
    a.hpre = save ? (bf16*)c.take(T * I * 2) : nullptr;     // gelu'(pre), or pre itself in lean mode
    a.hact = ws->lean ? ws->hact_t : (bf16*)c.take(T * I * 2);
    a.z2 = (bf16*)c.take(T * H * 2);
    a.stats2 = (float*)c.take(T * 2 * 4);
    a.out = (bf16*)c.take(T * H * 2);
  }
  if (save) {
    ws->gA = (bf16*)c.take(T * H * 2);
    ws->gB = (bf16*)c.take(T * H * 2);
    ws->gB2 = (bf16*)c.take(T * H * 2);  // dz * mask/(1-p): the Linear-side gradient when hidden dropout is on
    ws->gH = (bf16*)c.take(T * I * 2);
    ws->gQKV = (bf16*)c.take(T * 3 * H * 2);
  } else {
    ws->gA = ws->gB = ws->gB2 = ws->gH = ws->gQKV = nullptr;
  }
  ws->bytes = c.off;
  return 0;
}

struct LayerW {
  const bf16 *wqkv, *wo, *w1, *w2;                                  // bf16 shadow
  const float *bqkv, *bo, *ln1g, *ln1b, *b1, *b2, *ln2g, *ln2b;     // fp32 master
  float *g_wqkv, *g_bqkv, *g_wo, *g_bo, *g_ln1g, *g_ln1b, *g_w1, *g_b1, *g_w2, *g_b2, *g_ln2g, *g_ln2b;
};

LayerW layer_w(const dprb_encoder_weights* w, int l) {
  const long long b = w->off_layer0 + (long long)l * w->layer_stride;
  const bf16* sh = reinterpret_cast<const bf16*>(w->shadow);
  const float* ms = w->master;
  float* gr = w->grads;
  LayerW r;
  r.wqkv = sh + b + w->rel_wqkv; r.wo = sh + b + w->rel_wo; r.w1 = sh + b + w->rel_w1; r.w2 = sh + b + w->rel_w2;
  r.bqkv = ms + b + w->rel_bqkv; r.bo = ms + b + w->rel_bo; r.ln1g = ms + b + w->rel_ln1_g; r.ln1b = ms + b + w->rel_ln1_b;
  r.b1 = ms + b + w->rel_b1; r.b2 = ms + b + w->rel_b2; r.ln2g = ms + b + w->rel_ln2_g; r.ln2b = ms + b + w->rel_ln2_b;
  if (gr != nullptr) {
    r.g_wqkv = gr + b + w->rel_wqkv; r.g_bqkv = gr + b + w->rel_bqkv; r.g_wo = gr + b + w->rel_wo; r.g_bo = gr + b + w->rel_bo;
    r.g_ln1g = gr + b + w->rel_ln1_g; r.g_ln1b = gr + b + w->rel_ln1_b; r.g_w1 = gr + b + w->rel_w1; r.g_b1 = gr + b + w->rel_b1;
    r.g_w2 = gr + b + w->rel_w2; r.g_b2 = gr + b + w->rel_b2; r.g_ln2g = gr + b + w->rel_ln2_g; r.g_ln2b = gr + b + w->rel_ln2_b;
  }
  return r;
}

unsigned long long site_seed(const dprb_encoder_batch* b, int layer, int site) {
  return drop_site_seed64(b->dropout_seed, layer, site);
}

// site seed with the row-key multiplier S in the high word: rows of the pruned last layer are CLS rows (token r*S)
unsigned long long site_seed_cls(const dprb_encoder_batch* b, int layer, int site) {
  return drop_site_seed64(b->dropout_seed, layer, site) | ((unsigned long long)b->S << 32);
}
bool prune_last_layer() {
  static const bool off = (std::getenv("DPRB_NO_CLS_PRUNE") != nullptr);
  return !off;
}

#define TRY(expr) do { if (int _rc = (expr)) return _rc; } while (0)

// The residual stream travels in fp16: the pre-LayerNorm sums z1 / z2 (saved, read again by the LayerNorm backward) and a
// transient fp16 copy of every LayerNorm output that the next residual add reads (rA: layer input / output, rB: x1).
// The bf16 copies of the LayerNorm outputs (x0, x1, out) remain the GEMM operands and what wgrad reads; everything else
// 16-bit (qkv, ctx, GELU tensors, all gradients) is bf16.  See common.cuh for the measured effect.
constexpr int RS_F16 = 1;
constexpr int X16 = DPRB_GEMM_AUX_F16, O16 = DPRB_GEMM_OUT_F16;

// The layer stack of both forward entry points.  pooled != nullptr: CLS output (fp32 [nseq, H]), last layer CLS-pruned
// unless DPRB_NO_CLS_PRUNE is set.  tokens != nullptr: every token of the last layer, bf16 [nseq*S, H], written by the
// final LayerNorm straight into the caller's buffer; the last layer is never pruned.
int forward_layers(const dprb_encoder_weights* w, const dprb_encoder_batch* b, float* pooled, bf16* tokens,
                   cudaStream_t stream) {
  Workspace ws;
  TRY(plan(w, b->nseq, b->S, b->save_for_backward, b->workspace, &ws));
  // position ids index a table of max_pos rows (RoBERTa's pad-derived ids need max_pos >= S + pad + 1: checked by the caller)
  DPRB_REQUIRE(b->S <= w->max_pos, "encoder_fwd: sequence length %d exceeds the position table (max_pos %d)", b->S, w->max_pos);
  DPRB_REQUIRE(b->workspace != nullptr && b->workspace_bytes >= ws.bytes, "encoder_fwd: workspace too small (%lld < %lld)",
               (long long)b->workspace_bytes, ws.bytes);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(b->workspace) & 255) == 0, "encoder_fwd: workspace must be 256-byte aligned");
  const int T = b->nseq * b->S, H = w->hidden, I = w->inter, L = w->layers;
  if (T == 0) return 0;
  const float* ms = w->master;
  TRY(dprb_embed_ln_fwd(b->ids, b->type_ids, b->pos_ids, ms + w->off_word, ms + w->off_pos, ms + w->off_type,
                        ms + w->off_emb_ln_g, ms + w->off_emb_ln_b, ws.x0, ws.emb_stats, T, H, w->vocab, w->max_pos,
                        w->type_vocab, w->ln_eps, b->dropout_p, b->dropout_seed, ws.rA, stream));
  const bf16* x = ws.x0;
  const float dp = b->dropout_p;
  DPRB_REQUIRE(dp >= 0.f && dp < 1.f, "encoder_fwd: dropout_p %f out of range", dp);
  const int GELU_EPI = DPRB_EPI_BIAS_GELU | (ws.lean ? DPRB_GEMM_SAVE_PRE : 0);
  for (int l = 0; l < L; ++l) {
    const LayerW lw = layer_w(w, l);
    LayerActs& a = ws.slot[b->save_for_backward ? l : (l & 1)];
    if (l == L - 1 && tokens == nullptr && prune_last_layer()) {
      // Last layer: only token 0 of each sequence is consumed downstream (hf_model.py:39).  K and V are needed for all
      // tokens, everything after the attention scores only for the nseq CLS rows (stored in the first nseq rows of
      // this layer's activation buffers; the saved probabilities reuse the lse buffer).
      const int R = b->nseq;
      TRY(dprb_gemm_bf16(x, lw.wqkv, a.qkv, T, 3 * H, H, H, H, 3 * H, 0, 0, DPRB_EPI_BIAS , lw.bqkv, nullptr, 0, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
      TRY(dprb_attn_cls_fwd(a.qkv, b->attn_mask, a.ctx, a.lse, b->nseq, b->S, w->heads, dp, site_seed(b, l, DROP_SITE_ATTN), stream));
      TRY(dprb_gemm_bf16(a.ctx, lw.wo, a.z1, R, H, H, H, H, H, 0, 0, DPRB_EPI_BIAS_RESIDUAL | X16 | O16, lw.bo, ws.rA, (long long)b->S * H, nullptr, 1.f, 1, nullptr, dp, site_seed_cls(b, l, DROP_SITE_ATTN_OUT), stream));
      TRY(dprb_ln_fwd(a.z1, lw.ln1g, lw.ln1b, a.x1, a.stats1, nullptr, 1, R, H, w->ln_eps, RS_F16, ws.rB, stream));
      TRY(dprb_gemm_bf16(a.x1, lw.w1, a.hact, R, I, H, H, H, I, 0, 0, GELU_EPI, lw.b1, nullptr, 0, a.hpre, 1.f, 1, nullptr, 0.f, 0, stream));
      TRY(dprb_gemm_bf16(a.hact, lw.w2, a.z2, R, H, I, I, I, H, 0, 0, DPRB_EPI_BIAS_RESIDUAL | X16 | O16, lw.b2, ws.rB, H, nullptr, 1.f, 1, nullptr, dp, site_seed_cls(b, l, DROP_SITE_FFN_OUT), stream));
      TRY(dprb_ln_fwd(a.z2, lw.ln2g, lw.ln2b, a.out, a.stats2, pooled, 1, R, H, w->ln_eps, RS_F16, nullptr, stream));
      x = a.out;
      continue;
    }
    TRY(dprb_gemm_bf16(x, lw.wqkv, a.qkv, T, 3 * H, H, H, H, 3 * H, 0, 0, DPRB_EPI_BIAS , lw.bqkv, nullptr, 0, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
    TRY(dprb_attn_fwd(a.qkv, b->attn_mask, a.ctx, a.lse, b->nseq, b->S, w->heads, dp, site_seed(b, l, DROP_SITE_ATTN), stream));
    TRY(dprb_gemm_bf16(a.ctx, lw.wo, a.z1, T, H, H, H, H, H, 0, 0, DPRB_EPI_BIAS_RESIDUAL | X16 | O16, lw.bo, ws.rA, H, nullptr, 1.f, 1, nullptr, dp, site_seed(b, l, DROP_SITE_ATTN_OUT), stream));
    TRY(dprb_ln_fwd(a.z1, lw.ln1g, lw.ln1b, a.x1, a.stats1, nullptr, 1, T, H, w->ln_eps, RS_F16, ws.rB, stream));
    TRY(dprb_gemm_bf16(a.x1, lw.w1, a.hact, T, I, H, H, H, I, 0, 0, GELU_EPI, lw.b1, nullptr, 0, a.hpre, 1.f, 1, nullptr, 0.f, 0, stream));
    TRY(dprb_gemm_bf16(a.hact, lw.w2, a.z2, T, H, I, I, I, H, 0, 0, DPRB_EPI_BIAS_RESIDUAL | X16 | O16, lw.b2, ws.rB, H, nullptr, 1.f, 1, nullptr, dp, site_seed(b, l, DROP_SITE_FFN_OUT), stream));
    const bool last = (l == L - 1);
    bf16* y = (last && tokens != nullptr) ? tokens : a.out;
    TRY(dprb_ln_fwd(a.z2, lw.ln2g, lw.ln2b, y, a.stats2, last ? pooled : nullptr, b->S, T, H, w->ln_eps, RS_F16, last ? nullptr : ws.rA, stream));
    x = y;
  }
  return 0;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int64_t dprb_encoder_workspace_bytes(const dprb_encoder_weights* w, int nseq, int S, int save) {
  Workspace ws;
  if (plan(w, nseq, S, save, nullptr, &ws)) return -1;
  return ws.bytes;
}

extern "C" int dprb_encoder_fwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, float* pooled,
                                dprb_stream_t stream) {
  return forward_layers(w, b, pooled, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int dprb_encoder_fwd_tokens(const dprb_encoder_weights* w, const dprb_encoder_batch* b, void* tokens,
                                       dprb_stream_t stream) {
  DPRB_REQUIRE(b->save_for_backward == 0, "encoder_fwd_tokens: forward only (save_for_backward must be 0)");
  DPRB_REQUIRE(tokens != nullptr || (long long)b->nseq * b->S == 0, "encoder_fwd_tokens: tokens output is NULL");
  return forward_layers(w, b, nullptr, reinterpret_cast<bf16*>(tokens), static_cast<cudaStream_t>(stream));
}

extern "C" int dprb_encoder_bwd(const dprb_encoder_weights* w, const dprb_encoder_batch* b, const float* dpooled,
                                int layer_lo, int layer_hi, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Workspace ws;
  DPRB_REQUIRE(b->save_for_backward, "encoder_bwd: forward was run without save_for_backward");
  DPRB_REQUIRE(w->grads != nullptr, "encoder_bwd: grads arena is NULL");
  TRY(plan(w, b->nseq, b->S, b->save_for_backward, b->workspace, &ws));
  DPRB_REQUIRE(b->workspace != nullptr && b->workspace_bytes >= ws.bytes, "encoder_bwd: workspace too small");
  const int DGELU_EPI = ws.lean ? DPRB_EPI_DGELU_PRE : DPRB_EPI_DGELU;
  const int T = b->nseq * b->S, H = w->hidden, I = w->inter, L = w->layers;
  DPRB_REQUIRE(0 <= layer_lo && layer_lo < layer_hi && layer_hi <= L, "encoder_bwd: bad layer range [%d,%d)", layer_lo, layer_hi);
  if (T == 0) return 0;
  for (int l = layer_hi - 1; l >= layer_lo; --l) {
    const LayerW lw = layer_w(w, l);
    LayerActs& a = ws.slot[l];
    const bf16* x = (l == 0) ? ws.x0 : ws.slot[l - 1].out;
    const bool last = (l == L - 1);
    const float dp = b->dropout_p;
    // with hidden dropout the Linear-side gradient is dz * mask/(1-p) (gB2); the residual branch keeps dz (gB)
    const bf16* gLin = dp > 0.f ? ws.gB2 : ws.gB;
    if (last && prune_last_layer()) {
      const int R = b->nseq;
      TRY(dprb_ln_bwd(nullptr, dpooled, 1, a.z2, a.stats2, lw.ln2g, ws.gB, lw.g_ln2g, lw.g_ln2b, lw.g_b2, R, H, ws.gB2, dp,
                      site_seed_cls(b, l, DROP_SITE_FFN_OUT), RS_F16, stream));
      TRY(dprb_gemm_bf16(gLin, a.hact, lw.g_w2, H, I, R, H, I, I, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
      TRY(dprb_gemm_bf16(gLin, lw.w2, ws.gH, R, I, H, H, I, I, 0, 1, DGELU_EPI, nullptr, a.hpre, I, nullptr, 1.f, 1, lw.g_b1, 0.f, 0, stream));
      TRY(dprb_gemm_bf16(ws.gH, a.x1, lw.g_w1, I, H, R, I, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
      TRY(dprb_gemm_bf16(ws.gH, lw.w1, ws.gA, R, H, I, I, H, H, 0, 1, DPRB_EPI_BIAS_RESIDUAL, nullptr, ws.gB, H, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
      TRY(dprb_ln_bwd(ws.gA, nullptr, 1, a.z1, a.stats1, lw.ln1g, ws.gB, lw.g_ln1g, lw.g_ln1b, lw.g_bo, R, H, ws.gB2, dp,
                      site_seed_cls(b, l, DROP_SITE_ATTN_OUT), RS_F16, stream));
      TRY(dprb_gemm_bf16(gLin, a.ctx, lw.g_wo, H, H, R, H, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
      TRY(dprb_gemm_bf16(gLin, lw.wo, ws.gA, R, H, H, H, H, H, 0, 1, DPRB_EPI_BIAS, nullptr, nullptr, 0, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
      TRY(dprb_attn_cls_bwd(a.qkv, a.lse, ws.gA, ws.gQKV, b->nseq, b->S, w->heads, dp, site_seed(b, l, DROP_SITE_ATTN), stream));
      TRY(dprb_colsum_bf16(ws.gQKV, 3 * H, lw.g_bqkv, T, 3 * H, stream));
      TRY(dprb_gemm_bf16(ws.gQKV, x, lw.g_wqkv, 3 * H, H, T, 3 * H, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
      // dx = dqkv Wqkv, plus the residual gradient dz1 on the CLS rows only
      TRY(dprb_gemm_bf16(ws.gQKV, lw.wqkv, ws.gA, T, H, 3 * H, 3 * H, H, H, 0, 1, DPRB_EPI_BIAS, nullptr, nullptr, 0, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
      TRY(add_rows_bf16(ws.gA, ws.gB, R, H, b->S, stream));
      continue;
    }
    // LN2 backward (+ db2)
    TRY(dprb_ln_bwd(last ? nullptr : ws.gA, last ? dpooled : nullptr, b->S, a.z2, a.stats2, lw.ln2g, ws.gB, lw.g_ln2g,
                    lw.g_ln2b, lw.g_b2, T, H, ws.gB2, dp, site_seed(b, l, DROP_SITE_FFN_OUT), RS_F16, stream));
    // lean activations: the GELU output was not kept - rebuild it from the saved pre-activation
    if (ws.lean) TRY(dprb_gelu_from_pre(a.hpre, a.hact, (long long)T * I, stream));
    // dW2 += dz2^T hact
    TRY(dprb_gemm_bf16(gLin, a.hact, lw.g_w2, H, I, T, H, I, I, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
    // dhpre = (dz2 W2) * gelu'(hpre)
    TRY(dprb_gemm_bf16(gLin, lw.w2, ws.gH, T, I, H, H, I, I, 0, 1, DGELU_EPI, nullptr, a.hpre, I, nullptr, 1.f, 1, lw.g_b1, 0.f, 0, stream));
    // (db1 = column sums of dhpre is fused into that epilogue: +58 us vs 129 us for a separate streaming pass)
    // dW1 += dhpre^T x1
    TRY(dprb_gemm_bf16(ws.gH, a.x1, lw.g_w1, I, H, T, I, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
    // dx1 = dhpre W1 + dz2
    TRY(dprb_gemm_bf16(ws.gH, lw.w1, ws.gA, T, H, I, I, H, H, 0, 1, DPRB_EPI_BIAS_RESIDUAL, nullptr, ws.gB, H, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
    // LN1 backward (+ dbo)
    TRY(dprb_ln_bwd(ws.gA, nullptr, 1, a.z1, a.stats1, lw.ln1g, ws.gB, lw.g_ln1g, lw.g_ln1b, lw.g_bo, T, H, ws.gB2, dp,
                    site_seed(b, l, DROP_SITE_ATTN_OUT), RS_F16, stream));
    // lean activations: the attention output was not kept - one more attention forward (same dropout stream)
    if (ws.lean) TRY(dprb_attn_fwd(a.qkv, b->attn_mask, a.ctx, a.lse, b->nseq, b->S, w->heads, dp, site_seed(b, l, DROP_SITE_ATTN), stream));
    // dWo += dz1^T ctx
    TRY(dprb_gemm_bf16(gLin, a.ctx, lw.g_wo, H, H, T, H, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
    // dctx = dz1 Wo
    TRY(dprb_gemm_bf16(gLin, lw.wo, ws.gA, T, H, H, H, H, H, 0, 1, DPRB_EPI_BIAS, nullptr, nullptr, 0, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
    // (+ dbqkv: column sums of dqkv fused into the attention-backward epilogue)
    TRY(dprb_attn_bwd(a.qkv, b->attn_mask, a.ctx, a.lse, ws.gA, ws.gQKV, lw.g_bqkv, b->nseq, b->S, w->heads, dp,
                      site_seed(b, l, DROP_SITE_ATTN), stream));
    // dWqkv += dqkv^T x
    TRY(dprb_gemm_bf16(ws.gQKV, x, lw.g_wqkv, 3 * H, H, T, 3 * H, H, H, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0, nullptr, 1.f, 0, nullptr, 0.f, 0, stream));
    // dx = dqkv Wqkv + dz1
    TRY(dprb_gemm_bf16(ws.gQKV, lw.wqkv, ws.gA, T, H, 3 * H, 3 * H, H, H, 0, 1, DPRB_EPI_BIAS_RESIDUAL, nullptr, ws.gB, H, nullptr, 1.f, 1, nullptr, 0.f, 0, stream));
  }
  if (layer_lo == 0) {
    const float* ms = w->master;
    float* gr = w->grads;
    TRY(dprb_embed_ln_bwd(ws.gA, b->ids, b->type_ids, b->pos_ids, ms + w->off_word, ms + w->off_pos, ms + w->off_type,
                          ms + w->off_emb_ln_g, ws.emb_stats, gr + w->off_word, gr + w->off_pos, gr + w->off_type,
                          gr + w->off_emb_ln_g, gr + w->off_emb_ln_b, T, H, b->dropout_p, b->dropout_seed, stream));
  }
  return 0;
}
