// Self-attention core (head_dim 64, S <= 512) forward + backward: shape checks, then the wgmma kernels of
// attention_wgmma.cu for S <= 256 (keys padded to 64, 128 or 256) or the key-blocked kernels of attention_long.cu for
// 256 < S <= 512.
//
// Replaces BertSelfAttention.forward's scaled_dot_product_attention (transformers' modeling_bert.py) and its
// autograd backward.
//
// Layout: qkv bf16 [nseq*S, 3H], row t = (seq, s); Q at column h*64, K at H + h*64, V at 2H + h*64.
#include "attention.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int DH = 64;
constexpr int SHORT_MAX = 256;   // longest sequence of the single-block kernels (attention_wgmma.cu)

int check_shape(int nseq, int S, int heads, const char* who) {
  DPRB_REQUIRE(nseq >= 0 && heads > 0, "%s: bad nseq=%d heads=%d", who, nseq, heads);
  DPRB_REQUIRE(S >= 1 && S <= 512, "%s: sequence length %d unsupported (1..512)", who, S);
  return 0;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_attn_fwd(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S,
                             int heads, float dropout_p, uint64_t site_seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_shape(nseq, S, heads, "attn_fwd")) return rc;
  if (nseq == 0) return 0;
  if (S > SHORT_MAX) return attn_fwd_long(qkv, attn_mask, ctx, lse, nseq, S, heads, dropout_p, site_seed, stream);
  return attn_fwd_wg(qkv, attn_mask, ctx, lse, nseq, S, heads, dropout_p, site_seed, stream);
}

extern "C" int dprb_attn_bwd(const void* qkv, const int32_t* attn_mask, const void* ctx, const float* lse,
                             const void* dctx, void* dqkv, float* dbias, int nseq, int S, int heads, float dropout_p,
                             uint64_t site_seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_shape(nseq, S, heads, "attn_bwd")) return rc;
  if (nseq == 0) return 0;
  // D = rowsum(P * dP) is rebuilt in fp32 from Q, K, V, dO and lse; ctx is not read.  The S <= 128 kernel sums the
  // QKV bias gradient itself.
  if (S <= SHORT_MAX)
    return attn_bwd_wg(qkv, attn_mask, lse, dctx, dqkv, dbias, nseq, S, heads, dropout_p, site_seed, stream);
  // D = rowsum(dO * ctx) in fp32
  if (int rc = attn_bwd_long(qkv, attn_mask, ctx, lse, dctx, dqkv, nseq, S, heads, dropout_p, site_seed, stream)) return rc;
  // the QKV bias gradient: column sums of the bf16 dQ / dK / dV
  if (dbias != nullptr) return dprb_colsum_bf16(dqkv, 3LL * heads * DH, dbias, nseq * S, 3 * heads * DH, stream);
  return 0;
}
