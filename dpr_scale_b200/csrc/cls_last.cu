// Last-layer pruning: the encoder's only output is the hidden state of token 0 (CLS) of the LAST layer
// (/root/reference/dpr_scale/models/hf_model.py:39), so in that layer only the CLS query row has to attend and only
// the CLS rows (1 of every S) have to go through attention-output / LayerNorm / FFN — the keys and values of all
// tokens are still needed.  HuggingFace computes (and back-propagates) all S rows and throws S-1 of them away.
//
// Kernels here: single-query attention forward / backward (one warp per (sequence, head), exact fp32 softmax over
// <= 512 keys: MAXK keys per lane, 8 for S <= 256 and 16 for 256 < S <= 512) and the scatter of the CLS-row residual
// gradient.  The GEMMs / LayerNorms of the pruned layer are the
// regular kernels run on nseq rows.
//
// Same arithmetic as BertSelfAttention (site-packages/transformers/models/bert/modeling_bert.py:168-207) restricted
// to query position 0.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

__device__ __forceinline__ void load_row64(const bf16* p, float (&v)[64]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 q = *reinterpret_cast<const uint4*>(p + i * 8);
    const float2 a = unpack_bf16x2(q.x), b = unpack_bf16x2(q.y), c = unpack_bf16x2(q.z), d = unpack_bf16x2(q.w);
    v[i * 8 + 0] = a.x; v[i * 8 + 1] = a.y; v[i * 8 + 2] = b.x; v[i * 8 + 3] = b.y;
    v[i * 8 + 4] = c.x; v[i * 8 + 5] = c.y; v[i * 8 + 6] = d.x; v[i * 8 + 7] = d.y;
  }
}
__device__ __forceinline__ float dot_row64(const bf16* p, const float (&q)[64]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 u = *reinterpret_cast<const uint4*>(p + i * 8);
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    s = fmaf(a.x, q[i * 8 + 0], s); s = fmaf(a.y, q[i * 8 + 1], s); s = fmaf(b.x, q[i * 8 + 2], s); s = fmaf(b.y, q[i * 8 + 3], s);
    s = fmaf(c.x, q[i * 8 + 4], s); s = fmaf(c.y, q[i * 8 + 5], s); s = fmaf(d.x, q[i * 8 + 6], s); s = fmaf(d.y, q[i * 8 + 7], s);
  }
  return s;
}
__device__ __forceinline__ void store_row64_scaled(bf16* p, const float (&v)[64], float s) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint4 q;
    q.x = pack_bf16x2(v[i * 8 + 0] * s, v[i * 8 + 1] * s); q.y = pack_bf16x2(v[i * 8 + 2] * s, v[i * 8 + 3] * s);
    q.z = pack_bf16x2(v[i * 8 + 4] * s, v[i * 8 + 5] * s); q.w = pack_bf16x2(v[i * 8 + 6] * s, v[i * 8 + 7] * s);
    *reinterpret_cast<uint4*>(p + i * 8) = q;
  }
}

// ctx_cls[seq, h*64 + d] = sum_j softmax_j(q_0 . k_j / 8 + mask_j) v_j[d];  probs[(seq*heads+h)*S + j] saved (fp32).
// MAXK: keys per lane (S <= 32 * MAXK).  MAXK = 16 asks for one CTA per SM so that its 16-key rows fit in registers
// without spilling; MAXK = 8 keeps the compiler's default (a minimum of 0 blocks is no constraint).
template <int MAXK>
__global__ void __launch_bounds__(256, MAXK == 8 ? 0 : 1)
attn_cls_fwd_kernel(const bf16* __restrict__ qkv, const int32_t* __restrict__ attn_mask, bf16* __restrict__ ctx_cls,
                    float* __restrict__ probs, int nseq, int S, int heads, Drop drop) {
  const int lane = threadIdx.x & 31;
  const int prob = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (prob >= nseq * heads) return;
  const int seq = prob / heads, h = prob - seq * heads, H = heads * 64;
  const bf16* base = qkv + (long long)seq * S * (3 * H) + h * 64;
  float q[64];
  load_row64(base, q);
  float s[MAXK];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    const int j = lane + 32 * i;
    s[i] = -INFINITY;
    if (j < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + j] != 0))
      s[i] = dot_row64(base + (long long)j * (3 * H) + H, q) * 0.125f;
    m = fmaxf(m, s[i]);
  }
  m = warp_max(m);
  const float e = (m == -INFINITY) ? 0.f : m;
  float l = 0.f;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) { s[i] = __expf(s[i] - e); l += s[i]; }
  l = warp_sum(l);
  const float inv = l > 0.f ? 1.f / l : 0.f;
  float pd[MAXK];
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    const int j = lane + 32 * i;
    s[i] *= inv;
    if (j < S && probs != nullptr) probs[(long long)prob * S + j] = s[i];
    pd[i] = s[i];
    if (drop.on() && j < S) pd[i] *= drop_one(drop, (uint32_t)(prob * S), (uint32_t)j);  // query row 0 of this problem
  }
  // o[d] for d = 2*lane, 2*lane+1: coalesced 128-byte reads of V rows, p_j broadcast from its owner lane
  float o0 = 0.f, o1 = 0.f;
  const bf16* vbase = base + 2 * H + 2 * lane;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    if (i * 32 < S) {
      for (int jj = 0; jj < 32; ++jj) {
        const int j = i * 32 + jj;
        const float pj = __shfl_sync(0xffffffffu, pd[i], jj);
        if (j < S) {
          const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vbase + (long long)j * (3 * H)));
          o0 = fmaf(pj, v.x, o0); o1 = fmaf(pj, v.y, o1);
        }
      }
    }
  }
  *reinterpret_cast<uint32_t*>(ctx_cls + (long long)seq * H + h * 64 + 2 * lane) = pack_bf16x2(o0, o1);
}

// Backward of the single-query attention: writes the FULL dqkv [T, 3H] (dQ: row 0 only, zeros elsewhere).
template <int MAXK>
__global__ void __launch_bounds__(256, MAXK == 8 ? 0 : 1)
attn_cls_bwd_kernel(const bf16* __restrict__ qkv, const float* __restrict__ probs, const bf16* __restrict__ dctx_cls,
                    bf16* __restrict__ dqkv, int nseq, int S, int heads, Drop drop) {
  const int lane = threadIdx.x & 31;
  const int prob = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (prob >= nseq * heads) return;
  const int seq = prob / heads, h = prob - seq * heads, H = heads * 64;
  const bf16* base = qkv + (long long)seq * S * (3 * H) + h * 64;
  bf16* dbase = dqkv + (long long)seq * S * (3 * H) + h * 64;
  float q[64], dO[64];
  load_row64(base, q);
  load_row64(dctx_cls + (long long)seq * H + h * 64, dO);
  float p[MAXK], pd[MAXK], dpm[MAXK];
  float D = 0.f;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    const int j = lane + 32 * i;
    p[i] = 0.f; pd[i] = 0.f; dpm[i] = 0.f;
    if (j < S) {
      p[i] = probs[(long long)prob * S + j];
      const float mj = drop.on() ? drop_one(drop, (uint32_t)(prob * S), (uint32_t)j) : 1.f;
      pd[i] = p[i] * mj;
      dpm[i] = dot_row64(base + (long long)j * (3 * H) + 2 * H, dO) * mj;  // dP_j = dO . v_j (masked + rescaled)
      D = fmaf(p[i], dpm[i], D);
    }
  }
  D = warp_sum(D);
  float ds[MAXK];
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    const int j = lane + 32 * i;
    ds[i] = p[i] * (dpm[i] - D) * 0.125f;
    if (j < S) {
      store_row64_scaled(dbase + (long long)j * (3 * H) + 2 * H, dO, pd[i]);  // dV_j = Pd_j dO
      store_row64_scaled(dbase + (long long)j * (3 * H) + H, q, ds[i]);       // dK_j = dS_j q_0
      if (j > 0) {                                                           // dQ rows other than the CLS query
#pragma unroll
        for (int c = 0; c < 8; ++c) *reinterpret_cast<uint4*>(dbase + (long long)j * (3 * H) + c * 8) = make_uint4(0, 0, 0, 0);
      }
    }
  }
  // dq_0[d] = sum_j dS_j k_j[d] for d = 2*lane, 2*lane+1
  float g0 = 0.f, g1 = 0.f;
  const bf16* kbase = base + H + 2 * lane;
#pragma unroll
  for (int i = 0; i < MAXK; ++i) {
    if (i * 32 < S) {
      for (int jj = 0; jj < 32; ++jj) {
        const int j = i * 32 + jj;
        const float dj = __shfl_sync(0xffffffffu, ds[i], jj);
        if (j < S) {
          const float2 k = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kbase + (long long)j * (3 * H)));
          g0 = fmaf(dj, k.x, g0); g1 = fmaf(dj, k.y, g1);
        }
      }
    }
  }
  *reinterpret_cast<uint32_t*>(dbase + 2 * lane) = pack_bf16x2(g0, g1);
}

// dst[r * stride_rows, :] += src[r, :]   (bf16, H % 8 == 0)
__global__ void add_rows_kernel(bf16* __restrict__ dst, const bf16* __restrict__ src, int nrows, int H, long long stride_rows) {
  const int chunks = H / 8;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < (long long)nrows * chunks;
       idx += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(idx / chunks), c = (int)(idx % chunks);
    uint4* d = reinterpret_cast<uint4*>(dst + (long long)r * stride_rows * H + c * 8);
    const uint4 a = *d, b = *reinterpret_cast<const uint4*>(src + (long long)r * H + c * 8);
    const uint32_t* pa = &a.x; const uint32_t* pb = &b.x;
    uint4 o; uint32_t* po = &o.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 x = unpack_bf16x2(pa[k]), y = unpack_bf16x2(pb[k]);
      po[k] = pack_bf16x2(x.x + y.x, x.y + y.y);
    }
    *d = o;
  }
}

}  // namespace

int add_rows_bf16(void* dst, const void* src, int nrows, int H, long long stride_rows, cudaStream_t stream) {
  DPRB_REQUIRE(H % 8 == 0, "add_rows: H %% 8 != 0");
  if (nrows == 0) return 0;
  const long long n = (long long)nrows * (H / 8);
  add_rows_kernel<<<(int)((n + 255) / 256), 256, 0, stream>>>((bf16*)dst, (const bf16*)src, nrows, H, stride_rows);
  DPRB_LAUNCH_CHECK();
  return 0;
}

}  // namespace dprb

using namespace dprb;

extern "C" int dprb_attn_cls_fwd(const void* qkv, const int32_t* attn_mask, void* ctx_cls, float* probs, int nseq,
                                 int S, int heads, float dropout_p, uint64_t site_seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(S >= 1 && S <= 512, "attn_cls_fwd: sequence length %d unsupported (1..512)", S);
  if (nseq == 0) return 0;
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int nprob = nseq * heads;
  if (S <= 256)
    attn_cls_fwd_kernel<8><<<(nprob + 7) / 8, 256, 0, stream>>>((const bf16*)qkv, attn_mask, (bf16*)ctx_cls, probs, nseq, S, heads, drop);
  else
    attn_cls_fwd_kernel<16><<<(nprob + 7) / 8, 256, 0, stream>>>((const bf16*)qkv, attn_mask, (bf16*)ctx_cls, probs, nseq, S, heads, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_attn_cls_bwd(const void* qkv, const float* probs, const void* dctx_cls, void* dqkv, int nseq,
                                 int S, int heads, float dropout_p, uint64_t site_seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(S >= 1 && S <= 512, "attn_cls_bwd: sequence length %d unsupported (1..512)", S);
  if (nseq == 0) return 0;
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int nprob = nseq * heads;
  if (S <= 256)
    attn_cls_bwd_kernel<8><<<(nprob + 7) / 8, 256, 0, stream>>>((const bf16*)qkv, probs, (const bf16*)dctx_cls, (bf16*)dqkv, nseq, S, heads, drop);
  else
    attn_cls_bwd_kernel<16><<<(nprob + 7) / 8, 256, 0, stream>>>((const bf16*)qkv, probs, (const bf16*)dctx_cls, (bf16*)dqkv, nseq, S, heads, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}
