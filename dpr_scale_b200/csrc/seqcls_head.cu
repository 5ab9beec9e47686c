// Sequence-classification head of a cross-encoder, after its dense layer:
//   logits[n, l] = tanh(pre[n, :]) . W[l, :] + b[l],   score[n] = max_l logits[n, l].
// `pre` is the fp32 output of the head's dense layer (BERT: pooler.dense, RoBERTa: classifier.dense), computed by the
// library's GEMM with the F32_STORE epilogue on the CLS rows.  One warp per row: the row's tanh stays in registers
// (H <= 1024: at most 8 float4 per lane) and is dotted with every label's weight row (fp32, L <= 16).
//
// Training (dprb_seqcls_group_ce): one relevance label (L = 1) and the softmax cross-entropy of each group of G
// consecutive rows against its label row, with the head's dropout on tanh(pre) and the whole backward of the head in
// the same pass.  One block per group: a row pass (one warp per row) forms the logits, warp 0 takes the group's
// softmax, then a column pass (four columns per thread, rows in order) writes dpre and sums the group's dW.  A
// one-launch final pass adds the per-group partials of dW, db and the loss in a fixed order: no atomics, so every
// output is bitwise repeatable.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {

namespace {

constexpr int kRowsPerBlock = 8;
constexpr int kMaxVec = 1024 / (32 * 4);   // float4 per lane at H = 1024

__global__ void __launch_bounds__(32 * kRowsPerBlock)
seqcls_head_kernel(const float* __restrict__ pre, const float* __restrict__ W, const float* __restrict__ b,
                   float* __restrict__ logits, float* __restrict__ score, int N, int H, int L) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * kRowsPerBlock + (threadIdx.x >> 5);
  if (n >= N) return;
  const int nvec = H >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(pre + (size_t)n * H);
  float4 t[kMaxVec];
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j) {
    const int c = lane + 32 * j;
    if (c < nvec) {
      const float4 v = x4[c];
      t[j] = make_float4(tanhf(v.x), tanhf(v.y), tanhf(v.z), tanhf(v.w));
    } else {
      t[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float best = -INFINITY;
  for (int l = 0; l < L; ++l) {
    const float4* w4 = reinterpret_cast<const float4*>(W + (size_t)l * H);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVec; ++j) {
      const int c = lane + 32 * j;
      if (c < nvec) {
        const float4 w = __ldg(w4 + c);
        acc = fmaf(t[j].x, w.x, acc);
        acc = fmaf(t[j].y, w.y, acc);
        acc = fmaf(t[j].z, w.z, acc);
        acc = fmaf(t[j].w, w.w, acc);
      }
    }
    acc = warp_sum(acc) + (b ? __ldg(b + l) : 0.f);
    if (lane == 0) logits[(size_t)n * L + l] = acc;
    best = fmaxf(best, acc);
  }
  if (score && lane == 0) score[n] = best;
}

constexpr int kGroupThreads = 256;
constexpr int kGroupWarps = kGroupThreads / 32;
constexpr int kMaxChunk8 = 1024 / (32 * 8);   // 8-column chunks per lane at H = 1024

__global__ void __launch_bounds__(kGroupThreads)
seqcls_group_ce_kernel(const float* __restrict__ pre, const float* __restrict__ W, const float* __restrict__ b,
                       const long long* __restrict__ labels, int B, int G, int H, Drop drop, float* __restrict__ logits,
                       bf16* __restrict__ dpre, float* __restrict__ dw_part, float* __restrict__ db_part,
                       float* __restrict__ loss_part) {
  __shared__ float logit_s[DPRB_SEQCLS_GROUP_MAX];
  __shared__ float dlog_s[DPRB_SEQCLS_GROUP_MAX];
  const int grp = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n8 = H >> 3;
  const float bias = b ? __ldg(b) : 0.f;
  // row pass: logit = W . (tanh(pre) * mask) + b
  for (int i = warp; i < G; i += kGroupWarps) {
    const int n = grp * G + i;
    const float* x = pre + (size_t)n * H;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxChunk8; ++j) {
      const int k = lane + 32 * j;
      if (k < n8) {
        const float4 a0 = *reinterpret_cast<const float4*>(x + 8 * k);
        const float4 a1 = *reinterpret_cast<const float4*>(x + 8 * k + 4);
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(W + 8 * k));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(W + 8 * k + 4));
        float2 m[4] = {make_float2(1.f, 1.f), make_float2(1.f, 1.f), make_float2(1.f, 1.f), make_float2(1.f, 1.f)};
        if (drop.on()) drop.mul8((uint32_t)n, (uint32_t)(8 * k), m);
        acc = fmaf(tanhf(a0.x) * m[0].x, w0.x, acc);
        acc = fmaf(tanhf(a0.y) * m[0].y, w0.y, acc);
        acc = fmaf(tanhf(a0.z) * m[1].x, w0.z, acc);
        acc = fmaf(tanhf(a0.w) * m[1].y, w0.w, acc);
        acc = fmaf(tanhf(a1.x) * m[2].x, w1.x, acc);
        acc = fmaf(tanhf(a1.y) * m[2].y, w1.y, acc);
        acc = fmaf(tanhf(a1.z) * m[3].x, w1.z, acc);
        acc = fmaf(tanhf(a1.w) * m[3].y, w1.w, acc);
      }
    }
    acc = warp_sum(acc) + bias;
    if (lane == 0) {
      logit_s[i] = acc;
      logits[n] = acc;
    }
  }
  __syncthreads();
  // the group's softmax cross-entropy; dlogit carries the 1/B of the mean over groups
  if (warp == 0) {
    const long long label = __ldg(labels + grp);
    const bool ok = label >= 0 && label < G;
    const float v0 = lane < G ? logit_s[lane] : -INFINITY;
    const float v1 = lane + 32 < G ? logit_s[lane + 32] : -INFINITY;
    float mx = fmaxf(v0, v1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e0 = lane < G ? expf(v0 - mx) : 0.f;
    const float e1 = lane + 32 < G ? expf(v1 - mx) : 0.f;
    const float sum = warp_sum(e0 + e1);
    const float invB = 1.f / (float)B;
    const float d0 = (e0 / sum - (ok && lane == label ? 1.f : 0.f)) * invB;
    const float d1 = (e1 / sum - (ok && lane + 32 == label ? 1.f : 0.f)) * invB;
    if (lane < G) dlog_s[lane] = d0;
    if (lane + 32 < G) dlog_s[lane + 32] = d1;
    const float dsum = warp_sum((lane < G ? d0 : 0.f) + (lane + 32 < G ? d1 : 0.f));
    if (lane == 0) {
      db_part[grp] = dsum;
      loss_part[grp] = ok ? mx + logf(sum) - logit_s[label] : __int_as_float(0x7fc00000);
    }
  }
  __syncthreads();
  // column pass: dpre = dlogit * W * mask * (1 - t^2) and this group's dW = sum_i dlogit_i * t_i * mask_i, rows in order
  const int c = 4 * threadIdx.x;
  if (c < H) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(W + c));
    float4 dw = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < G; ++i) {
      const int n = grp * G + i;
      const float4 a = *reinterpret_cast<const float4*>(pre + (size_t)n * H + c);
      float m0 = 1.f, m1 = 1.f, m2 = 1.f, m3 = 1.f;
      if (drop.on()) {
        drop.mul2((uint32_t)n, (uint32_t)c, m0, m1);
        drop.mul2((uint32_t)n, (uint32_t)c + 2u, m2, m3);
      }
      const float t0 = tanhf(a.x), t1 = tanhf(a.y), t2 = tanhf(a.z), t3 = tanhf(a.w);
      const float dl = dlog_s[i];
      dw.x = fmaf(dl, t0 * m0, dw.x);
      dw.y = fmaf(dl, t1 * m1, dw.y);
      dw.z = fmaf(dl, t2 * m2, dw.z);
      dw.w = fmaf(dl, t3 * m3, dw.w);
      uint2 out;
      out.x = pack_bf16x2(dl * w.x * m0 * (1.f - t0 * t0), dl * w.y * m1 * (1.f - t1 * t1));
      out.y = pack_bf16x2(dl * w.z * m2 * (1.f - t2 * t2), dl * w.w * m3 * (1.f - t3 * t3));
      *reinterpret_cast<uint2*>(dpre + (size_t)n * H + c) = out;
    }
    *reinterpret_cast<float4*>(dw_part + (size_t)grp * H + c) = dw;
  }
}

// dweight[c] = sum over groups of dw_part[., c] (one thread per column, groups in order); the last block reduces the
// loss and db partials in double through a fixed tree.
__global__ void __launch_bounds__(kGroupThreads)
seqcls_group_ce_final_kernel(const float* __restrict__ dw_part, const float* __restrict__ db_part,
                             const float* __restrict__ loss_part, int B, int H, float* __restrict__ dweight,
                             float* __restrict__ dbias, float* __restrict__ loss) {
  __shared__ double red[2][kGroupWarps];
  if (blockIdx.x + 1 < gridDim.x) {
    const int c = blockIdx.x * kGroupThreads + threadIdx.x;
    if (c < H) {
      float s = 0.f;
      for (int g = 0; g < B; ++g) s += dw_part[(size_t)g * H + c];
      dweight[c] = s;
    }
    return;
  }
  double l = 0.0, d = 0.0;
  for (int g = threadIdx.x; g < B; g += kGroupThreads) {
    l += (double)loss_part[g];
    d += (double)db_part[g];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_xor_sync(0xffffffffu, l, o);
    d += __shfl_xor_sync(0xffffffffu, d, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    red[0][warp] = l;
    red[1][warp] = d;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double lt = 0.0, dt = 0.0;
    for (int w = 0; w < kGroupWarps; ++w) {
      lt += red[0][w];
      dt += red[1][w];
    }
    loss[0] = (float)(lt / (double)B);
    dbias[0] = (float)dt;
  }
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_seqcls_head_fwd(const float* pre, const float* weight, const float* bias, float* logits,
                                    float* score, int N, int H, int L, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(N >= 0, "seqcls_head: N = %d must be >= 0", N);
  DPRB_REQUIRE(H > 0 && H % 8 == 0 && H <= 1024, "seqcls_head: hidden size %d must be a multiple of 8 and <= 1024", H);
  DPRB_REQUIRE(L >= 1 && L <= DPRB_SEQCLS_MAX_LABELS, "seqcls_head: %d labels (supported: 1 .. %d)", L,
               DPRB_SEQCLS_MAX_LABELS);
  DPRB_REQUIRE(pre && weight && logits, "seqcls_head: pre, weight and logits must be non-NULL");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(weight)) & 15) == 0,
               "seqcls_head: pre and weight must be 16-byte aligned");
  if (N == 0) return 0;
  const int blocks = (N + kRowsPerBlock - 1) / kRowsPerBlock;
  seqcls_head_kernel<<<blocks, 32 * kRowsPerBlock, 0, stream>>>(pre, weight, bias, logits, score, N, H, L);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t dprb_seqcls_group_ce_workspace_bytes(int B, int H) {
  return B > 0 && H > 0 ? ((long long)B * H + 2LL * B) * (long long)sizeof(float) : 0;
}

extern "C" int dprb_seqcls_group_ce(const float* pre, const float* weight, const float* bias, const int64_t* labels_,
                                    int B, int G, int H, float dropout_p, uint64_t dropout_seed, float* loss,
                                    float* logits, void* dpre, float* dweight, float* dbias, void* workspace,
                                    int64_t workspace_bytes, dprb_stream_t stream_) {
  const long long* labels = reinterpret_cast<const long long*>(labels_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(B >= 1, "seqcls_group_ce: %d groups (at least 1)", B);
  DPRB_REQUIRE(G >= 2 && G <= DPRB_SEQCLS_GROUP_MAX, "seqcls_group_ce: group size %d (supported: 2 .. %d)", G,
               DPRB_SEQCLS_GROUP_MAX);
  DPRB_REQUIRE((long long)B * G <= 0x7fffffffLL, "seqcls_group_ce: %d x %d rows exceed 2^31 - 1", B, G);
  DPRB_REQUIRE(H > 0 && H % 8 == 0 && H <= 1024, "seqcls_group_ce: hidden size %d must be a multiple of 8 and <= 1024",
               H);
  DPRB_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, "seqcls_group_ce: dropout p = %g must lie in [0, 1)",
               (double)dropout_p);
  DPRB_REQUIRE(pre && weight && labels && loss && logits && dpre && dweight && dbias,
               "seqcls_group_ce: only bias may be NULL");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(weight) |
                 reinterpret_cast<uintptr_t>(dpre) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
               "seqcls_group_ce: pre, weight, dpre and workspace must be 16-byte aligned");
  const long long need = dprb_seqcls_group_ce_workspace_bytes(B, H);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= need, "seqcls_group_ce: workspace of %lld bytes, %lld needed",
               (long long)workspace_bytes, need);
  float* dw_part = reinterpret_cast<float*>(workspace);
  float* db_part = dw_part + (size_t)B * H;
  float* loss_part = db_part + B;
  const Drop drop = make_drop(dropout_p, dropout_seed, 0, DROP_SITE_HEAD);
  seqcls_group_ce_kernel<<<B, kGroupThreads, 0, stream>>>(pre, weight, bias, labels, B, G, H, drop, logits,
                                                          reinterpret_cast<bf16*>(dpre), dw_part, db_part, loss_part);
  DPRB_LAUNCH_CHECK();
  const int col_blocks = (H + kGroupThreads - 1) / kGroupThreads;
  seqcls_group_ce_final_kernel<<<col_blocks + 1, kGroupThreads, 0, stream>>>(dw_part, db_part, loss_part, B, H,
                                                                             dweight, dbias, loss);
  DPRB_LAUNCH_CHECK();
  return 0;
}
