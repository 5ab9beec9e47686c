// Sequence-classification head of a cross-encoder, after its dense layer:
//   logits[n, l] = tanh(pre[n, :]) . W[l, :] + b[l],   score[n] = max_l logits[n, l].
// `pre` is the fp32 output of the head's dense layer (BERT: pooler.dense, RoBERTa: classifier.dense), computed by the
// library's GEMM with the F32_STORE epilogue on the CLS rows.  One warp per row: the row's tanh stays in registers
// (H <= 1024: at most 8 float4 per lane) and is dotted with every label's weight row (fp32, L <= 16).
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

}  // namespace

int seqcls_head_fwd(const float* pre, const float* weight, const float* bias, float* logits, float* score, int N,
                    int H, int L, cudaStream_t stream) {
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

}  // namespace dprb
