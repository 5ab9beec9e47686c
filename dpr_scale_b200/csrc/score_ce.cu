// Fused in-batch-negative scoring + softmax cross-entropy (forward: one pass over the similarity
// tiles with an online row log-sum-exp and the NLL pick; backward: dq for the rank-local query rows
// and dc for the rank-local context columns from the stored logits).
//
// Replaces /root/reference/dpr_scale/task/dpr_task.py:98-105 (sim_score), :197 (mask.repeat),
// :211 (scores /= temperature), :212 (nn.CrossEntropyLoss) and, for the multi-rank case, the gradient
// flow implied by :163-195 (remote slices are detached; only local rows/columns get gradients).
//
// All arithmetic is fp32 (the reference under AMP does this product in fp16); the work
// is 2*Q*C*d FLOP = 0.2 GFLOP (cfg 2) .. 12.9 GFLOP (cfg 3), latency-bound, so it stays on the FFMA pipe.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int QB = 8;        // query rows per CTA
constexpr int CW = 4;        // columns per warp step
constexpr int FWD_WARPS = 8;

__global__ void __launch_bounds__(FWD_WARPS * 32)
score_ce_fwd_kernel(const float* __restrict__ q, const float* __restrict__ c, const uint8_t* __restrict__ col_mask,
                    const uint8_t* __restrict__ pair_mask, const int64_t* __restrict__ labels, float inv_t, float* __restrict__ lse_out,
                    float* __restrict__ loss_sum, float* __restrict__ logits, int Q, int C, int d, int cols_per_split) {
  extern __shared__ float sm[];
  float* qs = sm;                       // [QB][d]
  float* red = sm + QB * d;             // [FWD_WARPS][QB][3]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * QB;
  for (int i = threadIdx.x; i < QB * d; i += blockDim.x) {
    const int r = i / d, k = i - r * d;
    qs[i] = (row0 + r < Q) ? q[(long long)(row0 + r) * d + k] : 0.f;
  }
  __syncthreads();
  long long lab[QB];
#pragma unroll
  for (int r = 0; r < QB; ++r) lab[r] = (row0 + r < Q) ? labels[row0 + r] : -1;

  float m[QB], l[QB], pick[QB];
#pragma unroll
  for (int r = 0; r < QB; ++r) { m[r] = -INFINITY; l[r] = 0.f; pick[r] = 0.f; }

  // gridDim.y > 1: this CTA only writes the logits of its column range; score_lse_kernel reduces the rows afterwards
  const int c_begin = blockIdx.y * cols_per_split, c_end = min(C, c_begin + cols_per_split);
  for (int cb = c_begin + warp * CW; cb < c_end; cb += FWD_WARPS * CW) {
    float acc[QB][CW];
#pragma unroll
    for (int r = 0; r < QB; ++r)
#pragma unroll
      for (int j = 0; j < CW; ++j) acc[r][j] = 0.f;
    for (int k = lane; k < d; k += 32) {
      float cv[CW];
#pragma unroll
      for (int j = 0; j < CW; ++j) cv[j] = (cb + j < C) ? __ldg(c + (long long)(cb + j) * d + k) : 0.f;
#pragma unroll
      for (int r = 0; r < QB; ++r) {
        const float qv = qs[r * d + k];
#pragma unroll
        for (int j = 0; j < CW; ++j) acc[r][j] = fmaf(qv, cv[j], acc[r][j]);
      }
    }
#pragma unroll
    for (int r = 0; r < QB; ++r)
#pragma unroll
      for (int j = 0; j < CW; ++j) acc[r][j] = warp_sum(acc[r][j]);
#pragma unroll
    for (int j = 0; j < CW; ++j) {
      const int col = cb + j;
      if (col < C) {
        const bool masked = col_mask != nullptr && col_mask[col] != 0;
#pragma unroll
        for (int r = 0; r < QB; ++r) {
          const bool pm = pair_mask != nullptr && row0 + r < Q && pair_mask[(long long)(row0 + r) * C + col] != 0;
          const float s = (masked || pm) ? -INFINITY : acc[r][j] * inv_t;
          if (logits != nullptr && lane == ((r * CW + j) & 31) && row0 + r < Q)
            logits[(long long)(row0 + r) * C + col] = s;
          if (s > m[r]) { l[r] = l[r] * __expf(m[r] - s) + 1.f; m[r] = s; }
          else if (s != -INFINITY) l[r] += __expf(s - m[r]);
          if ((long long)col == lab[r]) pick[r] = s;
        }
      }
    }
  }
  if (gridDim.y > 1) return;
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < QB; ++r) {
      red[(warp * QB + r) * 3 + 0] = m[r];
      red[(warp * QB + r) * 3 + 1] = l[r];
      red[(warp * QB + r) * 3 + 2] = pick[r];
    }
  }
  __syncthreads();
  if (warp == 0) {
    float loss = 0.f;
    if (lane < QB && row0 + lane < Q) {
      float M = -INFINITY;
      for (int w = 0; w < FWD_WARPS; ++w) M = fmaxf(M, red[(w * QB + lane) * 3]);
      float L = 0.f, P = 0.f;
      for (int w = 0; w < FWD_WARPS; ++w) {
        const float mw = red[(w * QB + lane) * 3], lw = red[(w * QB + lane) * 3 + 1];
        if (mw != -INFINITY) L += lw * __expf(mw - M);
        P += red[(w * QB + lane) * 3 + 2];  // exactly one warp saw the label column (others hold 0)
      }
      const float lse = M + logf(L);
      lse_out[row0 + lane] = lse;
      loss = lse - P;
    }
    loss = warp_sum(loss);
    if (lane == 0 && loss_sum != nullptr) atomicAdd(loss_sum, loss);
  }
}

// Row reduction over stored logits (one warp per query row): lse, NLL pick, loss accumulation.
__global__ void __launch_bounds__(256)
score_lse_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, float* __restrict__ lse_out,
                 float* __restrict__ loss_sum, int Q, int C) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  float loss = 0.f;
  if (r < Q) {
    const float* row = logits + (long long)r * C;
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) m = fmaxf(m, row[c]);
    m = warp_max(m);
    float l = 0.f;
    if (m != -INFINITY)
      for (int c = lane; c < C; c += 32) l += __expf(row[c] - m);     // exp(-inf - m) = 0 for masked columns
    l = warp_sum(l);
    const float lse = m + logf(l);
    if (lane == 0) {
      lse_out[r] = lse;
      const long long lab = labels[r];
      loss = lse - ((lab >= 0 && lab < C) ? row[lab] : 0.f);
    }
  }
  __shared__ float part[8];
  if (lane == 0) part[threadIdx.x >> 5] = loss;
  __syncthreads();
  if (threadIdx.x == 0 && loss_sum != nullptr) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += part[w];
    atomicAdd(loss_sum, t);
  }
}

// out[a, k] (+)= sum_b W(a, b) * X[b, k]   with W derived from the stored logits:
//   W = (exp(logit[r,c] - lse[r]) - [c == label[r]]) * scale
// MODE 0 (dq): a = query row r in [a0, a0+na), b = all columns c, X = c matrix.
// MODE 1 (dc): a = column c in [a0, a0+na), b = all query rows r, X = q matrix.
constexpr int AB = 8;    // output rows per CTA
constexpr int BT = 32;   // reduction chunk
template <int MODE>
__global__ void __launch_bounds__(256)
score_ce_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ lse,
                    const int64_t* __restrict__ labels, const float* __restrict__ X, float scale,
                    float* __restrict__ out, int Q, int C, int d, int a0, int na, int b_per_split) {
  __shared__ float W[BT][AB + 1];
  const int ab = blockIdx.x * AB;           // first local output row
  const int k = blockIdx.y * 256 + threadIdx.x;
  const int nb_all = MODE == 0 ? C : Q;
  // gridDim.z > 1: the reduction range is split over CTAs and the (pre-zeroed) output is accumulated with atomics
  const int b_begin = blockIdx.z * b_per_split;
  const int nb = min(nb_all, b_begin + b_per_split);
  float acc[AB];
#pragma unroll
  for (int i = 0; i < AB; ++i) acc[i] = 0.f;
  for (int b0 = b_begin; b0 < nb; b0 += BT) {
    {
      // 256 threads fill the BT x AB weight tile
      int bi, ai;
      if (MODE == 0) { ai = threadIdx.x >> 5; bi = threadIdx.x & 31; }  // rows: a, contiguous: b (= column)
      else { bi = threadIdx.x >> 3; ai = threadIdx.x & 7; }             // rows: b (= query row), contiguous: a (= column)
      const int a = a0 + ab + ai, b = b0 + bi;
      float w = 0.f;
      if (ab + ai < na && b < nb) {
        const int r = MODE == 0 ? a : b, cc = MODE == 0 ? b : a;
        const float lg = logits[(long long)r * C + cc];
        w = (lg == -INFINITY) ? 0.f : __expf(lg - lse[r]);
        if ((long long)cc == labels[r]) w -= 1.f;
        w *= scale;
      }
      W[bi][ai] = w;
    }
    __syncthreads();
    if (k < d) {
#pragma unroll 8
      for (int bi = 0; bi < BT; ++bi) {
        const int b = b0 + bi;
        if (b < nb) {
          const float x = __ldg(X + (long long)b * d + k);
#pragma unroll
          for (int i = 0; i < AB; ++i) acc[i] = fmaf(W[bi][i], x, acc[i]);
        }
      }
    }
    __syncthreads();
  }
  if (k < d) {
#pragma unroll
    for (int i = 0; i < AB; ++i)
      if (ab + i < na) {
        if (gridDim.z > 1) atomicAdd(out + (long long)(ab + i) * d + k, acc[i]);
        else out[(long long)(ab + i) * d + k] = acc[i];
      }
  }
}

}  // namespace

int score_ce_fwd(const float* q, const float* c, const uint8_t* col_mask, const uint8_t* pair_mask,
                 const int64_t* labels, float inv_t, float* lse, float* loss_sum, float* logits, int Q, int C, int d,
                 cudaStream_t stream) {
  DPRB_REQUIRE(Q >= 0 && C > 0 && d > 0, "score_ce_fwd: bad shape Q=%d C=%d d=%d", Q, C, d);
  DPRB_REQUIRE(lse != nullptr, "score_ce_fwd: lse output required");
  if (Q == 0) return 0;
  DPRB_NUM_SMS(sms);
  const size_t smem = (size_t)(QB * d + FWD_WARPS * QB * 3) * sizeof(float);
  DPRB_REQUIRE(smem <= 200 * 1024, "score_ce_fwd: embedding dim %d too large", d);
  static bool attr = false;
  if (!attr) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(score_ce_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  // With the logits stored anyway (training), spread the columns over ~4 CTAs per SM and reduce the rows in a second
  // small kernel: at Q x C = 1024 x 8192 (8 GPUs) the one-CTA-per-8-rows form took ms, not us.
  const int row_blocks = (Q + QB - 1) / QB;
  const int step = FWD_WARPS * CW;
  int splits = 1;
  if (logits != nullptr) {
    splits = (4 * sms + row_blocks - 1) / row_blocks;
    const int max_splits = (C + step - 1) / step;
    splits = splits < 1 ? 1 : (splits > max_splits ? max_splits : splits);
  }
  const int cols_per_split = ((C + splits - 1) / splits + step - 1) / step * step;
  splits = (C + cols_per_split - 1) / cols_per_split;
  dim3 grid(row_blocks, splits);
  score_ce_fwd_kernel<<<grid, FWD_WARPS * 32, smem, stream>>>(q, c, col_mask, pair_mask, labels, inv_t, lse, loss_sum,
                                                              logits, Q, C, d, cols_per_split);
  DPRB_LAUNCH_CHECK();
  if (splits > 1) {
    score_lse_kernel<<<(Q + 7) / 8, 256, 0, stream>>>(logits, labels, lse, loss_sum, Q, C);
    DPRB_LAUNCH_CHECK();
  }
  return 0;
}

int score_ce_bwd(const float* q, const float* c, const float* logits, const int64_t* labels, const float* lse,
                 float grad_scale, float inv_t, float* dq, float* dc, int Q, int C, int d, int q0, int nq, int c0,
                 int nc, cudaStream_t stream) {
  DPRB_REQUIRE(Q > 0 && C > 0 && d > 0, "score_ce_bwd: bad shape Q=%d C=%d d=%d", Q, C, d);
  DPRB_REQUIRE(q0 >= 0 && nq >= 0 && q0 + nq <= Q && c0 >= 0 && nc >= 0 && c0 + nc <= C,
               "score_ce_bwd: local ranges out of bounds (q0=%d nq=%d c0=%d nc=%d)", q0, nq, c0, nc);
  DPRB_REQUIRE(logits != nullptr && lse != nullptr, "score_ce_bwd: logits and lse from forward required");
  DPRB_NUM_SMS(sms);
  const float scale = grad_scale * inv_t / (float)Q;  // d(mean CE)/d(logit) * d(logit)/d(q.c)
  // split the reduction dimension until there are ~2 CTAs per SM (dq at 8 GPUs: 16 x 3 CTAs reducing 8192 columns)
  auto launch = [&](auto kern, const float* X, float* out, int a0, int na, int nb) -> int {
    const int base = ((na + AB - 1) / AB) * ((d + 255) / 256);
    int z = (2 * sms + base - 1) / base;
    const int max_z = (nb + 4 * BT - 1) / (4 * BT);
    z = z < 1 ? 1 : (z > max_z ? max_z : z);
    const int per = ((nb + z - 1) / z + BT - 1) / BT * BT;
    z = (nb + per - 1) / per;
    if (z > 1) DPRB_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)na * d * sizeof(float), stream));
    dim3 grid((na + AB - 1) / AB, (d + 255) / 256, z);
    kern<<<grid, 256, 0, stream>>>(logits, lse, labels, X, scale, out, Q, C, d, a0, na, per);
    DPRB_LAUNCH_CHECK();
    return 0;
  };
  if (nq > 0 && dq != nullptr)
    if (int rc = launch(score_ce_bwd_kernel<0>, c, dq, q0, nq, C)) return rc;
  if (nc > 0 && dc != nullptr)
    if (int rc = launch(score_ce_bwd_kernel<1>, q, dc, c0, nc, Q)) return rc;
  return 0;
}

}  // namespace dprb
