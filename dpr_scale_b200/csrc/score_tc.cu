// In-batch-negative scoring + softmax cross-entropy on the tensor cores, ONE pass:
// similarity tile (wgmma, fp32 accumulators staged in shared memory) -> row max / sum-exp / label pick (thread = row)
// -> per-row partials -> the last tile of a row block folds them into lse + loss.  No logits in HBM unless the caller
// asks.
//
// Replaces the reference task's sim_score, its masks, the division by the temperature and nn.CrossEntropyLoss and,
// in backward, their gradient flow (only rank-local rows / columns).
//
// fp32 fidelity on bf16 tensor cores ("bf16x3"): every fp32 operand x is split into two bf16 parts x ~ h + m
// (|x - h - m| <= 2^-18 |x|), and q.c is accumulated in fp32 from the three partial products h.m, m.h, h.h (the dropped
// m.m term is 2^-18 of the product).  Each term of the dot product is therefore exact to ~2^-17; measured against the
// fp64 product the logits agree to a few 1e-6 of max|logit| - inside a 1e-5 |logit| + 1e-3 tolerance -
// where the reference under AMP computes this product in fp16 (spacing 0.25 at |s| ~ 300).  (A three-part split with
// six products was measured first: 1.5x the L2 -> shared-memory traffic, which is what bounds this kernel, for
// accuracy nobody can observe behind the fp32 softmax.)  tests/test_score_fitted_gpu.py measures at most 5.4e-6 of a
// row's max |logit| for |logit| 20 ... 250 (H100 80GB HBM3, 700 W).
//
// Softmax in base 2 (s2 = logit * log2 e): the forward keeps, per row, the max M and L = sum_j 2^(s2_j - M) less
// the maximum's own term 1, and writes M and lg2(1 + L) to the workspace.  loss = (M - s2_label) ln2 + log1p(L):
// when the label is the maximum the first term is exactly 0 and the loss (down to 1e-30 in a fitted row) keeps a few
// ulp of itself, where lse - logit[label] would be a difference of two numbers rounded at |logit|.  The backward
// forms p = 2^((s2 - M) - lg2(1 + L)), so every row of W sums to 0 within a few ulp of 1 at any |logit|.
//
// Backward recomputes tiles instead of reading stored logits: one launch rebuilds W = softmax - onehot for the local
// row block [nq x C] and the local column block [Q x nc] (bf16 hi + lo), and dq = W_rows c, dc = W_cols^T q run as
// split-K launches of the encoder's GEMM (fp32 atomic accumulate) on the h / m parts.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int TM = 128, TN = 128, BK = 64;
constexpr int PART_BYTES = 128 * 128;          // [128 rows][64 bf16], 128B-swizzled
constexpr int STAGE_BYTES = 4 * PART_BYTES;    // q.h q.m c.h c.m of one k-block
constexpr int STAGES = 2;
constexpr int EPI_THREADS = 128;
constexpr int THREADS = 128 + EPI_THREADS;     // warp 0: TMA; warps 4..7 (warpgroup 1): wgmma + epilogue
constexpr int ACC_LD = TN + 4;                 // fp32 accumulator tile [128][ACC_LD] (padded: conflict-free row reads)
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + TM * ACC_LD * 4 + 2 * 128 * 4 + 256 + 1024;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

struct Region {            // a rectangle of the score matrix, tiled 128 x 128
  int r0, nr, c0, nc;      // rows [r0, r0+nr) x columns [c0, c0+nc)
  int n_rb, n_cb;
  bf16 *w_hi, *w_lo;       // MODE_W: output [nr][ldw]
  long long ldw;
};

struct ScoreParams {
  int Q, C, d, k_blocks;
  float inv_t;
  const uint8_t* col_mask;
  const uint8_t* pair_mask;
  const int64_t* labels;
  // forward
  float* lse;
  float* loss_sum;
  float* logits;
  float* part;             // [3][n_cb][Qpad]: m2, l, pick2
  int* counters;           // [n_rb]
  int Qpad;
  float* stat;             // [2][Qpad]: row max M and lg2(sum_j 2^(s2_j - M)); written by forward, read by W mode
  Region reg[2];
  int n_regions;
};

// two-way bf16 split of fp32 data: out[0] = h = bf16(x), out[1] = m = bf16(x - h)  (part stride n elements)
__global__ void __launch_bounds__(256)
split2_kernel(const float* __restrict__ x, bf16* __restrict__ out, long long n) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float a[4] = {v.x, v.y, v.z, v.w};
    float h[4], m[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      h[t] = __bfloat162float(__float2bfloat16_rn(a[t]));
      m[t] = a[t] - h[t];
    }
    uint2 s;
    s.x = pack_bf16x2(h[0], h[1]); s.y = pack_bf16x2(h[2], h[3]);
    reinterpret_cast<uint2*>(out)[i] = s;
    s.x = pack_bf16x2(m[0], m[1]); s.y = pack_bf16x2(m[2], m[3]);
    reinterpret_cast<uint2*>(out + n)[i] = s;
  }
}

template <int MODE>   // 0: forward (row statistics, optional logits)   1: W tiles for backward
__global__ void __launch_bounds__(THREADS, 1)
score_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_c, const ScoreParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  float* sAcc = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);    // [128][ACC_LD]
  float* sMask = sAcc + TM * ACC_LD;                                        // [2][128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sMask + 256);
  uint64_t *full_bar = bars, *empty_bar = bars + STAGES;
  int* sFlag = reinterpret_cast<int*>(empty_bar + STAGES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_c);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], EPI_THREADS / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles0 = p.reg[0].n_rb * p.reg[0].n_cb;
  const int tiles = tiles0 + (p.n_regions > 1 ? p.reg[1].n_rb * p.reg[1].n_cb : 0);
  // Every CTA owns a CONTIGUOUS range of tiles in row-block-major order: consecutive tiles share the query tile (L2 /
  // TMA reuse) and, in the forward, their row statistics merge in registers - a row block ends up with one partial per
  // CTA that touched it (~n_cb / tiles_per_cta) instead of one per tile.
  const int t_base = tiles / (int)gridDim.x, t_rem = tiles % (int)gridDim.x;
  const int t_begin = (int)blockIdx.x * t_base + min((int)blockIdx.x, t_rem);
  const int t_end = t_begin + t_base + ((int)blockIdx.x < t_rem ? 1 : 0);

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = t_begin; t < t_end; ++t) {
        const Region& g = p.reg[t < tiles0 ? 0 : 1];
        const int tt = t < tiles0 ? t : t - tiles0;
        const int row0 = g.r0 + (tt / g.n_cb) * TM, col0 = g.c0 + (tt % g.n_cb) * TN;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          uint8_t* base = smem + stage * STAGE_BYTES;
#pragma unroll
          for (int part = 0; part < 2; ++part) {
            tma_load_3d(base + part * PART_BYTES, &tm_q, &full_bar[stage], kb * BK, row0, part);
            tma_load_3d(base + (2 + part) * PART_BYTES, &tm_c, &full_bar[stage], kb * BK, col0, part);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    const int tid = threadIdx.x - 128;           // 0..127 = accumulator row of the tile
    const int quarter = warp & 3;
    const float sc2 = p.inv_t * LOG2E;
    int acc = 0;                     // mask buffer of the current tile
    int stage = 0;
    uint32_t phase = 0;
    // forward: statistics of the row block in progress (thread = row), flushed when the row block changes.  l is the
    // sum of 2^(s2 - m2) over the row's columns so far LESS the one term of the maximum (exactly 1): a row whose label
    // wins by a margin keeps its tiny loss in l instead of losing it below the ulp of 1 + l.
    float m2 = -INFINITY, l = 0.f, pick = 0.f;
    int cur_rb = -1;
    auto cta_of = [&](int t) {       // inverse of the contiguous tile ranges above
      const int big = t_rem * (t_base + 1);
      return t < big ? t / (t_base + 1) : t_rem + (t - big) / max(t_base, 1);
    };
    auto flush = [&](int rb) {
      // one partial per (row block, CTA); the LAST CTA to deliver one folds them into lse + loss
      const Region& g = p.reg[0];
      const int row = rb * TM + tid;
      const bool row_ok = row < p.Q;
      const int lo = cta_of(rb * g.n_cb), hi = cta_of(rb * g.n_cb + g.n_cb - 1);
      const int nslots = hi - lo + 1, slot = (int)blockIdx.x - lo;
      const long long plane = (long long)g.n_cb * p.Qpad;
      if (row_ok) {
        float* pm = p.part + (long long)slot * p.Qpad + row;
        __stcg(pm, m2);
        __stcg(pm + plane, l);
        __stcg(pm + 2 * plane, pick);
      }
      __threadfence();
      named_bar_sync(2, EPI_THREADS);
      if (tid == 0) *sFlag = (atomicAdd(p.counters + rb, 1) == nslots - 1) ? 1 : 0;
      named_bar_sync(2, EPI_THREADS);
      if (*sFlag) {
        __threadfence();
        float loss = 0.f;
        if (row_ok) {
          const float* base = p.part + row;
          float M = -INFINITY;
#pragma unroll 4
          for (int b = 0; b < nslots; ++b) M = fmaxf(M, __ldcg(base + (long long)b * p.Qpad));
          float L = 0.f, P = 0.f;                              // L: the row's sum less its maximum term
          bool top = false;                                    // the maximum term of one slot with mb == M is left out
          const float Mf = (M == -INFINITY) ? 0.f : M;       // all-masked row: every l is 0
#pragma unroll 4
          for (int b = 0; b < nslots; ++b) {
            const float mb = __ldcg(base + (long long)b * p.Qpad);
            const float lb = __ldcg(base + plane + (long long)b * p.Qpad);
            P += __ldcg(base + 2 * plane + (long long)b * p.Qpad);   // one slot saw the label, the others hold 0
            if (!top && mb == M) { L += lb; top = true; }
            else { const float r = ex2_approx(mb - Mf); L += fmaf(lb, r, r); }   // mb = -inf: lb = 0, ex2(-inf) = 0
          }
          // loss = lse - logit[label] = (M - pick2) ln2 + ln(1 + L): exact 0 difference when the label is the maximum,
          // and log1p keeps a fitted row's loss (L down to 1e-30) to a few ulp of itself
          const float lnL = log1pf(L);
          p.stat[row] = M;
          p.stat[p.Qpad + row] = lnL * LOG2E;
          const float lse = (M == -INFINITY) ? -INFINITY : fmaf(M, LN2, lnL);
          p.lse[row] = lse;
          loss = (M == -INFINITY) ? lse - P * LN2 : fmaf(M - P, LN2, lnL);
        }
        loss = warp_sum(loss);
        if (lane == 0 && p.loss_sum != nullptr) atomicAdd(p.loss_sum, loss);
        if (tid == 0) p.counters[rb] = 0;                      // ready for the next call
      }
      named_bar_sync(2, EPI_THREADS);                          // sFlag is rewritten by the next flush
    };
    for (int t = t_begin; t < t_end; ++t) {
      const Region& g = p.reg[t < tiles0 ? 0 : 1];
      const int tt = t < tiles0 ? t : t - tiles0;
      const int rb = tt / g.n_cb, cb = tt % g.n_cb;
      if (MODE == 0 && rb != cur_rb) {
        if (cur_rb >= 0) flush(cur_rb);
        m2 = -INFINITY; l = 0.f; pick = 0.f;
        cur_rb = rb;
      }
      const int row = g.r0 + rb * TM + tid;                  // global query row of this thread
      const int colbase = g.c0 + cb * TN;
      const int col_end = g.c0 + g.nc;                       // exclusive (== C in forward)
      const bool row_ok = row < g.r0 + g.nr;
      float* mk = sMask + acc * 128;
      {
        const int col = colbase + tid;
        const bool dead = col >= col_end || (p.col_mask != nullptr && p.col_mask[col] != 0);
        mk[tid] = dead ? -INFINITY : 0.f;
      }
      const long long lab = row_ok ? p.labels[row] : -1;
      named_bar_sync(1, EPI_THREADS);
      {
        // q.c over all k-blocks, small partial products first: (h,m) (m,h) (h,h); rows [0, 64) and [64, 128)
        float d0[64], d1[64];
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t base = smem_u32(smem + stage * STAGE_BYTES);
          constexpr int PA[3] = {0, 1, 0};
          constexpr int PB[3] = {1, 0, 0};
          wgmma_fence();
#pragma unroll
          for (int pr = 0; pr < 3; ++pr) {
            const uint64_t da = make_wgmma_desc_sw128(base + PA[pr] * PART_BYTES, 16, 1024);
            const uint64_t db = make_wgmma_desc_sw128(base + (2 + PB[pr]) * PART_BYTES, 16, 1024);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
              const int accum = (kb > 0 || pr > 0 || k > 0) ? 1 : 0;
              wgmma_m64n128_ss_bf16<0, 0>(d0, da + 2 * k, db + 2 * k, accum);
              wgmma_m64n128_ss_bf16<0, 0>(d1, da + 64 * 8 + 2 * k, db + 2 * k, accum);   // +64 rows of 128 B
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        store_acc_128x128<ACC_LD>(sAcc, d0, d1, quarter, lane);   // each thread then reads the row it owns
      }
      named_bar_sync(3, EPI_THREADS);
      const float* arow = sAcc + tid * ACC_LD;
      if (MODE == 0) {
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
          uint32_t r[32];
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(r + j) = *reinterpret_cast<const float4*>(arow + c * 32 + j);
          const int col0 = colbase + c * 32;
          float s2[32];
          float cmax = -INFINITY;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float v = __uint_as_float(r[j]) * sc2 + mk[c * 32 + j];
            if (p.pair_mask != nullptr && row_ok && col0 + j < col_end && p.pair_mask[(long long)row * p.C + col0 + j] != 0)
              v = -INFINITY;
            s2[j] = v;
            cmax = fmaxf(cmax, v);
          }
          if (p.logits != nullptr && row_ok) {
            float* dst = p.logits + (long long)row * p.C + col0;
            if (col0 + 32 <= col_end && (p.C & 3) == 0) {
#pragma unroll
              for (int j = 0; j < 32; j += 4)
                *reinterpret_cast<float4*>(dst + j) = make_float4(s2[j] * LN2, s2[j + 1] * LN2, s2[j + 2] * LN2, s2[j + 3] * LN2);
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) if (col0 + j < col_end) dst[j] = s2[j] * LN2;
            }
          }
          if (lab >= col0 && lab < col0 + 32) {
#pragma unroll
            for (int j = 0; j < 32; ++j) if (lab == col0 + j) pick = s2[j];
          }
          bool skip = false;                                   // a new maximum: its own term (1) stays out of l
          if (cmax > m2) {                                     // the old maximum term joins l, rescaled
            const float r = ex2_approx(m2 - cmax);             // m2 = -inf: l is 0, ex2(-inf) = 0
            l = fmaf(l, r, r);
            m2 = cmax;
            skip = true;
          }
          if (m2 != -INFINITY) {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float e = ex2_approx(s2[j] - m2);
              if (skip && s2[j] == m2) skip = false;           // an equal second maximum adds its 1 to l
              else l += e;
            }
          }
          __syncwarp();
        }
      } else {
        // p = 2^((s2 - M) - lg2(1 + L)) from the forward's row statistics: s2 - M is exact near the maximum, so every p
        // of a row carries only its own rounding and the row of W sums to 0 to a few ulp of 1 (a lse rounded at
        // |logit| would scale the whole row by 1 + O(ulp(|logit|)))
        const float m2r = row_ok ? p.stat[row] : INFINITY;
        const float lgr = row_ok ? p.stat[p.Qpad + row] : 0.f;
        const int lrow = rb * TM + tid;                       // row inside the region's W array
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
          uint32_t r[32];
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(r + j) = *reinterpret_cast<const float4*>(arow + c * 32 + j);
          const int col0 = colbase + c * 32;
          uint32_t hi[16], lo[16];
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            float w[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float v = __uint_as_float(r[j + e]) * sc2 + mk[c * 32 + j + e];
              if (p.pair_mask != nullptr && row_ok && col0 + j + e < p.C && p.pair_mask[(long long)row * p.C + col0 + j + e] != 0)
                v = -INFINITY;
              float pw = ex2_approx((v - m2r) - lgr);        // masked / out-of-range: ex2(-inf) = 0
              if (lab == col0 + j + e) pw -= 1.f;
              w[e] = pw;
            }
            const uint32_t h = pack_bf16x2(w[0], w[1]);
            const float2 hf = unpack_bf16x2(h);
            hi[j >> 1] = h;
            lo[j >> 1] = pack_bf16x2(w[0] - hf.x, w[1] - hf.y);
          }
          if (row_ok) {
            const long long off = (long long)lrow * g.ldw + (col0 - g.c0);
            if (col0 + 32 <= col_end) {
#pragma unroll
              for (int q4 = 0; q4 < 4; ++q4) {
                *reinterpret_cast<uint4*>(g.w_hi + off + q4 * 8) = make_uint4(hi[q4 * 4], hi[q4 * 4 + 1], hi[q4 * 4 + 2], hi[q4 * 4 + 3]);
                *reinterpret_cast<uint4*>(g.w_lo + off + q4 * 8) = make_uint4(lo[q4 * 4], lo[q4 * 4 + 1], lo[q4 * 4 + 2], lo[q4 * 4 + 3]);
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                if (col0 + j < col_end) {
                  const uint32_t hh = hi[j >> 1], ll = lo[j >> 1];
                  reinterpret_cast<uint16_t*>(g.w_hi)[off + j] = (uint16_t)((j & 1) ? (hh >> 16) : (hh & 0xFFFFu));
                  reinterpret_cast<uint16_t*>(g.w_lo)[off + j] = (uint16_t)((j & 1) ? (ll >> 16) : (ll & 0xFFFFu));
                }
              }
            }
          }
          __syncwarp();
        }
      }
      named_bar_sync(3, EPI_THREADS);                          // every row of sAcc read before the next tile
      acc ^= 1;
    }
    if (MODE == 0 && cur_rb >= 0) flush(cur_rb);
  }

  __syncthreads();
}

// bf16 [2 parts][rows][d]; box = [1][128 rows][64 cols], 128B swizzle; rows / columns beyond the extent are zero-filled
int make_tmap_parts(CUtensorMap* out, const void* base, long long rows, long long d) {
  const cuuint64_t dims[3] = {(cuuint64_t)d, (cuuint64_t)rows, 2};
  const cuuint64_t strides[2] = {(cuuint64_t)d * 2, (cuuint64_t)rows * d * 2};
  const cuuint32_t box[3] = {64u, 128u, 1u};
  return encode_tmap(out, "score", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

struct ScoreWs {
  bf16 *q3, *c3;
  float* part;
  float* stat;
  int* counters;
  bf16 *wr_hi, *wr_lo, *wc_hi, *wc_lo;
  long long ld_wr, ld_wc;
  int Qpad, n_rb, n_cb;
  long long bytes;
};

ScoreWs plan(void* base, int Q, int C, int d, int nq, int nc) {
  ScoreWs w;
  Carve cv(base);
  w.n_rb = (Q + TM - 1) / TM; w.n_cb = (C + TN - 1) / TN; w.Qpad = w.n_rb * TM;
  w.q3 = (bf16*)cv.take(2LL * Q * d * 2);
  w.c3 = (bf16*)cv.take(2LL * C * d * 2);
  w.part = (float*)cv.take(3LL * w.n_cb * w.Qpad * 4);
  w.stat = (float*)cv.take(2LL * w.Qpad * 4);
  w.counters = (int*)cv.take((long long)w.n_rb * 4);
  w.ld_wr = (C + 7) & ~7LL; w.ld_wc = ((long long)nc + 7) & ~7LL;
  w.wr_hi = (bf16*)cv.take((long long)nq * w.ld_wr * 2);
  w.wr_lo = (bf16*)cv.take((long long)nq * w.ld_wr * 2);
  w.wc_hi = (bf16*)cv.take((long long)Q * w.ld_wc * 2);
  w.wc_lo = (bf16*)cv.take((long long)Q * w.ld_wc * 2);
  w.bytes = cv.off;
  return w;
}

int set_attr() {
  static bool done = false;
  if (!done) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(score_tc_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(score_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    done = true;
  }
  return 0;
}

int grid_for(long long n4, int sms) {
  long long want = (n4 + 255) / 256;
  if (want < 1) want = 1;
  return (int)(want < (long long)sms * 4 ? want : (long long)sms * 4);
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int64_t dprb_score_tc_workspace_bytes(int Q, int C, int d, int nq, int nc) {
  return plan(nullptr, Q, C, d, nq < 0 ? Q : nq, nc < 0 ? C : nc).bytes;
}

extern "C" int dprb_score_tc_fwd(const float* q, const float* c, const uint8_t* col_mask, const uint8_t* pair_mask,
                                 const int64_t* labels, float inv_t, float* lse, float* loss_sum, float* logits, int Q,
                                 int C, int d, int nq, int nc, void* workspace, int64_t workspace_bytes,
                                 dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(Q >= 0 && C > 0 && d > 0, "score_tc_fwd: bad shape Q=%d C=%d d=%d", Q, C, d);
  DPRB_REQUIRE(d % 8 == 0, "score_tc_fwd: d=%d must be a multiple of 8 (16-byte rows for TMA)", d);
  if (Q == 0) return 0;
  DPRB_REQUIRE(lse != nullptr, "score_tc_fwd: lse output required");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(c)) & 15) == 0, "score_tc_fwd: q / c must be 16-byte aligned");
  ScoreWs w = plan(workspace, Q, C, d, nq < 0 ? Q : nq, nc < 0 ? C : nc);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= w.bytes && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
               "score_tc_fwd: workspace missing, misaligned or too small (%lld < %lld)", (long long)workspace_bytes,
               w.bytes);
  if (int rc = set_attr()) return rc;
  DPRB_NUM_SMS(sms);
  const long long nqd = (long long)Q * d, ncd = (long long)C * d;
  split2_kernel<<<grid_for(nqd >> 2, sms), 256, 0, stream>>>(q, w.q3, nqd);
  DPRB_LAUNCH_CHECK();
  split2_kernel<<<grid_for(ncd >> 2, sms), 256, 0, stream>>>(c, w.c3, ncd);
  DPRB_LAUNCH_CHECK();
  DPRB_CHECK_CUDA(cudaMemsetAsync(w.counters, 0, (size_t)w.n_rb * 4, stream));
  CUtensorMap tq, tc;
  if (int rc = make_tmap_parts(&tq, w.q3, Q, d)) return rc;
  if (int rc = make_tmap_parts(&tc, w.c3, C, d)) return rc;
  ScoreParams p = {};
  p.Q = Q; p.C = C; p.d = d; p.k_blocks = (d + BK - 1) / BK; p.inv_t = inv_t;
  p.col_mask = col_mask; p.pair_mask = pair_mask; p.labels = labels;
  p.lse = lse; p.loss_sum = loss_sum; p.logits = logits; p.part = w.part; p.counters = w.counters; p.Qpad = w.Qpad;
  p.stat = w.stat;
  p.n_regions = 1;
  p.reg[0] = Region{0, Q, 0, C, w.n_rb, w.n_cb, nullptr, nullptr, 0};
  const int tiles = w.n_rb * w.n_cb;
  score_tc_kernel<0><<<tiles < sms ? tiles : sms, THREADS, SMEM_BYTES, stream>>>(tq, tc, p);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_score_tc_bwd(const uint8_t* col_mask, const uint8_t* pair_mask, const int64_t* labels,
                                 const float* lse, float grad_scale, float inv_t, float* dq, float* dc, int Q, int C,
                                 int d, int q0, int nq, int c0, int nc, void* workspace, int64_t workspace_bytes,
                                 dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(Q > 0 && C > 0 && d > 0, "score_tc_bwd: bad shape Q=%d C=%d d=%d", Q, C, d);
  DPRB_REQUIRE(d % 8 == 0, "score_tc_bwd: d=%d must be a multiple of 8 (16-byte rows for TMA)", d);
  DPRB_REQUIRE(q0 >= 0 && nq >= 0 && q0 + nq <= Q && c0 >= 0 && nc >= 0 && c0 + nc <= C,
               "score_tc_bwd: local ranges out of bounds (q0=%d nq=%d c0=%d nc=%d)", q0, nq, c0, nc);
  ScoreWs w = plan(workspace, Q, C, d, nq, nc);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= w.bytes, "score_tc_bwd: workspace too small (the forward call must "
               "have been given the same nq / nc)");
  if (int rc = set_attr()) return rc;
  CUtensorMap tq, tc;
  if (int rc = make_tmap_parts(&tq, w.q3, Q, d)) return rc;
  if (int rc = make_tmap_parts(&tc, w.c3, C, d)) return rc;
  ScoreParams p = {};
  p.Q = Q; p.C = C; p.d = d; p.k_blocks = (d + BK - 1) / BK; p.inv_t = inv_t;
  p.col_mask = col_mask; p.pair_mask = pair_mask; p.labels = labels;
  p.stat = w.stat; p.Qpad = w.Qpad;                          // the forward's row statistics (lse is not read)
  int nreg = 0;
  const bool want_dq = nq > 0 && dq != nullptr, want_dc = nc > 0 && dc != nullptr;
  if (want_dq) p.reg[nreg++] = Region{q0, nq, 0, C, (nq + TM - 1) / TM, (C + TN - 1) / TN, w.wr_hi, w.wr_lo, w.ld_wr};
  if (want_dc) p.reg[nreg++] = Region{0, Q, c0, nc, (Q + TM - 1) / TM, (nc + TN - 1) / TN, w.wc_hi, w.wc_lo, w.ld_wc};
  if (nreg == 0) return 0;
  p.n_regions = nreg;
  int tiles = 0;
  for (int i = 0; i < nreg; ++i) tiles += p.reg[i].n_rb * p.reg[i].n_cb;
  DPRB_NUM_SMS(sms);
  score_tc_kernel<1><<<tiles < sms ? tiles : sms, THREADS, SMEM_BYTES, stream>>>(tq, tc, p);
  DPRB_LAUNCH_CHECK();
  const float scale = grad_scale * inv_t / (float)Q;        // d(mean CE)/d(logit) * d(logit)/d(q.c)
  const bf16 *c_h = w.c3, *c_m = w.c3 + (long long)C * d, *q_h = w.q3, *q_m = w.q3 + (long long)Q * d;
  if (want_dq) {
    // dq[nq, d] = W_rows[nq, C] c[C, d]  with  W = hi + lo, c = h + m  (the lo.m term is below 2^-17 of the result)
    DPRB_CHECK_CUDA(cudaMemsetAsync(dq, 0, (size_t)nq * d * sizeof(float), stream));
    const bf16* A[3] = {w.wr_hi, w.wr_hi, w.wr_lo};
    const bf16* B[3] = {c_h, c_m, c_h};
    for (int i = 0; i < 3; ++i)
      if (int rc = dprb_gemm_bf16(A[i], B[i], dq, nq, d, C, w.ld_wr, d, d, 0, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0,
                             nullptr, scale, 0, nullptr, 0.f, 0, stream)) return rc;
  }
  if (want_dc) {
    // dc[nc, d] = W_cols[Q, nc]^T q[Q, d]: both operands read MN-major in place
    DPRB_CHECK_CUDA(cudaMemsetAsync(dc, 0, (size_t)nc * d * sizeof(float), stream));
    const bf16* A[3] = {w.wc_hi, w.wc_hi, w.wc_lo};
    const bf16* B[3] = {q_h, q_m, q_h};
    for (int i = 0; i < 3; ++i)
      if (int rc = dprb_gemm_bf16(A[i], B[i], dc, nc, d, Q, w.ld_wc, d, d, 1, 1, DPRB_EPI_F32_ATOMIC_ADD, nullptr, nullptr, 0,
                             nullptr, scale, 0, nullptr, 0.f, 0, stream)) return rc;
  }
  return 0;
}
