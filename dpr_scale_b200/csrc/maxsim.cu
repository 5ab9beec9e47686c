// Late-interaction (ColBERT MaxSim) scoring of reranking pairs on the tensor cores, forward only.
//
// Replaces RerankMultiVecRetrieverTask.expert_sim_score of the reference (dpr_scale/task/citadel_eval_task.py:236-265,
// no expert ids): scores = bmm(q, d^T) [B, LQ, LD], then max over LD and sum (or max) over LQ, where q / d are the
// encoders' projected last-layer tokens without token 0, multiplied by their attention masks
// (dpr_scale/models/citadel_models/colbert_model.py:39-44).
//
// One CTA per pair: warp 4 streams (query chunk, passage chunk) stages with TMA - 64 query rows x 64 of P and 128 passage
// rows x 64 of P, K-major, 128B-swizzled, zero-filled beyond P and beyond the sequence - and warps 0-3 (one warpgroup)
// run S = Q D^T with wgmma m64n128k16 into fp32 registers, keep a running max per query row over the passage blocks,
// then reduce the rows of the 64-row query block in a fixed order.  Query blocks (LQ > 64) are visited one after the
// other by the same CTA and combined by its thread 0 in block order, so a score is bitwise repeatable.
//
// The reference's padding semantics are reproduced, not fixed: a masked token is a zero vector there, so
//   * a masked passage column inside the batch's width scores exactly 0 and takes part in the max;
//   * a masked query row scores exactly 0 (adds 0 under sum, offers 0 under max);
//   * columns / rows beyond the tensor width (LD = SD - 1, LQ = SQ - 1) do not exist.
//
// maxsim_expert_kernel is the same pipeline with the expert-matching rule of COIL and CITADEL (the expert-id branch of
// expert_sim_score, citadel_eval_task.py:240-258): query token i has KQ (id, weight) pairs, passage token j has KD, and
// the (i, a) x (j, b) entry of the score matrix is S[i][j] * (wq[i][a] * wd[j][b]) where the ids agree and exactly 0
// where they differ.  Rows are (i, a), columns (j, b): each thread keeps a running max per (row, a) in registers over
// every (j, b), with the passage's ids and weights staged once in shared memory.  The masks enter through the weights
// alone (a masked token has weight 0 on its side), and an optional CLS dot product is added in fp32 at the end.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int QROWS = 64, DCOLS = 128, BK = 64;
constexpr int Q_BYTES = QROWS * BK * 2;             // [64 rows][64 bf16], 128B-swizzled
constexpr int D_BYTES = DCOLS * BK * 2;             // [128 rows][64 bf16]
constexpr int STAGE_BYTES = Q_BYTES + D_BYTES;
constexpr int STAGES = 4;
constexpr int MAX_S = 512;
constexpr int THREADS = 128 + 32;                   // warps 0-3: wgmma + reduction; warp 4: TMA producer
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + MAX_S * 4 + 2 * 4 * 4 + 2 * STAGES * 8 + 1024;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");

// passage column kinds
constexpr int COL_REAL = 0, COL_ZERO = 1, COL_NONE = 2;

struct MaxSimParams {
  const int32_t* q_mask;     // [nq, SQ] (NULL: all tokens real)
  const int32_t* d_mask;     // [B, SD]  (NULL: all tokens real)
  const int32_t* q_index;    // [B]
  float* score;              // [B]
  int nq, SQ, SD, P, pool;
};

// The stage ring of maxsim_expert_kernel (maxsim_kernel keeps its own inline copy of the same two loops, so that its
// machine code stays exactly what it was).
// warp 4, lane 0: streams the (query chunk, passage chunk) stages of every (query block, passage block, k chunk) in the
// order the consumers take them
__device__ __forceinline__ void produce_stages(const CUtensorMap& tm_q, const CUtensorMap& tm_d, uint8_t* smem,
                                               uint64_t* full_bar, uint64_t* empty_bar, int qi, int pair, int n_qb,
                                               int n_db, int n_k) {
  int stage = 0;
  uint32_t phase = 0;
  for (int qb = 0; qb < n_qb; ++qb)
    for (int db = 0; db < n_db; ++db)
      for (int kc = 0; kc < n_k; ++kc) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
        uint8_t* base = smem + stage * STAGE_BYTES;
        tma_load_3d(base, &tm_q, &full_bar[stage], kc * BK, 1 + qb * QROWS, qi);             // token 0 skipped
        tma_load_3d(base + Q_BYTES, &tm_d, &full_bar[stage], kc * BK, 1 + db * DCOLS, pair);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
}

// warps 0-3: acc = the 64 x 128 tile S = Q D^T of one (query block, passage block), over its n_k stages
__device__ __forceinline__ void mma_tile(float (&acc)[64], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                         int& stage, uint32_t& phase, int n_k, int lane) {
  for (int kc = 0; kc < n_k; ++kc) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t base = smem_u32(smem + stage * STAGE_BYTES);
    const uint64_t da = make_wgmma_desc_sw128(base, 16, 1024);
    const uint64_t dd = make_wgmma_desc_sw128(base + Q_BYTES, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) wgmma_m64n128_ss_bf16<0, 0>(acc, da + 2 * k, dd + 2 * k, (kc > 0 || k > 0) ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
}

__global__ void __launch_bounds__(THREADS, 1)
maxsim_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_d, const MaxSimParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  int* sCol = reinterpret_cast<int*>(smem + STAGES * STAGE_BYTES);          // [MAX_S] passage column kinds
  float* sWarp = reinterpret_cast<float*>(sCol + MAX_S);                     // [2][4] per-warp partials
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sWarp + 8);
  uint64_t* empty_bar = full_bar + STAGES;

  const int pair = (int)blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qi = p.q_index[pair];
  if (qi < 0 || qi >= p.nq) {                        // the host checks the indices; never read another pair's rows
    if (threadIdx.x == 0) p.score[pair] = __int_as_float(0x7fc00000);
    return;
  }
  const int LQ = p.SQ - 1, LD = p.SD - 1;
  const int n_qb = (LQ + QROWS - 1) / QROWS, n_db = (LD + DCOLS - 1) / DCOLS, n_k = (p.P + BK - 1) / BK;

  for (int j = threadIdx.x; j < n_db * DCOLS; j += THREADS) {
    int kind = COL_NONE;
    if (j < LD) kind = (p.d_mask == nullptr || p.d_mask[(long long)pair * p.SD + j + 1] != 0) ? COL_REAL : COL_ZERO;
    sCol[j] = kind;
  }
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_d);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int qb = 0; qb < n_qb; ++qb)
        for (int db = 0; db < n_db; ++db)
          for (int kc = 0; kc < n_k; ++kc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
            uint8_t* base = smem + stage * STAGE_BYTES;
            tma_load_3d(base, &tm_q, &full_bar[stage], kc * BK, 1 + qb * QROWS, qi);             // token 0 skipped
            tma_load_3d(base + Q_BYTES, &tm_d, &full_bar[stage], kc * BK, 1 + db * DCOLS, pair);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
    }
    return;
  }

  const int q4 = lane & 3;
  int stage = 0;
  uint32_t phase = 0;
  float total = 0.f;                                 // thread 0: the pair's score over the query blocks so far
  for (int qb = 0; qb < n_qb; ++qb) {
    float m0 = -INFINITY, m1 = -INFINITY;            // running max of rows r0 and r0 + 8 over the passage columns
    for (int db = 0; db < n_db; ++db) {
      float acc[64];
      for (int kc = 0; kc < n_k; ++kc) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t base = smem_u32(smem + stage * STAGE_BYTES);
        const uint64_t da = make_wgmma_desc_sw128(base, 16, 1024);
        const uint64_t dd = make_wgmma_desc_sw128(base + Q_BYTES, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_m64n128_ss_bf16<0, 0>(acc, da + 2 * k, dd + 2 * k, (kc > 0 || k > 0) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      const int* kinds = sCol + db * DCOLS;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kind = kinds[8 * c + 2 * q4 + e];
          float v0 = acc[4 * c + e], v1 = acc[4 * c + 2 + e];
          if (kind != COL_REAL) {
            v0 = v1 = (kind == COL_ZERO) ? 0.f : -INFINITY;
          }
          m0 = fmaxf(m0, v0);
          m1 = fmaxf(m1, v1);
        }
      }
    }
    // the four lanes of a quad hold disjoint columns of the same two rows
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    const float none = p.pool == DPRB_MAXSIM_SUM ? 0.f : -INFINITY;
    float v[2] = {m0, m1};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = qb * QROWS + warp * 16 + (lane >> 2) + 8 * h;       // query token r + 1
      if (r >= LQ) v[h] = none;
      else if (p.q_mask != nullptr && p.q_mask[(long long)qi * p.SQ + r + 1] == 0) v[h] = 0.f;
    }
    float s = p.pool == DPRB_MAXSIM_SUM ? v[0] + v[1] : fmaxf(v[0], v[1]);
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, s, o);
      s = p.pool == DPRB_MAXSIM_SUM ? s + t : fmaxf(s, t);
    }
    float* sw = sWarp + 4 * (qb & 1);
    if (lane == 0) sw[warp] = s;
    named_bar_sync(1, 128);
    if (threadIdx.x == 0) {
      const float b = p.pool == DPRB_MAXSIM_SUM ? (sw[0] + sw[1]) + (sw[2] + sw[3])
                                                : fmaxf(fmaxf(sw[0], sw[1]), fmaxf(sw[2], sw[3]));
      total = qb == 0 ? b : (p.pool == DPRB_MAXSIM_SUM ? total + b : fmaxf(total, b));
    }
  }
  if (threadIdx.x == 0) p.score[pair] = total;
}

constexpr int MAX_EXPERTS = 8, MAX_PC = 1024;
constexpr int EXPERT_SMEM_BYTES = STAGES * STAGE_BYTES + MAX_S * MAX_EXPERTS * 8 + 3 * 4 * 4 + 2 * STAGES * 8 + 1024;
static_assert(EXPERT_SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");

struct MaxSimExpertParams {
  const int32_t* q_ids;      // [nq, SQ, KQ]
  const float* q_w;          // [nq, SQ, KQ]
  const int32_t* d_ids;      // [B, SD, KD]
  const float* d_w;          // [B, SD, KD]
  const __nv_bfloat16* q_cls;  // [nq, Pc] (NULL: no CLS term)
  const __nv_bfloat16* d_cls;  // [B, Pc]
  const int32_t* q_index;    // [B]
  float* score;              // [B]
  int nq, SQ, SD, P, KQ, KD, Pc, pool;
};

// KQ_MAX: the query experts held per row in registers (KQ rounded up to 1, 2, 4 or 8; the rest are never matched and
// take no part in the row reduction)
template <int KQ_MAX>
__global__ void __launch_bounds__(THREADS, 1)
maxsim_expert_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_d,
                     const MaxSimExpertParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  int2* sCol = reinterpret_cast<int2*>(smem + STAGES * STAGE_BYTES);       // [LD][KD] (id, weight bits), tokens 1..
  float* sWarp = reinterpret_cast<float*>(sCol + MAX_S * MAX_EXPERTS);      // [2][4] per-warp partials
  float* sCls = sWarp + 8;                                                  // [4] per-warp CLS partials
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sCls + 4);
  uint64_t* empty_bar = full_bar + STAGES;

  const int pair = (int)blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qi = p.q_index[pair];
  if (qi < 0 || qi >= p.nq) {                        // the host checks the indices; never read another pair's rows
    if (threadIdx.x == 0) p.score[pair] = __int_as_float(0x7fc00000);
    return;
  }
  const int LQ = p.SQ - 1, LD = p.SD - 1, KD = p.KD;
  const int n_qb = (LQ + QROWS - 1) / QROWS, n_db = (LD + DCOLS - 1) / DCOLS, n_k = (p.P + BK - 1) / BK;

  {
    const long long o = ((long long)pair * p.SD + 1) * KD;
    for (int e = threadIdx.x; e < LD * KD; e += THREADS)
      sCol[e] = make_int2(p.d_ids[o + e], __float_as_int(p.d_w[o + e]));
  }
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_d);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) produce_stages(tm_q, tm_d, smem, full_bar, empty_bar, qi, pair, n_qb, n_db, n_k);
    return;
  }

  // CLS term while the first stages land: fixed-order partials per thread, per warp, then over the warps (thread 0)
  if (p.q_cls != nullptr) {
    const __nv_bfloat16* qc = p.q_cls + (long long)qi * p.Pc;
    const __nv_bfloat16* dc = p.d_cls + (long long)pair * p.Pc;
    float c = 0.f;
    for (int k = 8 * threadIdx.x; k < p.Pc; k += 8 * 128) {
      const uint4 a = *reinterpret_cast<const uint4*>(qc + k), b = *reinterpret_cast<const uint4*>(dc + k);
      const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const float2 x = unpack_bf16x2(av[h]), y = unpack_bf16x2(bv[h]);
        c = fmaf(x.x, y.x, c);
        c = fmaf(x.y, y.y, c);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) sCls[warp] = c;                   // read by thread 0 after the first query block's barrier
  }

  const int q4 = lane & 3;
  const float none = p.pool == DPRB_MAXSIM_SUM ? 0.f : -INFINITY;
  int stage = 0;
  uint32_t phase = 0;
  float total = 0.f;                                 // thread 0: the pair's score over the query blocks so far
  for (int qb = 0; qb < n_qb; ++qb) {
    // this thread's two query rows r0 and r0 + 8: their expert ids / weights and one running max per expert
    int qid[2][KQ_MAX];
    float qw[2][KQ_MAX], m[2][KQ_MAX];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = qb * QROWS + warp * 16 + (lane >> 2) + 8 * h;       // query token r + 1
      const long long o = ((long long)qi * p.SQ + r + 1) * p.KQ;
#pragma unroll
      for (int a = 0; a < KQ_MAX; ++a) {
        const bool real = r < LQ && a < p.KQ;
        qid[h][a] = real ? p.q_ids[o + a] : 0;
        qw[h][a] = real ? p.q_w[o + a] : 0.f;        // weight 0: the entry is 0 whatever the ids
        m[h][a] = -INFINITY;
      }
    }
    for (int db = 0; db < n_db; ++db) {
      float acc[64];
      mma_tile(acc, smem, full_bar, empty_bar, stage, phase, n_k, lane);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = db * DCOLS + 8 * c + 2 * q4 + e;                // passage token j + 1
          if (j >= LD) continue;                                         // beyond the width: no column
          const float s[2] = {acc[4 * c + e], acc[4 * c + 2 + e]};
          const int2* col = sCol + j * KD;
          for (int b = 0; b < KD; ++b) {
            const int2 iw = col[b];
            const float wd = __int_as_float(iw.y);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int a = 0; a < KQ_MAX; ++a) {
                const float w = qid[h][a] == iw.x ? qw[h][a] * wd : 0.f;
                m[h][a] = fmaxf(m[h][a], w != 0.f ? s[h] * w : 0.f);
              }
          }
        }
      }
    }
    // the four lanes of a quad hold disjoint columns of the same two rows; rows (i, a) reduce h-major, then a
    float s = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = qb * QROWS + warp * 16 + (lane >> 2) + 8 * h;
#pragma unroll
      for (int a = 0; a < KQ_MAX; ++a) {
        float v = m[h][a];
        v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
        v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
        if (r >= LQ || a >= p.KQ) v = none;
        s = (h == 0 && a == 0) ? v : (p.pool == DPRB_MAXSIM_SUM ? s + v : fmaxf(s, v));
      }
    }
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, s, o);
      s = p.pool == DPRB_MAXSIM_SUM ? s + t : fmaxf(s, t);
    }
    float* sw = sWarp + 4 * (qb & 1);
    if (lane == 0) sw[warp] = s;
    named_bar_sync(1, 128);
    if (threadIdx.x == 0) {
      const float b = p.pool == DPRB_MAXSIM_SUM ? (sw[0] + sw[1]) + (sw[2] + sw[3])
                                                : fmaxf(fmaxf(sw[0], sw[1]), fmaxf(sw[2], sw[3]));
      total = qb == 0 ? b : (p.pool == DPRB_MAXSIM_SUM ? total + b : fmaxf(total, b));
    }
  }
  if (threadIdx.x == 0) {
    if (p.q_cls != nullptr) total += (sCls[0] + sCls[1]) + (sCls[2] + sCls[3]);
    p.score[pair] = total;
  }
}

// bf16 [n][S][P], box = [64 of P][rows][1]; everything beyond P or S reads as zero
int make_tmap_tokens(CUtensorMap* out, const void* base, long long n, int S, int P, int rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)P, (cuuint64_t)S, (cuuint64_t)n};
  const cuuint64_t strides[2] = {(cuuint64_t)P * 2, (cuuint64_t)S * P * 2};
  const cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)rows, 1u};
  return encode_tmap(out, "maxsim", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

template <int KQ_MAX>
int launch_maxsim_expert(const CUtensorMap& tq, const CUtensorMap& td, const MaxSimExpertParams& prm, int B,
                         cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_expert_kernel<KQ_MAX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         EXPERT_SMEM_BYTES));
    attr_done = true;
  }
  maxsim_expert_kernel<KQ_MAX><<<(unsigned)B, THREADS, EXPERT_SMEM_BYTES, stream>>>(tq, td, prm);
  DPRB_LAUNCH_CHECK();
  return 0;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_maxsim_fwd(const void* q, const void* d, const int32_t* q_mask, const int32_t* d_mask,
                               const int32_t* q_index, int nq, int SQ, int B, int SD, int P, int pool, float* score,
                               dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(P % 8 == 0 && P >= 8 && P <= 1024, "maxsim_fwd: P=%d unsupported (multiple of 8, at most 1024)", P);
  DPRB_REQUIRE(SQ >= 2 && SQ <= MAX_S && SD >= 2 && SD <= MAX_S,
               "maxsim_fwd: sequence lengths SQ=%d SD=%d unsupported (2 .. 512, token 0 is skipped)", SQ, SD);
  DPRB_REQUIRE(pool == DPRB_MAXSIM_SUM || pool == DPRB_MAXSIM_MAX, "maxsim_fwd: pool %d unknown", pool);
  DPRB_REQUIRE(nq >= 1 && B >= 0, "maxsim_fwd: nq=%d B=%d", nq, B);
  if (B == 0) return 0;
  DPRB_REQUIRE(q != nullptr && d != nullptr && q_index != nullptr && score != nullptr, "maxsim_fwd: NULL operand");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(d)) & 15) == 0,
               "maxsim_fwd: q / d must be 16-byte aligned");
  const long long grid = B;
  DPRB_REQUIRE(grid < (1LL << 31), "maxsim_fwd: grid too large");
  static bool attr_done = false;
  if (!attr_done) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_done = true;
  }
  CUtensorMap tq, td;
  if (int rc = make_tmap_tokens(&tq, q, nq, SQ, P, QROWS)) return rc;
  if (int rc = make_tmap_tokens(&td, d, B, SD, P, DCOLS)) return rc;
  MaxSimParams prm = {q_mask, d_mask, q_index, score, nq, SQ, SD, P, pool};
  maxsim_kernel<<<(unsigned)grid, THREADS, SMEM_BYTES, stream>>>(tq, td, prm);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_maxsim_expert_fwd(const void* q, const void* d, const int32_t* q_ids, const float* q_w,
                                      const int32_t* d_ids, const float* d_w, const void* q_cls, const void* d_cls,
                                      const int32_t* q_index, int nq, int SQ, int B, int SD, int P, int KQ, int KD,
                                      int Pc, int pool, float* score, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(P % 8 == 0 && P >= 8 && P <= 1024, "maxsim_expert_fwd: P=%d unsupported (multiple of 8, at most 1024)",
               P);
  DPRB_REQUIRE(SQ >= 2 && SQ <= MAX_S && SD >= 2 && SD <= MAX_S,
               "maxsim_expert_fwd: sequence lengths SQ=%d SD=%d unsupported (2 .. 512, token 0 is skipped)", SQ, SD);
  DPRB_REQUIRE(KQ >= 1 && KQ <= MAX_EXPERTS && KD >= 1 && KD <= MAX_EXPERTS,
               "maxsim_expert_fwd: KQ=%d KD=%d unsupported (1 .. 8 experts per token)", KQ, KD);
  DPRB_REQUIRE(pool == DPRB_MAXSIM_SUM || pool == DPRB_MAXSIM_MAX, "maxsim_expert_fwd: pool %d unknown", pool);
  DPRB_REQUIRE((q_cls == nullptr) == (d_cls == nullptr), "maxsim_expert_fwd: give both CLS operands or neither");
  if (q_cls != nullptr) {
    DPRB_REQUIRE(Pc % 8 == 0 && Pc >= 8 && Pc <= MAX_PC,
                 "maxsim_expert_fwd: Pc=%d unsupported (multiple of 8, at most 1024)", Pc);
    DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(q_cls) | reinterpret_cast<uintptr_t>(d_cls)) & 15) == 0,
                 "maxsim_expert_fwd: q_cls / d_cls must be 16-byte aligned");
  }
  DPRB_REQUIRE(nq >= 1 && B >= 0, "maxsim_expert_fwd: nq=%d B=%d", nq, B);
  if (B == 0) return 0;
  DPRB_REQUIRE(q != nullptr && d != nullptr && q_ids != nullptr && q_w != nullptr && d_ids != nullptr &&
                   d_w != nullptr && q_index != nullptr && score != nullptr,
               "maxsim_expert_fwd: NULL operand");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(d)) & 15) == 0,
               "maxsim_expert_fwd: q / d must be 16-byte aligned");
  DPRB_REQUIRE((long long)B < (1LL << 31), "maxsim_expert_fwd: grid too large");
  CUtensorMap tq, td;
  if (int rc = make_tmap_tokens(&tq, q, nq, SQ, P, QROWS)) return rc;
  if (int rc = make_tmap_tokens(&td, d, B, SD, P, DCOLS)) return rc;
  const MaxSimExpertParams prm = {q_ids, q_w, d_ids, d_w, static_cast<const __nv_bfloat16*>(q_cls),
                                  static_cast<const __nv_bfloat16*>(d_cls), q_index, score, nq, SQ, SD, P, KQ, KD,
                                  q_cls != nullptr ? Pc : 0, pool};
  if (KQ == 1) return launch_maxsim_expert<1>(tq, td, prm, B, stream);
  if (KQ == 2) return launch_maxsim_expert<2>(tq, td, prm, B, stream);
  if (KQ <= 4) return launch_maxsim_expert<4>(tq, td, prm, B, stream);
  return launch_maxsim_expert<8>(tq, td, prm, B, stream);
}
