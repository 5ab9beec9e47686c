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

// bf16 [n][S][P], box = [64 of P][rows][1]; everything beyond P or S reads as zero
int make_tmap_tokens(CUtensorMap* out, const void* base, long long n, int S, int P, int rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)P, (cuuint64_t)S, (cuuint64_t)n};
  const cuuint64_t strides[2] = {(cuuint64_t)P * 2, (cuuint64_t)S * P * 2};
  const cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)rows, 1u};
  return encode_tmap(out, "maxsim", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

}  // namespace

int maxsim_fwd(const void* q, const void* d, const int32_t* q_mask, const int32_t* d_mask, const int32_t* q_index,
               int nq, int SQ, int B, int SD, int P, int pool, float* score, cudaStream_t stream) {
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

}  // namespace dprb
