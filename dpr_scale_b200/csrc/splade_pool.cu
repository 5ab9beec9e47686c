// SPLADE vocabulary max-pool on the tensor cores, forward only:
//
//   out[n, v] = log1p( max(0, max_{r in [off[n], off[n+1])} ( x[r, :K] . W[v, :K] + bias[v] ) ) )    (0: empty range)
//
// Replaces SPLADEEncoder.forward's pooling of the reference (dpr_scale/models/citadel_models/splade_model.py):
//     logits = masked-LM decoder over every token                       # [N, S, V], materialised
//     max over tokens 1.. of log(1 + relu(logits)) * attention_mask     # several passes over [N, S, V]
// Every valid token contributes log(1 + relu(l)) >= 0 and every masked token exactly 0, so the masked max is
// log1p(relu(max over the valid tokens)), or 0 for a sequence without one.  The caller compacts the valid tokens (token
// 0 and masked tokens dropped) into contiguous rows per sequence, so the decoder never computes padding.
//
// Design: a persistent 1-D grid walks 128-row x 256-column tiles of the [rows, V] logit matrix (grouped by 16 row tiles,
// so a wave shares its decoder tiles through L2).  Warpgroup 0 is the TMA producer (one thread, K-major 128B-swizzled
// fp16 tiles of x and W into a 4-stage mbarrier ring); warpgroups 1 and 2 each run wgmma m64n256k16 over 64 rows with
// fp32 accumulators.  The logits never leave registers: the epilogue reduces each column over the rows of the same
// sequence (a segmented max scan over the quad rows of each warp; segments are contiguous because off is sorted), adds
// the fp32 bias and the relu to each segment's maximum (rounding is monotone, so max_r fl(a_r + b) = fl(max_r a_r + b)),
// and folds the positive ones into `out` with an integer atomicMax on their fp32 bit patterns.  Non-negative floats
// order like their bit patterns, so the result does not depend on the order of the atomics, nor on how the sequences
// are grouped into tiles: out is bitwise repeatable.  A first kernel zeroes out[N, V], a last one applies log1p.
// Non-finite logits are out of contract.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int BLOCK_M = 128, BLOCK_N = 256, BK = 64;   // 64 fp16 = one 128-byte swizzle row
constexpr int STAGES = 4;
constexpr int A_BYTES = BLOCK_M * BK * 2;               // 16 KB
constexpr int B_BYTES = BLOCK_N * BK * 2;               // 32 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NUM_CONSUMERS = 2;
constexpr int THREADS = (NUM_CONSUMERS + 1) * 128;      // warpgroup 0: producer; 1, 2: wgmma + epilogue
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 2 * STAGES * 8;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int GROUP_M = 16;                             // row tiles per group of the tile order
constexpr int MAX_K = 1024;

struct PoolParams {
  const float* bias;     // [V] or NULL
  const int32_t* off;    // [N + 1]
  float* out;            // [N, ldo]
  long long ldo;
  int N, V, K;
  int m_tiles, n_tiles, units;
};

// unit u -> (row tile, column tile): groups of GROUP_M row tiles, column-major inside a group
__device__ __forceinline__ void unit_tile(const PoolParams& p, int u, int& mt, int& nt) {
  const int per_group = GROUP_M * p.n_tiles;
  const int g = u / per_group, local = u - g * per_group;
  const int rows = min(GROUP_M, p.m_tiles - g * GROUP_M);
  mt = g * GROUP_M + local % rows;
  nt = local / rows;
}

// the sequence of row r: the largest n with off[n] <= r (off[0] <= r < off[N])
__device__ __forceinline__ int seq_of(const int32_t* off, int N, int r) {
  int lo = 0, hi = N;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= r) lo = mid;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(THREADS, 1)
splade_pool_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                   const PoolParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // rows [r_begin, r_end) hold the sequences; row tiles start at r_begin, so rows before it are never loaded
  const int r_begin = __ldg(p.off), r_end = __ldg(p.off + p.N);
  const int n_k = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMERS * 4);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================ TMA producer ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        int mt, nt;
        unit_tile(p, u, mt, nt);
        const int r0 = r_begin + mt * BLOCK_M;
        if (r0 >= r_end) continue;
        for (int kb = 0; kb < n_k; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          tma_load_2d(sa, &tm_x, &full_bar[stage], kb * BK, r0);
          tma_load_2d(sa + A_BYTES, &tm_w, &full_bar[stage], kb * BK, nt * BLOCK_N);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = (warp >> 2) - 1;
  const int q = lane & 3, i8 = lane >> 2;             // quad column pair, row inside the 8-row group
  const int lr = (warp & 3) * 16 + i8;                // the thread's rows lr and lr + 8 of the warpgroup's 64

  float acc[128];
  int stage = 0;
  uint32_t phase = 0;
  for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
    int mt, nt;
    unit_tile(p, u, mt, nt);
    const int r0 = r_begin + mt * BLOCK_M;
    if (r0 >= r_end) continue;
    {
      int prev = -1;
      for (int kb = 0; kb < n_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + (uint32_t)wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
        const uint64_t da = make_wgmma_desc_sw128(sa, 16, 1024);
        const uint64_t db = make_wgmma_desc_sw128(sb, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_m64n256_ss_f16<0, 0>(acc, da + 2 * k, db + 2 * k, (kb > 0 || k > 0) ? 1 : 0);
        wgmma_commit();
        // keep one k-block of MMAs in flight; the one before it has retired and its stage can be refilled
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }

    // ================================ epilogue ================================
    // sequence of each of the thread's two rows (-1: beyond r_end, never part of a maximum)
    const int ra = r0 + wg * 64 + lr;
    int seg[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = ra + 8 * h;
      seg[h] = r < r_end ? seq_of(p.off, p.N, r) : -1;
    }
    // segmented inclusive max scan over the 8 rows of each half (rows are lanes 4 apart): at step s a row takes the
    // row 2^s above it when both belong to the same sequence
    bool take[2][3];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int src = __shfl_up_sync(0xffffffffu, seg[h], 4 << s);
        take[h][s] = i8 >= (1 << s) && src == seg[h];
      }
    // the first half's last row (i8 = 7) sits right above the second half's first row (i8 = 0)
    const int seg7 = __shfl_sync(0xffffffffu, seg[0], 28 + q);
    const bool carry = seg[1] == seg7;
    const int next0 = __shfl_down_sync(0xffffffffu, seg[0], 4);
    const int first1 = __shfl_sync(0xffffffffu, seg[1], q);
    const int next1 = __shfl_down_sync(0xffffffffu, seg[1], 4);
    const bool tail0 = seg[0] >= 0 && (i8 < 7 ? next0 != seg[0] : first1 != seg[0]);
    const bool tail1 = seg[1] >= 0 && (i8 == 7 || next1 != seg[1]);
#pragma unroll
    for (int j = 0; j < 64; ++j) {                    // acc[4c + e] row lr, acc[4c + 2 + e] row lr + 8
      const int c = j >> 1, e = j & 1;
      float v0 = seg[0] >= 0 ? acc[4 * c + e] : -INFINITY;
      float v1 = seg[1] >= 0 ? acc[4 * c + 2 + e] : -INFINITY;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float t0 = __shfl_up_sync(0xffffffffu, v0, 4 << s);
        const float t1 = __shfl_up_sync(0xffffffffu, v1, 4 << s);
        if (take[0][s]) v0 = fmaxf(v0, t0);
        if (take[1][s]) v1 = fmaxf(v1, t1);
      }
      const float t7 = __shfl_sync(0xffffffffu, v0, 28 + q);
      if (carry) v1 = fmaxf(v1, t7);
      acc[4 * c + e] = v0;
      acc[4 * c + 2 + e] = v1;
    }
    if (tail0 || tail1) {
      const int col0 = nt * BLOCK_N + 2 * q;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!(h == 0 ? tail0 : tail1)) continue;
        unsigned int* orow = reinterpret_cast<unsigned int*>(p.out + (long long)seg[h] * p.ldo);
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          const int c = j >> 1, e = j & 1;
          const int col = col0 + 8 * c + e;
          if (col >= p.V) continue;
          float v = acc[4 * c + 2 * h + e];
          if (p.bias != nullptr) v += __ldg(p.bias + col);
          if (v > 0.f) atomicMax(orow + col, __float_as_uint(v));     // fp32 bit order = value order for v > 0
        }
      }
    }
  }
}

__global__ void zero_rows_kernel(float* out, long long ldo, int N, int V) {
  const long long total = (long long)N * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / V;
    out[n * ldo + (i - n * V)] = 0.f;
  }
}

__global__ void log1p_rows_kernel(float* out, long long ldo, int N, int V) {
  const long long total = (long long)N * V;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / V;
    float* o = out + n * ldo + (i - n * V);
    *o = log1pf(*o);
  }
}

// fp16 [rows][ld], the first K columns; box = [64 of K][box_rows]; everything beyond K or the rows reads as zero
int make_tmap_rows(CUtensorMap* out, const void* base, long long rows, int K, long long ld, int box_rows) {
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  return encode_tmap(out, "splade_pool", CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_splade_pool_fwd(const void* x, int64_t ldx, const void* W, int64_t ldw, const float* bias,
                                    const int32_t* off, int64_t T, int N, int V, int K, float* out, int64_t ldo,
                                    dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(K % 8 == 0 && K >= 8 && K <= MAX_K, "splade_pool_fwd: K=%d unsupported (multiple of 8, 8 .. 1024)", K);
  DPRB_REQUIRE(ldx >= K && ldx % 8 == 0 && ldw >= K && ldw % 8 == 0,
               "splade_pool_fwd: ldx=%lld ldw=%lld must be multiples of 8 and at least K=%d", (long long)ldx,
               (long long)ldw, K);
  DPRB_REQUIRE(V >= 1 && N >= 1, "splade_pool_fwd: V=%d N=%d (both at least 1)", V, N);
  DPRB_REQUIRE(ldo >= V, "splade_pool_fwd: ldo=%lld < V=%d", (long long)ldo, V);
  DPRB_REQUIRE(T >= 0 && T < 0x7FFFFF00LL, "splade_pool_fwd: T=%lld rows outside [0, 2^31) (32-bit row indices)",
               (long long)T);
  DPRB_REQUIRE(off != nullptr && out != nullptr && (T == 0 || (x != nullptr && W != nullptr)),
               "splade_pool_fwd: NULL operand");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
               "splade_pool_fwd: x / W must be 16-byte aligned");
  const long long m_tiles = (T + BLOCK_M - 1) / BLOCK_M, n_tiles = (V + BLOCK_N - 1) / BLOCK_N;
  DPRB_REQUIRE(m_tiles * n_tiles < (1LL << 31), "splade_pool_fwd: %lld x %lld tiles exceed 2^31", m_tiles, n_tiles);
  DPRB_NUM_SMS(sms);
  static bool attr_done = false;
  if (!attr_done) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(splade_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_done = true;
  }
  CUtensorMap tx, tw;
  if (T > 0) {
    if (int rc = make_tmap_rows(&tx, x, T, K, ldx, BLOCK_M)) return rc;
    if (int rc = make_tmap_rows(&tw, W, V, K, ldw, BLOCK_N)) return rc;
  }
  const long long elems = (long long)N * V;
  const int ew_blocks = (int)(elems < (long long)sms * 8 * 256 ? (elems + 255) / 256 : (long long)sms * 8);
  zero_rows_kernel<<<ew_blocks, 256, 0, stream>>>(out, ldo, N, V);
  DPRB_LAUNCH_CHECK();
  if (T > 0) {
    PoolParams prm = {bias, off, out, ldo, N, V, K, (int)m_tiles, (int)n_tiles, (int)(m_tiles * n_tiles)};
    const int grid = (int)(prm.units < sms ? prm.units : sms);
    splade_pool_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(tx, tw, prm);
    DPRB_LAUNCH_CHECK();
  }
  log1p_rows_kernel<<<ew_blocks, 256, 0, stream>>>(out, ldo, N, V);
  DPRB_LAUNCH_CHECK();
  return 0;
}
