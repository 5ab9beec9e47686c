// The accumulator the index searches (expert_search.cu, sparse_search.cu) share, and its per-query top-k.
//
// Accumulator: int64 [Qb, N] fixed point at 2^-32, one row per query of a block, carved from the caller's workspace
// together with the searches' work counter and zeroed before the scoring launch.  Integer addition is associative, so
// sums built from atomics are bitwise repeatable.  The block size Qb keeps it within a fixed 2 GiB budget.
//
// Selection: one CTA per query reads its acc row, score = float(acc * 2^-32), and finds the k-th largest monotone key
// by four 8-bit radix passes (warp-aggregated shared-memory histograms), then collects the rows above it and the
// lowest-row ties in row order (block scans), sorts the k (score, ~row) keys bitonically and writes the scores and the
// corpus ids of the rows.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int SEL_THREADS = 1024, SEL_WARPS = SEL_THREADS / 32;
constexpr long long ACC_BUDGET = 2LL << 30;        // bytes of int64 accumulator per query block

__device__ __forceinline__ uint32_t ord_u32(float v) {   // monotone float -> unsigned
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_u32(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}

// block-wide exclusive scan of one int per thread (SEL_THREADS threads); total in `sum`
__device__ __forceinline__ int sel_excl_scan(int v, int& sum, int* warp_tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += t;
  }
  if (lane == 31) warp_tot[warp] = x;
  __syncthreads();
  int before = 0;
  sum = 0;
  for (int w = 0; w < SEL_WARPS; ++w) {
    const int t = warp_tot[w];
    if (w < warp) before += t;
    sum += t;
  }
  __syncthreads();
  return x - v + before;
}

__device__ __forceinline__ uint32_t row_key(const unsigned long long* arow, long long i) {
  const long long a = (long long)__ldcs(arow + i);
  return ord_u32((float)((double)a * (1.0 / 4294967296.0)));
}

// one CTA per query of the block
__global__ void __launch_bounds__(SEL_THREADS)
fixed_select_kernel(const unsigned long long* acc, long long N, int k, int kpad, const long long* row_ids,
                    float* out_scores, long long* out_ids) {
  __shared__ uint32_t hist[256];
  __shared__ unsigned long long s_out[1024];
  __shared__ int warp_tot[SEL_WARPS];
  __shared__ uint32_t s_prefix, s_need, s_ngt;
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const unsigned long long* arow = acc + (long long)q * N;
  if (tid == 0) { s_prefix = 0; s_need = (uint32_t)k; s_ngt = 0; }
  uint32_t mask = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = tid; i < 256; i += SEL_THREADS) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (long long base = 0; base < N; base += SEL_THREADS) {
      const long long i = base + tid;
      int dg = -1;
      if (i < N) {
        const uint32_t key = row_key(arow, i);
        if ((key & mask) == prefix) dg = (int)((key >> shift) & 255u);
      }
      const unsigned peers = __match_any_sync(0xffffffffu, dg);
      if (dg >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[dg], (uint32_t)__popc(peers));
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t need = s_need, above = 0;
      int d = 255;
      for (; d > 0; --d) {
        if (above + hist[d] >= need) break;
        above += hist[d];
      }
      s_need = need - above;                        // rows of digit d still needed (>= 1)
      s_prefix = prefix | ((uint32_t)d << shift);
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  const uint32_t T = s_prefix, need = s_need;       // the k-th largest key, and how many rows equal to it to take
  const uint32_t ngt_total = (uint32_t)k - need;
  for (int i = tid; i < kpad; i += SEL_THREADS) s_out[i] = 0ull;
  __syncthreads();
  uint32_t eq_before = 0;
  for (long long base = 0; base < N; base += SEL_THREADS) {
    const long long i = base + tid;
    uint32_t key = 0;
    if (i < N) key = row_key(arow, i);
    const bool eq = i < N && key == T;
    const unsigned long long packed = ((unsigned long long)key << 32) | (unsigned long long)(~(uint32_t)i);
    if (i < N && key > T) s_out[atomicAdd(&s_ngt, 1u)] = packed;
    int tot;
    const int r = sel_excl_scan(eq ? 1 : 0, tot, warp_tot);
    if (eq && eq_before + (uint32_t)r < need) s_out[ngt_total + eq_before + r] = packed;
    eq_before += (uint32_t)tot;
  }
  for (int size = 2; size <= kpad; size <<= 1) {    // bitonic sort, descending
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      if (tid < kpad) {
        const int j = tid ^ stride;
        if (j > tid) {
          const bool up = (tid & size) == 0;
          const unsigned long long a = s_out[tid], b = s_out[j];
          if ((a < b) == up) { s_out[tid] = b; s_out[j] = a; }
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < k; i += SEL_THREADS) {
    const unsigned long long key = s_out[i];
    const long long row = (long long)(~(uint32_t)key);
    out_scores[(long long)q * k + i] = unord_u32((uint32_t)(key >> 32));
    out_ids[(long long)q * k + i] = row_ids != nullptr ? row_ids[row] : row;
  }
}

}  // namespace

int fixed_acc_block_queries(long long N) {
  if (N < 1) return 0;
  const long long qb = ACC_BUDGET / (8 * N);
  return (int)(qb < 1 ? 1 : (qb > (1 << 20) ? (1 << 20) : qb));
}

long long fixed_acc_workspace_bytes(long long N, int Qb) {
  if (N < 1 || Qb < 1) return 0;
  Carve c(nullptr);
  c.take((long long)Qb * N * 8);
  c.take(256);
  return c.off;
}

int fixed_acc_init(void* workspace, long long N, int Qb, FixedAcc* out, cudaStream_t stream) {
  Carve c(workspace);
  out->acc = static_cast<unsigned long long*>(c.take((long long)Qb * N * 8));
  out->counter = static_cast<int*>(c.take(256));
  DPRB_CHECK_CUDA(cudaMemsetAsync(out->acc, 0, (size_t)Qb * N * 8, stream));
  DPRB_CHECK_CUDA(cudaMemsetAsync(out->counter, 0, 4, stream));
  return 0;
}

int fixed_acc_select(const unsigned long long* acc, long long N, int Qb, int k, const long long* row_ids,
                     float* out_scores, long long* out_ids, cudaStream_t stream) {
  int kpad = 2;
  while (kpad < k) kpad <<= 1;
  fixed_select_kernel<<<Qb, SEL_THREADS, 0, stream>>>(acc, N, k, kpad, row_ids, out_scores, out_ids);
  DPRB_LAUNCH_CHECK();
  return 0;
}

}  // namespace dprb
