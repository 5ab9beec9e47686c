// Squared-error sum and its gradient in one pass, for query-encoder distillation:
//
//   loss_sum[0] = sum_{r, c} (x[r, c] - t[r, c])^2          dx[r, c] = 2 (x[r, c] - t[r, c])   (when dx is given)
//
// Replaces the reference's MSELoss(reduction="sum") and the autograd backward through it in DPRDistillTask
// (dpr_scale/task/dpr_distill_task.py:43, :167, :186).  The fp32 difference is formed once; dx = 2 * diff is exact,
// so dx equals torch's fp32 2 * (x - t) bit for bit.  Each diff^2 is rounded to fp32 and summed in double.
//
// Design: a fixed grid of at most MAX_BLOCKS blocks of 8 warps; warp w of the grid walks rows w, w + warps, ... and its
// lanes stride the columns (16-byte vectors when every operand allows them, scalars otherwise).  Each block reduces its
// threads' double sums in a fixed tree and writes one partial to the workspace; a one-block final pass adds the
// partials in a fixed order and rounds once to fp32.  The grid depends only on rows, there are no atomics, so the loss
// is bitwise repeatable on any device.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_BLOCKS = 1024;

int sqerr_blocks(int rows) {
  const int b = (rows + WARPS - 1) / WARPS;
  return b < MAX_BLOCKS ? b : MAX_BLOCKS;
}

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (warp == 0) {
    s = lane < WARPS ? red[lane] : 0.0;
#pragma unroll
    for (int o = WARPS / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  return s;   // valid in thread 0
}

template <bool VEC>
__global__ void __launch_bounds__(THREADS)
sqerr_partial_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ t, long long ldt, int rows,
                     int d, float* __restrict__ dx, long long lddx, double* __restrict__ partial) {
  __shared__ double red[WARPS];
  const int lane = threadIdx.x & 31;
  const int gwarp = blockIdx.x * WARPS + (threadIdx.x >> 5), nwarps = gridDim.x * WARPS;
  double acc = 0.0;
  for (int r = gwarp; r < rows; r += nwarps) {
    const float* xr = x + (long long)r * ldx;
    const float* tr = t + (long long)r * ldt;
    float* dr = dx != nullptr ? dx + (long long)r * lddx : nullptr;
    if (VEC) {
      const int n4 = d >> 2;
#pragma unroll 4
      for (int c = lane; c < n4; c += 32) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(xr) + c);
        const float4 b = __ldg(reinterpret_cast<const float4*>(tr) + c);
        const float4 e = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
        acc += (double)(e.x * e.x) + (double)(e.y * e.y) + (double)(e.z * e.z) + (double)(e.w * e.w);
        if (dr != nullptr)
          reinterpret_cast<float4*>(dr)[c] = make_float4(2.f * e.x, 2.f * e.y, 2.f * e.z, 2.f * e.w);
      }
    } else {
#pragma unroll 4
      for (int c = lane; c < d; c += 32) {
        const float e = __ldg(xr + c) - __ldg(tr + c);
        acc += (double)(e * e);
        if (dr != nullptr) dr[c] = 2.f * e;
      }
    }
  }
  const double s = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(THREADS)
sqerr_final_kernel(const double* __restrict__ partial, int n, float* __restrict__ loss_sum) {
  __shared__ double red[WARPS];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += THREADS) acc += partial[i];
  const double s = block_sum(acc, red);
  if (threadIdx.x == 0) loss_sum[0] = (float)s;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

// The workspace holds one double per block, and the grid depends on rows alone: d does not size it.
extern "C" int64_t dprb_sqerr_workspace_bytes(int rows, int d) {
  (void)d;
  return rows > 0 ? (long long)sqerr_blocks(rows) * (long long)sizeof(double) : 0;
}

extern "C" int dprb_sqerr_fwd(const float* x, int64_t ldx, const float* t, int64_t ldt, int rows, int d, float* loss_sum,
                              float* dx, int64_t lddx, void* workspace, int64_t workspace_bytes, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(rows >= 0 && d >= 1, "sqerr_fwd: rows=%d d=%d (rows >= 0, d >= 1)", rows, d);
  DPRB_REQUIRE(ldx >= d && ldt >= d && (dx == nullptr || lddx >= d),
               "sqerr_fwd: ldx=%lld ldt=%lld lddx=%lld must be at least d=%d", (long long)ldx, (long long)ldt,
               (long long)lddx, d);
  DPRB_REQUIRE(loss_sum != nullptr && (rows == 0 || (x != nullptr && t != nullptr)), "sqerr_fwd: NULL operand");
  const long long need = dprb_sqerr_workspace_bytes(rows, d);
  DPRB_REQUIRE(workspace_bytes >= need && (need == 0 || workspace != nullptr),
               "sqerr_fwd: workspace of %lld bytes, %lld needed", (long long)workspace_bytes, need);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "sqerr_fwd: workspace must be 8-byte aligned");
  double* partial = reinterpret_cast<double*>(workspace);
  const int blocks = rows > 0 ? sqerr_blocks(rows) : 0;
  if (blocks > 0) {
    const uintptr_t addr = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(t) |
                           reinterpret_cast<uintptr_t>(dx);
    const bool vec = d % 4 == 0 && ldx % 4 == 0 && ldt % 4 == 0 && (dx == nullptr || lddx % 4 == 0) && (addr & 15) == 0;
    if (vec)
      sqerr_partial_kernel<true><<<blocks, THREADS, 0, stream>>>(x, ldx, t, ldt, rows, d, dx, lddx, partial);
    else
      sqerr_partial_kernel<false><<<blocks, THREADS, 0, stream>>>(x, ldx, t, ldt, rows, d, dx, lddx, partial);
    DPRB_LAUNCH_CHECK();
  }
  sqerr_final_kernel<<<1, THREADS, 0, stream>>>(partial, blocks, loss_sum);
  DPRB_LAUNCH_CHECK();
  return 0;
}
