// Fused optimizer step over the flat fp32 parameter arena: global-norm clip + AdamW + bf16 shadow
// refresh in one pass (28 B/param read+write fp32 state, +2 B/param shadow), plus the sum-of-squares
// reduction that feeds the clip coefficient without a host round trip.
//
// Replaces torch.optim.AdamW as configured by /root/reference/dpr_scale/conf/task/optim/adamw.yaml
// (instantiated at dpr_scale/task/dpr_task.py:124) and Lightning's gradient_clip_val
// (conf/trainer/gpu_1_host.yaml:8 -> torch.nn.utils.clip_grad_norm_).  LAMB (conf/task/optim/lamb.yaml) and MADGRAD
// (conf/task/optim/madgrad.yaml) take the same clip coefficient and refresh the shadow in the same pass.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ g, long long n, float* __restrict__ out) {
  __shared__ float red[8];
  float s = 0.f;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = g4[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[(n4 << 2) + threadIdx.x]; s += v * v; }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 8) {
    s = red[threadIdx.x];
    s += __shfl_xor_sync(0xffu, s, 4); s += __shfl_xor_sync(0xffu, s, 2); s += __shfl_xor_sync(0xffu, s, 1);
    if (threadIdx.x == 0) atomicAdd(out, s);
  }
}

// grad_scale * min(1, max_norm / (||grad_scale * g|| + 1e-6)): the global-norm clip, read from the device-side sum of
// squares so no step waits on the host.
__device__ __forceinline__ float clip_gmul(float grad_scale, const float* sumsq, float max_norm) {
  float gmul = grad_scale;
  if (sumsq != nullptr && max_norm > 0.f) {
    const float total = sqrtf(*sumsq) * grad_scale;
    const float coef = max_norm / (total + 1e-6f);
    gmul *= fminf(coef, 1.f);
  }
  return gmul;
}

struct AdamArgs {
  float lr, beta1, beta2, eps, wd, bc1, bc2_rsqrt, grad_scale, max_norm;
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, const AdamArgs& a, float gmul) {
  g *= gmul;
  p *= (1.f - a.lr * a.wd);
  m = a.beta1 * m + (1.f - a.beta1) * g;
  v = a.beta2 * v + (1.f - a.beta2) * g * g;
  const float denom = sqrtf(v) * a.bc2_rsqrt + a.eps;
  p -= (a.lr / a.bc1) * (m / denom);
}

__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             bf16* __restrict__ shadow, long long n, AdamArgs a, const float* __restrict__ sumsq) {
  const float gmul = clip_gmul(a.grad_scale, sumsq, a.max_norm);
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    adam_one(pp.x, gg.x, mm.x, vv.x, a, gmul); adam_one(pp.y, gg.y, mm.y, vv.y, a, gmul);
    adam_one(pp.z, gg.z, mm.z, vv.z, a, gmul); adam_one(pp.w, gg.w, mm.w, vv.w, a, gmul);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (shadow != nullptr) {
      uint2 s2; s2.x = pack_bf16x2(pp.x, pp.y); s2.y = pack_bf16x2(pp.z, pp.w);
      reinterpret_cast<uint2*>(shadow)[i] = s2;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    float pp = p[i], mm = m[i], vv = v[i];
    adam_one(pp, g[i], mm, vv, a, gmul);
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (shadow != nullptr) shadow[i] = __float2bfloat16(pp);
  }
}

__global__ void __launch_bounds__(256)
cast_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    uint2 s2; s2.x = pack_bf16x2(v.x, v.y); s2.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(dst)[i] = s2;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    dst[i] = __float2bfloat16(src[i]);
  }
}

__global__ void __launch_bounds__(256)
uncast_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const uint2 s2 = reinterpret_cast<const uint2*>(src)[i];
    const float2 a = unpack_bf16x2(s2.x), b = unpack_bf16x2(s2.y);
    reinterpret_cast<float4*>(dst)[i] = make_float4(a.x, a.y, b.x, b.y);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    dst[i] = __bfloat162float(src[i]);
  }
}

// ---------------------------------------------------------------- LAMB (torch_optimizer.Lamb 0.3.x)
// The arena is cut into segments (one per parameter tensor) and every segment into chunks (a few thousand elements,
// chosen by the caller) that never straddle a segment.  Pass 1 updates the moments and writes per-chunk partial sums of p^2 and
// u^2; a second launch reduces each segment's partials in a fixed order into its trust ratio; pass 2 recomputes u from
// the updated moments and applies it.  Every sum has one fixed order, so the update is bitwise repeatable for any grid.
//
// Plan (int64, built once per layout by the caller): chunk_off[C+1] | chunk_seg[C] | seg_chunk[S+1].
struct LambArgs {
  float beta1, beta2, eps, wd, clamp_value, step_size, grad_scale, max_norm;
  int adam;
};

__device__ __forceinline__ float lamb_u(float p, float m, float v, const LambArgs& a) {
  return m / (sqrtf(v) + a.eps) + a.wd * p;
}

__device__ __forceinline__ float lamb_moments(float p, float g, float& m, float& v, const LambArgs& a, float gmul) {
  g *= gmul;
  m = a.beta1 * m + (1.f - a.beta1) * g;
  v = a.beta2 * v + (1.f - a.beta2) * g * g;
  return lamb_u(p, m, v, a);
}

__global__ void __launch_bounds__(256)
lamb_moments_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                    float* __restrict__ v, const long long* __restrict__ plan, int nchunks, LambArgs a,
                    const float* __restrict__ sumsq, float* __restrict__ partials) {
  __shared__ float red[2][8];
  const float gmul = clip_gmul(a.grad_scale, sumsq, a.max_norm);
  for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
    const long long lo = plan[c] >> 2, hi = plan[c + 1] >> 2;
    float pp = 0.f, uu = 0.f;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const float4 p4 = reinterpret_cast<const float4*>(p)[i];
      const float4 g4 = reinterpret_cast<const float4*>(g)[i];
      float4 m4 = reinterpret_cast<float4*>(m)[i];
      float4 v4 = reinterpret_cast<float4*>(v)[i];
      const float ux = lamb_moments(p4.x, g4.x, m4.x, v4.x, a, gmul);
      const float uy = lamb_moments(p4.y, g4.y, m4.y, v4.y, a, gmul);
      const float uz = lamb_moments(p4.z, g4.z, m4.z, v4.z, a, gmul);
      const float uw = lamb_moments(p4.w, g4.w, m4.w, v4.w, a, gmul);
      reinterpret_cast<float4*>(m)[i] = m4;
      reinterpret_cast<float4*>(v)[i] = v4;
      pp += p4.x * p4.x + p4.y * p4.y + p4.z * p4.z + p4.w * p4.w;
      uu += ux * ux + uy * uy + uz * uz + uw * uw;
    }
    pp = warp_sum(pp);
    uu = warp_sum(uu);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = pp; red[1][threadIdx.x >> 5] = uu; }
    __syncthreads();
    if (threadIdx.x < 2) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
      partials[2 * (long long)c + threadIdx.x] = s;
    }
    __syncthreads();
  }
}

// One warp per segment: trust[s] = min(||p||, clamp) / ||u|| (1 when either is 0, or in adam mode), times step_size.
__global__ void __launch_bounds__(256)
lamb_trust_kernel(const long long* __restrict__ plan, int nchunks, int nseg, const float* __restrict__ partials,
                  LambArgs a, float* __restrict__ scale) {
  const int s = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= nseg) return;
  const long long* seg_chunk = plan + 2 * (long long)nchunks + 1;
  float pp = 0.f, uu = 0.f;
  for (long long c = seg_chunk[s] + lane; c < seg_chunk[s + 1]; c += 32) {
    pp += partials[2 * c];
    uu += partials[2 * c + 1];
  }
  pp = warp_sum(pp);
  uu = warp_sum(uu);
  if (lane == 0) {
    const float w_norm = fminf(sqrtf(pp), a.clamp_value), u_norm = sqrtf(uu);
    const float trust = (w_norm == 0.f || u_norm == 0.f || a.adam) ? 1.f : w_norm / u_norm;
    scale[s] = a.step_size * trust;
  }
}

__global__ void __launch_bounds__(256)
lamb_apply_kernel(float* __restrict__ p, const float* __restrict__ m, const float* __restrict__ v,
                  bf16* __restrict__ shadow, const long long* __restrict__ plan, int nchunks, LambArgs a,
                  const float* __restrict__ scale) {
  const long long* chunk_seg = plan + nchunks + 1;
  for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
    const long long lo = plan[c] >> 2, hi = plan[c + 1] >> 2;
    const float k = scale[chunk_seg[c]];
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      float4 p4 = reinterpret_cast<float4*>(p)[i];
      const float4 m4 = reinterpret_cast<const float4*>(m)[i];
      const float4 v4 = reinterpret_cast<const float4*>(v)[i];
      p4.x -= k * lamb_u(p4.x, m4.x, v4.x, a);
      p4.y -= k * lamb_u(p4.y, m4.y, v4.y, a);
      p4.z -= k * lamb_u(p4.z, m4.z, v4.z, a);
      p4.w -= k * lamb_u(p4.w, m4.w, v4.w, a);
      reinterpret_cast<float4*>(p)[i] = p4;
      if (shadow != nullptr) {
        uint2 s2; s2.x = pack_bf16x2(p4.x, p4.y); s2.y = pack_bf16x2(p4.z, p4.w);
        reinterpret_cast<uint2*>(shadow)[i] = s2;
      }
    }
  }
}

// ---------------------------------------------------------------- MADGRAD (dpr_scale/optim/madgrad.py, dense branch)
struct MadgradArgs {
  float lamb, eps, wd, momentum, ck, grad_scale, max_norm;
};

__device__ __forceinline__ void madgrad_one(float& p, float g, float& nu, float& s, float x0, const MadgradArgs& a,
                                            float gmul) {
  g *= gmul;
  if (a.wd != 0.f) g += a.wd * p;  // coupled decay, only when set (as the reference: NaN/Inf p stays out of g)
  if (a.momentum == 0.f) x0 = p + s / (cbrtf(nu) + a.eps);  // x0 rebuilt from the state before nu moves
  nu += a.lamb * (g * g);
  s += a.lamb * g;
  const float z = x0 - s / (cbrtf(nu) + a.eps);
  p = a.momentum == 0.f ? z : a.momentum * p + a.ck * z;
}

__global__ void __launch_bounds__(256)
madgrad_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ nu, float* __restrict__ s,
               const float* __restrict__ x0, bf16* __restrict__ shadow, long long n, MadgradArgs a,
               const float* __restrict__ sumsq) {
  const float gmul = clip_gmul(a.grad_scale, sumsq, a.max_norm);
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 nn = reinterpret_cast<float4*>(nu)[i];
    float4 ss = reinterpret_cast<float4*>(s)[i];
    const float4 xx = x0 != nullptr ? reinterpret_cast<const float4*>(x0)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    madgrad_one(pp.x, gg.x, nn.x, ss.x, xx.x, a, gmul); madgrad_one(pp.y, gg.y, nn.y, ss.y, xx.y, a, gmul);
    madgrad_one(pp.z, gg.z, nn.z, ss.z, xx.z, a, gmul); madgrad_one(pp.w, gg.w, nn.w, ss.w, xx.w, a, gmul);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(nu)[i] = nn;
    reinterpret_cast<float4*>(s)[i] = ss;
    if (shadow != nullptr) {
      uint2 s2; s2.x = pack_bf16x2(pp.x, pp.y); s2.y = pack_bf16x2(pp.z, pp.w);
      reinterpret_cast<uint2*>(shadow)[i] = s2;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    float pp = p[i], nn = nu[i], ss = s[i];
    madgrad_one(pp, g[i], nn, ss, x0 != nullptr ? x0[i] : 0.f, a, gmul);
    p[i] = pp; nu[i] = nn; s[i] = ss;
    if (shadow != nullptr) shadow[i] = __float2bfloat16(pp);
  }
}

int stream_grid(long long n4, int sms) {
  long long want = (n4 + 255) / 256;
  long long cap = (long long)sms * 8;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_sumsq_f32(const float* g, int64_t n, float* out, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(n >= 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0, "sumsq: buffer must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  sumsq_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(g, n, out);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_adamw_step(float* p, const float* g, float* m, float* v, void* shadow, int64_t n, float lr,
                               float beta1, float beta2, float eps, float wd, int step, float grad_scale,
                               const float* sumsq, float max_norm, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(step >= 1, "adamw_step: step must start at 1 (got %d)", step);
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(shadow) & 7) == 0,
               "adamw_step: arenas must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  // In double, rounded once: 1 - beta2^step cancels, and fp32 powf would leave a few 1e-6 of error in every update.
  a.bc1 = (float)(1.0 - pow((double)beta1, step));
  a.bc2_rsqrt = (float)(1.0 / sqrt(1.0 - pow((double)beta2, step)));
  a.grad_scale = grad_scale; a.max_norm = max_norm;
  adamw_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(p, g, m, v, (bf16*)shadow, n, a, sumsq);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t dprb_lamb_workspace_bytes(int nchunks, int nseg) {
  if (nchunks < 1 || nseg < 1) return -1;
  return ((2LL * nchunks + nseg) * (long long)sizeof(float) + 255) & ~255LL;
}

extern "C" int dprb_lamb_step(float* p, const float* g, float* m, float* v, void* shadow, int64_t n,
                              const int64_t* plan_, int nchunks, int nseg, float lr, float beta1, float beta2,
                              float eps, float wd, float clamp_value, int adam, int debias, int step, float grad_scale,
                              const float* sumsq, float max_norm, void* workspace, int64_t workspace_bytes,
                              dprb_stream_t stream_) {
  const long long* plan = reinterpret_cast<const long long*>(plan_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(step >= 1, "lamb_step: step must start at 1 (got %d)", step);
  DPRB_REQUIRE(n >= 0 && (n & 3) == 0, "lamb_step: arena length must be a multiple of 4 (got %lld)", (long long)n);
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(shadow) & 7) == 0 && (reinterpret_cast<uintptr_t>(plan) & 7) == 0,
               "lamb_step: arenas must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_REQUIRE(plan != nullptr && nchunks >= nseg && nseg >= 1, "lamb_step: need a plan with 1 <= nseg <= nchunks "
               "(got nchunks %d, nseg %d)", nchunks, nseg);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= dprb_lamb_workspace_bytes(nchunks, nseg),
               "lamb_step: workspace of %lld bytes is smaller than dprb_lamb_workspace_bytes = %lld",
               (long long)workspace_bytes, (long long)dprb_lamb_workspace_bytes(nchunks, nseg));
  DPRB_NUM_SMS(sms);
  LambArgs a;
  a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd; a.clamp_value = clamp_value; a.adam = adam != 0;
  a.step_size = debias ? (float)((double)lr * sqrt(1.0 - pow((double)beta2, step)) / (1.0 - pow((double)beta1, step)))
                       : lr;
  a.grad_scale = grad_scale; a.max_norm = max_norm;
  float* partials = static_cast<float*>(workspace);
  float* scale = partials + 2LL * nchunks;
  const int grid = nchunks < sms * 8 ? nchunks : sms * 8;
  lamb_moments_kernel<<<grid, 256, 0, stream>>>(p, g, m, v, plan, nchunks, a, sumsq, partials);
  DPRB_LAUNCH_CHECK();
  lamb_trust_kernel<<<(nseg + 7) / 8, 256, 0, stream>>>(plan, nchunks, nseg, partials, a, scale);
  DPRB_LAUNCH_CHECK();
  lamb_apply_kernel<<<grid, 256, 0, stream>>>(p, m, v, (bf16*)shadow, plan, nchunks, a, scale);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_madgrad_step(float* p, const float* g, float* nu, float* s, const float* x0, void* shadow,
                                 int64_t n, float lr, float momentum, float wd, float eps, int k, float grad_scale,
                                 const float* sumsq, float max_norm, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(k >= 0, "madgrad_step: k counts steps from 0 (got %d)", k);
  DPRB_REQUIRE(momentum >= 0.f && momentum < 1.f, "madgrad_step: momentum must be in [0, 1) (got %g)", momentum);
  DPRB_REQUIRE((momentum == 0.f) == (x0 == nullptr), "madgrad_step: x0 is required exactly when momentum != 0");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(nu) |
                 reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(x0)) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(shadow) & 7) == 0,
               "madgrad_step: arenas must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  MadgradArgs a;
  const double lr_eff = (double)lr + (double)eps;  // the reference adds eps to the group lr
  a.lamb = (float)(lr_eff * sqrt((double)k + 1.0));
  a.eps = eps; a.wd = wd; a.momentum = momentum;
  a.ck = (float)(1.0 - (double)momentum);
  a.grad_scale = grad_scale; a.max_norm = max_norm;
  madgrad_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(p, g, nu, s, x0, (bf16*)shadow, n, a, sumsq);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_cast_f32_bf16(const float* src, void* dst, int64_t n, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "cast_f32_bf16: buffers must be 16/8-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  cast_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(src, (bf16*)dst, n);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_cast_bf16_f32(const void* src, float* dst, int64_t n, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(dst) & 15) == 0 && (reinterpret_cast<uintptr_t>(src) & 7) == 0,
               "cast_bf16_f32: buffers must be 8/16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  uncast_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>((const bf16*)src, dst, n);
  DPRB_LAUNCH_CHECK();
  return 0;
}
