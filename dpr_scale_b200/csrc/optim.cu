// Fused optimizer step over the flat fp32 parameter arena: global-norm clip + AdamW + bf16 shadow
// refresh in one pass (28 B/param read+write fp32 state, +2 B/param shadow), plus the sum-of-squares
// reduction that feeds the clip coefficient without a host round trip.
//
// Replaces torch.optim.AdamW as configured by /root/reference/dpr_scale/conf/task/optim/adamw.yaml
// (instantiated at dpr_scale/task/dpr_task.py:124) and Lightning's gradient_clip_val
// (conf/trainer/gpu_1_host.yaml:8 -> torch.nn.utils.clip_grad_norm_).
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
  float gmul = a.grad_scale;
  if (sumsq != nullptr && a.max_norm > 0.f) {
    const float total = sqrtf(*sumsq) * a.grad_scale;
    const float coef = a.max_norm / (total + 1e-6f);
    gmul *= fminf(coef, 1.f);
  }
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

int stream_grid(long long n4, int sms) {
  long long want = (n4 + 255) / 256;
  long long cap = (long long)sms * 8;
  if (want < 1) want = 1;
  return (int)(want < cap ? want : cap);
}

}  // namespace

int sumsq_f32(const float* g, long long n, float* out, cudaStream_t stream) {
  DPRB_REQUIRE(n >= 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0, "sumsq: buffer must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  sumsq_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(g, n, out);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int adamw_step(float* p, const float* g, float* m, float* v, void* shadow, long long n, float lr, float beta1,
               float beta2, float eps, float wd, int step, float grad_scale, const float* sumsq, float max_norm,
               cudaStream_t stream) {
  DPRB_REQUIRE(step >= 1, "adamw_step: step must start at 1 (got %d)", step);
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                 reinterpret_cast<uintptr_t>(v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(shadow) & 7) == 0,
               "adamw_step: arenas must be 16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  a.bc1 = 1.f - powf(beta1, (float)step);
  a.bc2_rsqrt = 1.f / sqrtf(1.f - powf(beta2, (float)step));
  a.grad_scale = grad_scale; a.max_norm = max_norm;
  adamw_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(p, g, m, v, (bf16*)shadow, n, a, sumsq);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t stream) {
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "cast_f32_bf16: buffers must be 16/8-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  cast_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>(src, (bf16*)dst, n);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t stream) {
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(dst) & 15) == 0 && (reinterpret_cast<uintptr_t>(src) & 7) == 0,
               "cast_bf16_f32: buffers must be 8/16-byte aligned");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  uncast_kernel<<<stream_grid(n >> 2, sms), 256, 0, stream>>>((const bf16*)src, dst, n);
  DPRB_LAUNCH_CHECK();
  return 0;
}

}  // namespace dprb
