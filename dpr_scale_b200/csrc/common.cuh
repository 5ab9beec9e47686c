// dprb — H100 (sm_90a) kernels for the dpr-scale bi-encoder training path.
// Shared device helpers: PTX wrappers for mbarrier / TMA / wgmma, small math,
// warp reductions, error plumbing.  Everything here targets sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "wgmma.cuh"

#ifndef DPRB_HANG_GUARD
#define DPRB_HANG_GUARD 1
#endif

namespace dprb {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------- host-side error plumbing
// printf-checked: the entry points format their int64_t parameters with %lld, which needs a (long long) cast
void set_last_error(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
#define DPRB_CHECK_CUDA(expr)                                                        \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      dprb::set_last_error("%s:%d CUDA error %d (%s) in `%s`", __FILE__, __LINE__,   \
                           (int)_e, cudaGetErrorString(_e), #expr);                  \
      return 2;                                                                      \
    }                                                                                \
  } while (0)
#define DPRB_REQUIRE(cond, ...)                                                      \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      dprb::set_last_error(__VA_ARGS__);                                             \
      return 1;                                                                      \
    }                                                                                \
  } while (0)

int num_sms();  // cached SM count of the current device; -1 (with the message set) when the query fails
// Declares `const int var` = num_sms(); a failed query makes the calling entry point return 2.  Two statements: use it
// only as a statement of its own at block scope (never as the body of an unbraced if / for).
#define DPRB_NUM_SMS(var)           \
  const int var = dprb::num_sms();  \
  if (var <= 0) return 2

// Every kernel launch of the library goes through this (one call per <<<>>> / cudaLaunchKernelEx): the running total is
// exported as dprb_launch_count() so callers can report a MEASURED launch count instead of an estimate.
void count_launch();
#define DPRB_LAUNCH_CHECK()                \
  do {                                     \
    dprb::count_launch();                  \
    DPRB_CHECK_CUDA(cudaGetLastError());   \
  } while (0)

// ---------------------------------------------------------------- small device helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// SWIZZLE_128B tiles (TMA and wgmma) must start 1024-byte aligned
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}

// fp16 twins: the encoder keeps its RESIDUAL STREAM (LayerNorm inputs and outputs) in fp16 - 11 significand bits
// instead of bf16's 8 at the same 2 bytes - because those tensors are re-read by every residual add and their rounding
// error accumulates over 2L LayerNorms (measured at BERT-base: embedding rel-L2 1.1e-2 with a bf16 stream, 5.2e-3 with
// fp16; the reference's own bf16 autocast: 6.5e-3).  They are O(1..100) by construction, far from fp16's range limits.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 t = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t u) {
  __half2 t = *reinterpret_cast<__half2*>(&u);
  return __half22float2(t);
}
__device__ __forceinline__ uint32_t pack_16x2(float lo, float hi, bool f16) { return f16 ? pack_f16x2(lo, hi) : pack_bf16x2(lo, hi); }
__device__ __forceinline__ float2 unpack_16x2(uint32_t u, bool f16) { return f16 ? unpack_f16x2(u) : unpack_bf16x2(u); }

// Element pairs in fp32 with explicit rounding (no contraction), so every pair operation rounds exactly once.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// erf-GELU (HF "gelu", modeling_bert.py BertIntermediate) through a fitted Gaussian CDF:
// Phi(x) = sigma(z(x)), z = a0 x + a1 x^3 + a2 x^5 (least-squares fit on [-6,6], argument clamped to [-8,8]):
// max |Phi err| 5.8e-5, max |x*Phi - gelu_erf(x)| 3.0e-5 over all x, max |derivative err| 1.2e-4 — two orders of
// magnitude below the bf16 rounding of the stored activation.  The libm-style erf (~24 instructions + IEEE rcp / exp
// fix-ups) made the FFN-in GEMM epilogue 2.3x slower than the tensor-core work it follows: at K = 768 there are only
// ~24 issue slots per output element.
// single-MUFU approximations (ex2.approx / rcp.approx: ~2 ulp), no denormal / range fix-up code
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// GELU and its derivative from ONE evaluation of sigma(z(x)) (2 MUFU for both): the forward GEMM epilogue stores
// gelu'(pre) instead of the pre-activation, so the backward epilogue is a plain multiply.
__device__ __forceinline__ void gelu_and_grad(float x, float& g, float& gd) {
  const float xc = fminf(fmaxf(x, -8.f), 8.f);
  const float x2 = xc * xc;
  float pz = fmaf(x2, 1.03455483e-3f, -1.06900513e-1f);
  pz = fmaf(pz, x2, -2.30098511f);
  const float e = ex2_approx(pz * xc);          // exp(-z)
  const float sg = rcp_approx(1.f + e);         // sigma(z) ~ Phi(x)
  float zp = fmaf(x2, -3.58549371e-3f, 2.22293380e-1f);   // z'(x) = a0 + 3 a1 x^2 + 5 a2 x^4
  zp = fmaf(zp, x2, 1.59492135f);
  const float inside = (x == xc) ? zp : 0.f;    // clamp region: z is constant
  g = x * sg;
  gd = sg * fmaf(xc * e * sg, inside, 1.f);
}
// The same function on PAIRS of elements (the form every epilogue uses).  Changes against the scalar form, all exact
// in effect: the argument clamp becomes one min on x^2 (the fit's odd polynomial must not be
// evaluated beyond |x| = 8, where its x^5 term would turn it around); 1 - sigma replaces e * sigma (same quantity,
// no inf * 0 when e overflows), which also removes the select that zeroed the derivative term in the clamped region.
__device__ __forceinline__ void gelu_and_grad2(float2 x, float2& g, float2& gd) {
  float2 x2 = fmul2(x, x);
  x2.x = fminf(x2.x, 64.f);
  x2.y = fminf(x2.y, 64.f);
  const float2 one = make_float2(1.f, 1.f);
  float2 pz = ffma2(x2, make_float2(1.03455483e-3f, 1.03455483e-3f), make_float2(-1.06900513e-1f, -1.06900513e-1f));
  pz = ffma2(pz, x2, make_float2(-2.30098511f, -2.30098511f));
  const float2 ex = fmul2(pz, x);
  const float2 e = make_float2(ex2_approx(ex.x), ex2_approx(ex.y));        // exp(-z)
  const float2 den = fadd2(e, one);
  const float2 sg = make_float2(rcp_approx(den.x), rcp_approx(den.y));     // sigma(z) ~ Phi(x)
  float2 zp = ffma2(x2, make_float2(-3.58549371e-3f, -3.58549371e-3f), make_float2(2.22293380e-1f, 2.22293380e-1f));
  zp = ffma2(zp, x2, make_float2(1.59492135f, 1.59492135f));          // z'(x)
  g = fmul2(x, sg);
  const float2 t = ffma2(sg, make_float2(-1.f, -1.f), one);           // 1 - sigma
  const float2 w = ffma2(fmul2(x, t), zp, one);
  gd = fmul2(sg, w);
}
// Counter-based dropout RNG.  One 32-bit hash (lowbias32 finaliser, 9 integer instructions) decides TWO horizontally
// adjacent elements (16 bits each), keyed by (row, column group of 8, pair in the group, site seed): element (r, c) is kept iff its 16-bit lane
// is >= thresh16 = round(p * 65536); kept values are scaled by 1 / (1 - thresh16/65536) (p = 0.1 -> 0.100006).
// thresh16 == 0 disables the site (p = 0 / eval mode).  Masks are never stored: backward re-derives them.
struct Drop {
  uint32_t seed;
  uint32_t thresh16;
  float scale;
  uint32_t row_mul;  // row key = r * row_mul (the pruned last layer runs on the CLS rows only: key = row * S)
  __host__ __device__ bool on() const { return thresh16 != 0u; }
  // One hash chain per GROUP OF 8 columns: a shared first round keyed by (row, column / 8, site seed), then one cheap
  // finaliser per column pair (four odd multipliers).  A quarter of the mixing work of a full hash per pair - the
  // dropout epilogues, the LayerNorm backward and the attention passes are all bound by instruction issue.
  __device__ __forceinline__ uint32_t group_mix(uint32_t r, uint32_t c8) const {   // c8 = column / 8
    uint32_t x = (r * row_mul) * 0x9E3779B1u + c8 * 0x85EBCA6Bu + seed;
    x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15;
    return x;
  }
  __device__ __forceinline__ static uint32_t pair_word(uint32_t x, uint32_t w) {  // w = pair index 0..3 in the group
    const uint32_t k = w == 0u ? 0x846CA68Bu : (w == 1u ? 0xC2B2AE35u : (w == 2u ? 0x27D4EB2Fu : 0x165667B1u));
    uint32_t h = x * k;
    h ^= h >> 16;
    return h;
  }
  __device__ __forceinline__ uint32_t pair_hash(uint32_t r, uint32_t c_even) const {
    return pair_word(group_mix(r, c_even >> 3), (c_even >> 1) & 3u);
  }
  __device__ __forceinline__ void lanes(uint32_t h, float& m0, float& m1) const {
    m0 = (h & 0xFFFFu) >= thresh16 ? scale : 0.f;
    m1 = (h >> 16) >= thresh16 ? scale : 0.f;
  }
  // multipliers (scale or 0) for elements (r, c_even) and (r, c_even + 1); c_even must be even
  __device__ __forceinline__ void mul2(uint32_t r, uint32_t c_even, float& m0, float& m1) const {
    lanes(pair_hash(r, c_even), m0, m1);
  }
  // the same multipliers for the 8 columns c0 .. c0+7 (c0 a multiple of 8) as four pairs: one group_mix for all
  __device__ __forceinline__ void mul8(uint32_t r, uint32_t c0, float2 (&m)[4]) const {
    const uint32_t x = group_mix(r, c0 >> 3);
#pragma unroll
    for (int w = 0; w < 4; ++w) lanes(pair_word(x, (uint32_t)w), m[w].x, m[w].y);
  }
};
// keep multiplier of element (r, c) for a single column c (the pair hash covers columns c & ~1 and c | 1)
__device__ __forceinline__ float drop_one(const Drop& d, uint32_t r, uint32_t c) {
  float m0, m1;
  d.mul2(r, c & ~1u, m0, m1);
  return (c & 1u) ? m1 : m0;
}
inline Drop make_drop(float p, uint64_t seed, int layer, int site) {
  const uint64_t s64 = seed + (uint64_t)(layer * 8 + site + 1) * 0x9E3779B97F4A7C15ull;
  Drop d;
  d.seed = (uint32_t)(s64 ^ (s64 >> 32));
  d.thresh16 = (p > 0.f) ? (uint32_t)((double)p * 65536.0 + 0.5) : 0u;
  if (d.thresh16 > 65535u) d.thresh16 = 65535u;
  d.scale = d.thresh16 ? 1.f / (1.f - (float)d.thresh16 / 65536.f) : 1.f;
  d.row_mul = 1u;
  return d;
}
// derived 32-bit site seed handed across the C ABI (uint64 for headroom)
inline uint64_t drop_site_seed64(uint64_t seed, int layer, int site) { return make_drop(0.5f, seed, layer, site).seed; }
// site_seed: low 32 bits = derived seed, high 32 bits = row-key multiplier (0 means 1)
inline Drop drop_from_site(float p, uint64_t site_seed) {
  Drop d = make_drop(p, 0, 0, 0);
  d.seed = (uint32_t)site_seed;
  d.row_mul = (uint32_t)(site_seed >> 32) ? (uint32_t)(site_seed >> 32) : 1u;
  return d;
}
enum { DROP_SITE_EMBED = 0, DROP_SITE_ATTN = 1, DROP_SITE_ATTN_OUT = 2, DROP_SITE_FFN_OUT = 3,
       // cross-encoder classification head, layer 0: after tanh (dprb_seqcls_group_ce) and, for RoBERTa, on the CLS
       // rows before the head's dense layer (applied by the caller from dprb_dropout_mask)
       DROP_SITE_HEAD = 4, DROP_SITE_HEAD_IN = 5 };

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t tx_bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(tx_bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (-> CUDA error surfaced to the caller) instead of
// hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if DPRB_HANG_GUARD
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
#else
  while (!mbar_try_wait(bar, parity)) {}
#endif
}

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates are (c0 = innermost/contiguous, c1 = row).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// 3-D tiled load / store (coordinates innermost first)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// 2-D tiled store smem -> global (bulk async-group completion); out-of-bounds parts of the box are clipped.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all prior bulk stores of this thread have finished reading their shared-memory source
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- cp.async (LDGSTS)
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// 16-byte copy that zero-fills when `valid` is false (src-size 0)
__device__ __forceinline__ void cp_async_16_zfill(void* smem_dst, const void* gmem_src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_8(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---------------------------------------------------------------- vector global access
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}  // namespace dprb
