// HBM-bound fused kernels of the encoder: embedding-gather + LayerNorm, LayerNorm fwd/bwd (with the
// CLS-pooling store / CLS-only upstream gradient fused in), bias-gradient column sums.
// One warp per token row, 128-bit loads, warp-shuffle reductions, fp32 statistics.
//
// Replaces (reference path, via dpr_scale/models/hf_model.py:38):
//   BertEmbeddings.forward            site-packages/transformers/models/bert/modeling_bert.py:72-112
//   BertSelfOutput/BertOutput LN      modeling_bert.py:294-298, :352-356
//   CLS pooling + clone               dpr_scale/models/hf_model.py:39-41
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int WARPS = 8;
constexpr int THREADS = WARPS * 32;
constexpr int PF_DEPTH = 4;  // rows of dy / z in flight per warp in the LayerNorm backward


__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {
  uint4 q = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(q.x), b = unpack_bf16x2(q.y), c = unpack_bf16x2(q.z), d = unpack_bf16x2(q.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void unpack8(const uint4& q, float (&v)[8]) {
  float2 a = unpack_bf16x2(q.x), b = unpack_bf16x2(q.y), c = unpack_bf16x2(q.z), d = unpack_bf16x2(q.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
// 16-bit rows whose format is a runtime choice (bf16, or fp16 for the encoder's residual stream)
__device__ __forceinline__ void unpack8x(const uint4& q, float (&v)[8], bool f16) {
  float2 a = unpack_16x2(q.x, f16), b = unpack_16x2(q.y, f16), c = unpack_16x2(q.z, f16), d = unpack_16x2(q.w, f16);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void load8x(const bf16* p, float (&v)[8], bool f16) {
  unpack8x(*reinterpret_cast<const uint4*>(p), v, f16);
}
__device__ __forceinline__ void store8x(bf16* p, const float (&v)[8], bool f16) {
  uint4 q;
  q.x = pack_16x2(v[0], v[1], f16); q.y = pack_16x2(v[2], v[3], f16);
  q.z = pack_16x2(v[4], v[5], f16); q.w = pack_16x2(v[6], v[7], f16);
  *reinterpret_cast<uint4*>(p) = q;
}
__device__ __forceinline__ void load8f(const float* p, float (&v)[8]) {
  float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {
  uint4 q;
  q.x = pack_bf16x2(v[0], v[1]); q.y = pack_bf16x2(v[2], v[3]);
  q.z = pack_bf16x2(v[4], v[5]); q.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = q;
}
__device__ __forceinline__ void store8f(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// mean / rstd of one row held as x[MAXC][8] per lane (inactive chunks hold zeros and are excluded via `act`).
template <int MAXC>
__device__ __forceinline__ void row_stats(const float (&x)[MAXC][8], const bool (&act)[MAXC], int H, float eps,
                                          float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s += x[i][j];
  mean = warp_sum(s) / (float)H;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXC; ++i)
    if (act[i]) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { float d = x[i][j] - mean; q += d * d; }
    }
  float var = warp_sum(q) / (float)H;
  rstd = rsqrtf(var + eps);
}

// ------------------------------------------------------------------ LayerNorm forward
template <int MAXC, bool EMBED, bool ZF16>
__global__ void __launch_bounds__(THREADS, 4)
ln_fwd_kernel(const bf16* __restrict__ z, const int64_t* __restrict__ ids, const int64_t* __restrict__ tts,
              const int64_t* __restrict__ pids, const float* __restrict__ word, const float* __restrict__ pos,
              const float* __restrict__ type, const float* __restrict__ gamma, const float* __restrict__ beta,
              bf16* __restrict__ y, bf16* __restrict__ y_res, float* __restrict__ stats, float* __restrict__ cls_out,
              int cls_stride, int T, int H, float eps, Drop drop, int z_f16) {
  // y: bf16 (the next GEMM's A operand, saved for wgrad).  y_res (optional): the same values in fp16 - the copy the
  // next residual add reads (a tensor-core MMA cannot mix an fp16 operand with bf16 weights, so the stream that must
  // stay precise travels beside the GEMM operand instead of replacing it).  z_f16: the input sum holds fp16.
  constexpr bool f16 = ZF16;      // compile-time: a run-time format select costs two conversions + a select per pair
  (void)z_f16;
  // gamma / beta live in shared memory (8 KB at H = 1024), not in 48 registers per thread: at 110 registers only two
  // 8-warp CTAs fit an SM and 16 rows in flight leave the kernel latency-bound (ncu r2: 3.4 TB/s); at ~64 registers
  // four CTAs are resident.
  __shared__ __align__(16) float s_gb[2 * 1024];
  for (int i = threadIdx.x; i < H; i += THREADS) { s_gb[i] = gamma[i]; s_gb[1024 + i] = beta[i]; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * WARPS;
  bool act[MAXC];
#pragma unroll
  for (int i = 0; i < MAXC; ++i) act[i] = (lane + 32 * i) * 8 < H;
  for (int row = warp_global; row < T; row += nwarps) {
    float x[MAXC][8];
    if (EMBED) {
      const long long id = ids[row], tt = tts ? tts[row] : 0, pp = pids[row];
#pragma unroll
      for (int i = 0; i < MAXC; ++i) {
        const int c = (lane + 32 * i) * 8;
        if (act[i]) {
          float w[8], p8[8], t8[8];
          load8f(word + id * H + c, w); load8f(pos + pp * H + c, p8); load8f(type + tt * H + c, t8);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[i][j] = (w[j] + t8[j]) + p8[j];  // HF order: (word + type) + pos
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) x[i][j] = 0.f;
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < MAXC; ++i) {
        const int c = (lane + 32 * i) * 8;
        if (act[i]) load8x(z + (long long)row * H + c, x[i], f16);
        else {
#pragma unroll
          for (int j = 0; j < 8; ++j) x[i][j] = 0.f;
        }
      }
    }
    float mean, rstd;
    row_stats<MAXC>(x, act, H, eps, mean, rstd);
    const bool is_cls = (cls_out != nullptr) && (row % cls_stride == 0);
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      const int c = (lane + 32 * i) * 8;
      if (act[i]) {
        float o[8], g8[8], b8[8];
        load8f(s_gb + c, g8);
        load8f(s_gb + 1024 + c, b8);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (x[i][j] - mean) * rstd * g8[j] + b8[j];
        if (EMBED && drop.on()) {  // embedding dropout (modeling_bert.py:111)
#pragma unroll
          for (int j = 0; j < 8; j += 8) {
            float2 m[4];
            drop.mul8((uint32_t)row, (uint32_t)c, m);
#pragma unroll
            for (int w = 0; w < 4; ++w) { o[2 * w] *= m[w].x; o[2 * w + 1] *= m[w].y; }
          }
        }
        store8(y + (long long)row * H + c, o);
        if (y_res != nullptr) store8x(y_res + (long long)row * H + c, o, true);
        if (is_cls) store8f(cls_out + (long long)(row / cls_stride) * H + c, o);
      }
    }
    if (lane == 0) { stats[2 * (long long)row] = mean; stats[2 * (long long)row + 1] = rstd; }
  }
}

// ------------------------------------------------------------------ LayerNorm backward
// Column accumulators (dgamma, dbeta, dbias / type-table grads) live in registers per lane and are
// flushed once per CTA through shared memory + one atomicAdd per column.
template <int MAXC>
__device__ __forceinline__ void flush_cols(float (&acc)[MAXC][8], const bool (&act)[MAXC], float* smem /*[WARPS][H]*/,
                                           float* __restrict__ out, int H) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < MAXC; ++i)
    if (act[i]) {
      const int c = (lane + 32 * i) * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) smem[warp * H + c + j] = acc[i][j];
    }
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += THREADS) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) s += smem[w * H + c];
    if (s != 0.f) atomicAdd(out + c, s);
  }
}

template <int MAXC, bool EMBED, bool ZF16>
__global__ void __launch_bounds__(THREADS)
ln_bwd_kernel(const bf16* __restrict__ dy, const float* __restrict__ dy_cls, int cls_stride,
              const bf16* __restrict__ z, const int64_t* __restrict__ ids, const int64_t* __restrict__ tts,
              const int64_t* __restrict__ pids, const float* __restrict__ word, const float* __restrict__ pos,
              const float* __restrict__ type, const float* __restrict__ stats, const float* __restrict__ gamma,
              bf16* __restrict__ dz, float* __restrict__ dword, float* __restrict__ dpos, float* __restrict__ dtype,
              float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int T, int H,
              bf16* __restrict__ dzm, Drop drop, int z_f16) {
  extern __shared__ float smem_f[];
  constexpr bool zf16 = ZF16;     // the saved pre-LayerNorm sum z holds fp16 (gradients dy / dz stay bf16)
  (void)z_f16;
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * WARPS;
  bool act[MAXC];
  float g[MAXC][8], ag[MAXC][8], ab[MAXC][8], az[MAXC][8], az1[MAXC][8];
  // EMBED: position-table gradient of the position this warp is currently seeing.  With absolute positions
  // (pos = token index mod S) and a warp stride that is a multiple of S - the common case - every row of a warp has
  // the SAME position, so its 1 024-way contended atomics (131 072 tokens onto 128 rows) become one flush per warp.
  float apos[EMBED ? MAXC : 1][8];
  long long cur_pp = -1;
#pragma unroll
  for (int i = 0; i < MAXC; ++i) {
    const int c = (lane + 32 * i) * 8;
    act[i] = c < H;
    if (act[i]) load8f(gamma + c, g[i]);
#pragma unroll
    for (int j = 0; j < 8; ++j) { ag[i][j] = 0.f; ab[i][j] = 0.f; az[i][j] = 0.f; az1[i][j] = 0.f; }
    if (EMBED) {
#pragma unroll
      for (int j = 0; j < 8; ++j) apos[i][j] = 0.f;
    }
  }
  auto flush_pos = [&]() {
    if (EMBED && cur_pp >= 0) {
#pragma unroll
      for (int i = 0; i < MAXC; ++i)
        if (act[i]) {
          const int c = (lane + 32 * i) * 8;
          red_add_v4_f32(dpos + cur_pp * H + c, apos[i][0], apos[i][1], apos[i][2], apos[i][3]);
          red_add_v4_f32(dpos + cur_pp * H + c + 4, apos[i][4], apos[i][5], apos[i][6], apos[i][7]);
#pragma unroll
          for (int j = 0; j < 8; ++j) apos[i][j] = 0.f;
        }
    }
  };
  // Dense path: each lane stages its own 16-byte chunks of the next PF_DEPTH rows in shared memory with cp.async
  // (a per-lane FIFO: no cross-lane visibility needed), so PF_DEPTH rows of dy and z are in flight per warp —
  // at one 8-warp CTA per SM (register-bound) a single row in flight leaves the kernel latency-bound at ~2.5 TB/s.
  const bool sparse_dy = (dy_cls != nullptr);
  const bool dense_path = !EMBED && !sparse_dy;
  constexpr int SLOT_BYTES = 2 * MAXC * 512 + 16;  // z chunks | dy chunks | (mean, rstd)
  uint8_t* ring = reinterpret_cast<uint8_t*>(smem_f) + (size_t)(threadIdx.x >> 5) * PF_DEPTH * SLOT_BYTES;
  auto stage = [&](int r, int slot) {
    if (r < T) {
#pragma unroll
      for (int i = 0; i < MAXC; ++i)
        if (act[i]) {
          const long long o = (long long)r * H + (lane + 32 * i) * 8;
          uint8_t* dst = ring + slot * SLOT_BYTES + i * 512 + lane * 16;
          cp_async_16(dst, z + o);
          cp_async_16(dst + MAXC * 512, dy + o);
        }
      if (lane == 0) cp_async_8(ring + slot * SLOT_BYTES + 2 * MAXC * 512, stats + 2 * (long long)r);
    }
    cp_async_commit();
  };
  if (dense_path) {
#pragma unroll
    for (int d = 0; d < PF_DEPTH - 1; ++d) stage(warp_global + d * nwarps, d);
  }
  int it = 0;
  for (int row = warp_global; row < T; row += nwarps, ++it) {
    uint4 cz[MAXC], cdy[MAXC];
    float pf_mean = 0.f, pf_rstd = 0.f;
    if (dense_path) {
      stage(row + (PF_DEPTH - 1) * nwarps, (it + PF_DEPTH - 1) % PF_DEPTH);
      cp_async_wait<PF_DEPTH - 1>();
      const int slot = it % PF_DEPTH;
#pragma unroll
      for (int i = 0; i < MAXC; ++i)
        if (act[i]) {
          const uint8_t* src = ring + slot * SLOT_BYTES + i * 512 + lane * 16;
          cz[i] = *reinterpret_cast<const uint4*>(src);
          cdy[i] = *reinterpret_cast<const uint4*>(src + MAXC * 512);
        }
      __syncwarp();  // lane 0's (mean, rstd) copy must be visible to the whole warp
      const float2 st = *reinterpret_cast<const float2*>(ring + slot * SLOT_BYTES + 2 * MAXC * 512);
      pf_mean = st.x; pf_rstd = st.y;
    }
    if (sparse_dy && (row % cls_stride != 0)) {
      // upstream gradient is identically zero for this row, and so is its dropped copy (the next GEMMs read every row)
#pragma unroll
      for (int i = 0; i < MAXC; ++i)
        if (act[i]) {
          const long long o = (long long)row * H + (lane + 32 * i) * 8;
          if (dz != nullptr) *reinterpret_cast<uint4*>(dz + o) = make_uint4(0, 0, 0, 0);
          if (dzm != nullptr) *reinterpret_cast<uint4*>(dzm + o) = make_uint4(0, 0, 0, 0);
        }
      continue;
    }
    const float mean = dense_path ? pf_mean : stats[2 * (long long)row];
    const float rstd = dense_path ? pf_rstd : stats[2 * (long long)row + 1];
    long long id = 0, tt = 0, pp = 0;
    if (EMBED) {
      id = ids[row]; tt = tts ? tts[row] : 0; pp = pids[row];
      if (pp != cur_pp) { flush_pos(); cur_pp = pp; }    // warp-uniform
    }
    float xh[MAXC][8], d[MAXC][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      const int c = (lane + 32 * i) * 8;
      if (act[i]) {
        float x[8];
        if (EMBED) {
          float w[8], p8[8], t8[8];
          load8f(word + id * H + c, w); load8f(pos + pp * H + c, p8); load8f(type + tt * H + c, t8);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = (w[j] + t8[j]) + p8[j];
        } else if (dense_path) {
          unpack8x(cz[i], x, zf16);
        } else {
          load8x(z + (long long)row * H + c, x, zf16);
        }
        if (sparse_dy) load8f(dy_cls + (long long)(row / cls_stride) * H + c, d[i]);
        else if (dense_path) unpack8(cdy[i], d[i]);
        else load8(dy + (long long)row * H + c, d[i]);
        if (EMBED && drop.on()) {  // upstream gradient is w.r.t. the dropped embedding output
#pragma unroll
          for (int j = 0; j < 8; j += 8) {
            float2 m[4];
            drop.mul8((uint32_t)row, (uint32_t)c, m);
#pragma unroll
            for (int w = 0; w < 4; ++w) { d[i][2 * w] *= m[w].x; d[i][2 * w + 1] *= m[w].y; }
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = (x[j] - mean) * rstd;
          ag[i][j] += d[i][j] * xh[i][j];
          ab[i][j] += d[i][j];
          d[i][j] *= g[i][j];  // dxhat
          s1 += d[i][j];
          s2 += d[i][j] * xh[i][j];
        }
      }
    }
    s1 = warp_sum(s1) / (float)H;
    s2 = warp_sum(s2) / (float)H;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      const int c = (lane + 32 * i) * 8;
      if (act[i]) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (d[i][j] - s1 - xh[i][j] * s2);
        if (EMBED) {
          // scatter-add into the table gradients with 16-byte vector reductions (red.global.add.v4.f32: a quarter of
          // the atomic instructions of the scalar form); the (tiny) type table is accumulated in registers
          red_add_v4_f32(dword + id * H + c, o[0], o[1], o[2], o[3]);
          red_add_v4_f32(dword + id * H + c + 4, o[4], o[5], o[6], o[7]);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            apos[EMBED ? i : 0][j] += o[j];
            if (tt == 0) az[i][j] += o[j];
            else if (tt == 1) az1[i][j] += o[j];
            else atomicAdd(dtype + tt * H + c + j, o[j]);
          }
        } else {
          store8(dz + (long long)row * H + c, o);
          if (dzm != nullptr) {
            // hidden dropout sat between the Linear and this residual+LayerNorm: the Linear's output gradient is
            // dz * mask / (1-p) (second output), while the residual branch takes dz itself
#pragma unroll
            for (int j = 0; j < 8; j += 8) {
              float2 m[4];
              drop.mul8((uint32_t)row, (uint32_t)c, m);
#pragma unroll
              for (int w = 0; w < 4; ++w) { o[2 * w] *= m[w].x; o[2 * w + 1] *= m[w].y; }
            }
            store8(dzm + (long long)row * H + c, o);
          }
          if (dbias != nullptr) {
            // accumulate the bf16-rounded value: it is what the downstream GEMMs consume
#pragma unroll
            for (int j = 0; j < 8; ++j) az[i][j] += __bfloat162float(__float2bfloat16(o[j]));
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  flush_pos();
  flush_cols<MAXC>(ag, act, smem_f, dgamma, H);
  flush_cols<MAXC>(ab, act, smem_f, dbeta, H);
  if (EMBED) {
    flush_cols<MAXC>(az, act, smem_f, dtype, H);
    flush_cols<MAXC>(az1, act, smem_f, dtype + H, H);
  } else if (dbias != nullptr) {
    flush_cols<MAXC>(az, act, smem_f, dbias, H);
  }
}

// ------------------------------------------------------------------ full-width rows: H == MAXC * 256, dense dy
// The encoder's LayerNorms (H = 768 / 1024, every row has an upstream gradient) take these two kernels.  They do the
// same arithmetic as ln_fwd_kernel / ln_bwd_kernel on PAIRS of columns, without the per-chunk width predicates, and
// keep gamma / beta in shared memory in a bank-conflict-free layout: the generic kernels spend most of their issue
// slots on those predicates and index computations.
//
// Shared-memory layout of a per-column vector v[H] ("pair layout"): chunk i of lane l holds columns c .. c+7 with
// c = (32 i + l) * 8; columns c..c+3 live at [i*256 + l*4], columns c+4..c+7 at [i*256 + 128 + l*4], so both 16-byte
// reads of a lane are conflict-free.
__device__ __forceinline__ int pair_layout(int col) {
  const int i = col >> 8, r = col & 255, l = r >> 3, j = r & 7;
  return i * 256 + (j >> 2) * 128 + l * 4 + (j & 3);
}
__device__ __forceinline__ void lds8_pairs(const float* base, int i, int lane, float2 (&v)[4]) {
  const float4 a = *reinterpret_cast<const float4*>(base + i * 256 + lane * 4);
  const float4 b = *reinterpret_cast<const float4*>(base + i * 256 + 128 + lane * 4);
  v[0] = make_float2(a.x, a.y); v[1] = make_float2(a.z, a.w); v[2] = make_float2(b.x, b.y); v[3] = make_float2(b.z, b.w);
}
__device__ __forceinline__ void unpack8_pairs(const uint4& q, float2 (&v)[4], bool f16) {
  v[0] = unpack_16x2(q.x, f16); v[1] = unpack_16x2(q.y, f16); v[2] = unpack_16x2(q.z, f16); v[3] = unpack_16x2(q.w, f16);
}

template <int MAXC, bool ZF16>
__global__ void __launch_bounds__(THREADS, 4)
ln_fwd_full_kernel(const bf16* __restrict__ z, const float* __restrict__ gamma, const float* __restrict__ beta,
                   bf16* __restrict__ y, bf16* __restrict__ y_res, float* __restrict__ stats,
                   float* __restrict__ cls_out, int cls_stride, int T, float eps) {
  constexpr int H = MAXC * 256;
  __shared__ __align__(16) float s_g[H];
  __shared__ __align__(16) float s_b[H];
  for (int i = threadIdx.x; i < H; i += THREADS) { s_g[pair_layout(i)] = gamma[i]; s_b[pair_layout(i)] = beta[i]; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * WARPS;
  for (int row = warp_global; row < T; row += nwarps) {
    const uint4* zr = reinterpret_cast<const uint4*>(z + (long long)row * H) + lane;
    uint4 q[MAXC];
#pragma unroll
    for (int i = 0; i < MAXC; ++i) q[i] = ldg_nc_v4(zr + 32 * i);
    float2 x[MAXC][4];
#pragma unroll
    for (int i = 0; i < MAXC; ++i) unpack8_pairs(q[i], x[i], ZF16);
    float2 s = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < MAXC; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k) s = fadd2(s, x[i][k]);
    const float mean = warp_sum(s.x + s.y) / (float)H;
    const float2 nm = make_float2(-mean, -mean);
    float2 qq = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < MAXC; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k) { x[i][k] = fadd2(x[i][k], nm); qq = ffma2(x[i][k], x[i][k], qq); }
    const float var = warp_sum(qq.x + qq.y) / (float)H;
    const float rstd = rsqrtf(var + eps);
    const float2 r2 = make_float2(rstd, rstd);
    const bool is_cls = (cls_out != nullptr) && (row % cls_stride == 0);
    uint4* yr = reinterpret_cast<uint4*>(y + (long long)row * H) + lane;
    uint4* yres = y_res ? reinterpret_cast<uint4*>(y_res + (long long)row * H) + lane : nullptr;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      float2 g[4], b[4], o[4];
      lds8_pairs(s_g, i, lane, g);
      lds8_pairs(s_b, i, lane, b);
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = ffma2(fmul2(x[i][k], r2), g[k], b[k]);
      yr[32 * i] = make_uint4(pack_bf16x2(o[0].x, o[0].y), pack_bf16x2(o[1].x, o[1].y), pack_bf16x2(o[2].x, o[2].y),
                              pack_bf16x2(o[3].x, o[3].y));
      if (yres != nullptr)
        yres[32 * i] = make_uint4(pack_f16x2(o[0].x, o[0].y), pack_f16x2(o[1].x, o[1].y), pack_f16x2(o[2].x, o[2].y),
                                  pack_f16x2(o[3].x, o[3].y));
      if (is_cls) {
        float* co = cls_out + (long long)(row / cls_stride) * H + (lane + 32 * i) * 8;
        *reinterpret_cast<float4*>(co) = make_float4(o[0].x, o[0].y, o[1].x, o[1].y);
        *reinterpret_cast<float4*>(co + 4) = make_float4(o[2].x, o[2].y, o[3].x, o[3].y);
      }
    }
    if (lane == 0) *reinterpret_cast<float2*>(stats + 2 * (long long)row) = make_float2(mean, rstd);
  }
}

template <int MAXC, bool ZF16>
__global__ void __launch_bounds__(THREADS)
ln_bwd_full_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z, const float* __restrict__ stats,
                   const float* __restrict__ gamma, bf16* __restrict__ dz, float* __restrict__ dgamma,
                   float* __restrict__ dbeta, float* __restrict__ dbias, int T, bf16* __restrict__ dzm, Drop drop) {
  constexpr int H = MAXC * 256;
  constexpr int SLOT_BYTES = 2 * MAXC * 512 + 16;  // z chunks | dy chunks | (mean, rstd)
  constexpr int RING_BYTES = WARPS * PF_DEPTH * SLOT_BYTES;
  constexpr int FLUSH_BYTES = WARPS * H * 4;
  constexpr int FRONT_BYTES = RING_BYTES > FLUSH_BYTES ? RING_BYTES : FLUSH_BYTES;
  extern __shared__ float smem_f[];
  float* s_g = smem_f + FRONT_BYTES / 4;           // gamma in pair layout, behind the ring / flush area
  for (int i = threadIdx.x; i < H; i += THREADS) s_g[pair_layout(i)] = gamma[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp_global = blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * WARPS;
  float2 ag[MAXC][4], ab[MAXC][4], az[MAXC][4];
#pragma unroll
  for (int i = 0; i < MAXC; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) { ag[i][k] = make_float2(0.f, 0.f); ab[i][k] = ag[i][k]; az[i][k] = ag[i][k]; }
  // per-lane FIFO of the next PF_DEPTH rows (see ln_bwd_kernel)
  uint8_t* ring = reinterpret_cast<uint8_t*>(smem_f) + (size_t)(threadIdx.x >> 5) * PF_DEPTH * SLOT_BYTES;
  auto stage = [&](int r, int slot) {
    if (r < T) {
      const bf16* zs = z + (long long)r * H + lane * 8;
      const bf16* ds = dy + (long long)r * H + lane * 8;
      uint8_t* dst = ring + slot * SLOT_BYTES + lane * 16;
#pragma unroll
      for (int i = 0; i < MAXC; ++i) {
        cp_async_16(dst + i * 512, zs + i * 256);
        cp_async_16(dst + (MAXC + i) * 512, ds + i * 256);
      }
      if (lane == 0) cp_async_8(ring + slot * SLOT_BYTES + 2 * MAXC * 512, stats + 2 * (long long)r);
    }
    cp_async_commit();
  };
#pragma unroll
  for (int d = 0; d < PF_DEPTH - 1; ++d) stage(warp_global + d * nwarps, d);
  const bool do_drop = (dzm != nullptr);
  const bool do_bias = (dbias != nullptr);
  int slot = 0;
  for (int row = warp_global; row < T; row += nwarps) {
    stage(row + (PF_DEPTH - 1) * nwarps, (slot + PF_DEPTH - 1) % PF_DEPTH);
    cp_async_wait<PF_DEPTH - 1>();
    const uint8_t* src = ring + slot * SLOT_BYTES + lane * 16;
    uint4 cz[MAXC], cdy[MAXC];
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      cz[i] = *reinterpret_cast<const uint4*>(src + i * 512);
      cdy[i] = *reinterpret_cast<const uint4*>(src + (MAXC + i) * 512);
    }
    __syncwarp();  // lane 0's (mean, rstd) copy must be visible to the whole warp
    const float2 st = *reinterpret_cast<const float2*>(ring + slot * SLOT_BYTES + 2 * MAXC * 512);
    slot = (slot + 1) % PF_DEPTH;
    const float mean = st.x, rstd = st.y;
    const float2 nm = make_float2(-mean, -mean), r2 = make_float2(rstd, rstd);
    float2 xh[MAXC][4], d[MAXC][4];
    float2 s1 = make_float2(0.f, 0.f), s2 = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      float2 g[4];
      lds8_pairs(s_g, i, lane, g);
      unpack8_pairs(cz[i], xh[i], ZF16);
      unpack8_pairs(cdy[i], d[i], false);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        xh[i][k] = fmul2(fadd2(xh[i][k], nm), r2);
        ag[i][k] = ffma2(d[i][k], xh[i][k], ag[i][k]);
        ab[i][k] = fadd2(ab[i][k], d[i][k]);
        d[i][k] = fmul2(d[i][k], g[k]);       // dxhat
        s1 = fadd2(s1, d[i][k]);
        s2 = ffma2(d[i][k], xh[i][k], s2);
      }
    }
    const float m1 = warp_sum(s1.x + s1.y) / (float)H;
    const float m2 = warp_sum(s2.x + s2.y) / (float)H;
    const float2 nm1 = make_float2(-m1, -m1), nm2 = make_float2(-m2, -m2);
    uint4* dzr = reinterpret_cast<uint4*>(dz + (long long)row * H) + lane;
    uint4* dzmr = do_drop ? reinterpret_cast<uint4*>(dzm + (long long)row * H) + lane : nullptr;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
      float2 o[4];
      uint32_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        o[k] = fmul2(r2, fadd2(ffma2(xh[i][k], nm2, d[i][k]), nm1));   // rstd * (d - s1 - xh * s2)
        w[k] = pack_bf16x2(o[k].x, o[k].y);
      }
      dzr[32 * i] = make_uint4(w[0], w[1], w[2], w[3]);
      if (do_drop) {
        // hidden dropout sat between the Linear and this residual+LayerNorm: the Linear's output gradient is
        // dz * mask / (1-p) (second output), while the residual branch takes dz itself
        float2 m[4];
        drop.mul8((uint32_t)row, (uint32_t)(lane + 32 * i) * 8u, m);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 om = fmul2(o[k], m[k]);
          w[k] = pack_bf16x2(om.x, om.y);
        }
        dzmr[32 * i] = make_uint4(w[0], w[1], w[2], w[3]);
      }
      if (do_bias) {
        // the Linear's bias gradient: column sums of ITS output gradient (the masked copy when dropout is on), as the
        // bf16-rounded values the downstream GEMMs consume
#pragma unroll
        for (int k = 0; k < 4; ++k) az[i][k] = fadd2(az[i][k], unpack_bf16x2(w[k]));
      }
    }
  }
  cp_async_wait<0>();
  bool act[MAXC];
  float t[MAXC][8];
#pragma unroll
  for (int i = 0; i < MAXC; ++i) act[i] = true;
  auto flush = [&](float2 (&a)[MAXC][4], float* out) {
#pragma unroll
    for (int i = 0; i < MAXC; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k) { t[i][2 * k] = a[i][k].x; t[i][2 * k + 1] = a[i][k].y; }
    flush_cols<MAXC>(t, act, smem_f, out, H);
  };
  flush(ag, dgamma);
  flush(ab, dbeta);
  if (do_bias) flush(az, dbias);
}

// ------------------------------------------------------------------ column sums (bias gradients)
__global__ void __launch_bounds__(THREADS)
colsum_kernel(const bf16* __restrict__ x, long long ld, float* __restrict__ out, int T, int N, int rows_per_cta) {
  __shared__ float red[WARPS][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, T);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c < N) {
    for (int r = r0 + warp; r < r1; r += WARPS) {
      float v[8];
      load8(x + (long long)r * ld + c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int cc = blockIdx.x * 256 + threadIdx.x;
  if (threadIdx.x < 256 && cc < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) s += red[w][threadIdx.x];
    atomicAdd(out + cc, s);
  }
}

// hact = gelu(pre) over a flat bf16 array (8 elements per thread): the "lean activations" backward rebuilds the GELU
// output it did not save, as the operand of the FFN-out weight gradient.
__global__ void __launch_bounds__(256)
gelu_from_pre_kernel(const bf16* __restrict__ pre, bf16* __restrict__ out, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 q = ldg_nc_v4(pre + i * 8);
    const uint32_t in[4] = {q.x, q.y, q.z, q.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float2 g, d;
      gelu_and_grad2(unpack_bf16x2(in[t]), g, d);
      o[t] = pack_bf16x2(g.x, g.y);
    }
    *reinterpret_cast<uint4*>(out + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int grid_for_rows(int T, int sms) {
  long long want = ((long long)T + WARPS - 1) / WARPS;
  long long cap = (long long)sms * 4;
  return (int)(want < cap ? want : cap);
}

}  // namespace

#define DISPATCH_MAXC(H, CALL)                                    \
  do {                                                            \
    const int _c = ((H) + 255) / 256;                             \
    if (_c == 1) { CALL(1); } else if (_c == 2) { CALL(2); }      \
    else if (_c == 3) { CALL(3); } else { CALL(4); }              \
  } while (0)

// A/B aid for tools/ln_bench.py: DPRB_LN_GENERIC=1 sends full-width rows through the generic kernels too.
static bool ln_generic_forced() {
  const char* e = getenv("DPRB_LN_GENERIC");
  return e != nullptr && e[0] == '1';
}

static int check_h(int H, const char* who) {
  DPRB_REQUIRE(H > 0 && H % 8 == 0 && H <= 1024, "%s: hidden size %d unsupported (need H %% 8 == 0, H <= 1024)", who, H);
  return 0;
}

__global__ void dropout_mask_kernel(uint8_t* out, long long rows, int cols, Drop drop) {
  const long long n = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)(i / cols), c = (uint32_t)(i % cols);
    float m0, m1;
    drop.mul2(r, c & ~1u, m0, m1);
    out[i] = drop.on() ? (uint8_t)(((c & 1u) ? m1 : m0) != 0.f) : (uint8_t)1;
  }
}

}  // namespace dprb

using namespace dprb;

extern "C" int dprb_embed_ln_fwd(const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids, const float* word,
                                 const float* pos, const float* type, const float* gamma, const float* beta, void* y,
                                 float* stats, int T, int H, int vocab, int max_pos, int type_vocab, float eps,
                                 float dropout_p, uint64_t seed, void* y_res, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Drop drop = make_drop(dropout_p, seed, 0, DROP_SITE_EMBED);
  if (int rc = check_h(H, "embed_ln_fwd")) return rc;
  if (T == 0) return 0;
  (void)vocab; (void)max_pos; (void)type_vocab;
  DPRB_NUM_SMS(sms);
  const int grid = grid_for_rows(T, sms);
#define CALL(C) ln_fwd_kernel<C, true, false><<<grid, THREADS, 0, stream>>>(nullptr, ids, type_ids, pos_ids, word, pos, type, gamma, beta, (bf16*)y, (bf16*)y_res, stats, nullptr, 1, T, H, eps, drop, 0)
  DISPATCH_MAXC(H, CALL);
#undef CALL
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_ln_fwd(const void* z, const float* gamma, const float* beta, void* y, float* stats, float* cls_out,
                           int cls_stride, int T, int H, float eps, int z_f16, void* y_res, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = check_h(H, "ln_fwd")) return rc;
  if (T == 0) return 0;
  DPRB_REQUIRE(cls_out == nullptr || cls_stride > 0, "ln_fwd: cls_stride must be positive");
  DPRB_NUM_SMS(sms);
  const int grid = grid_for_rows(T, sms);
  if (H % 256 == 0 && !ln_generic_forced()) {   // full-width rows (the encoder's H = 768 / 1024): paired-column kernel
#define CALLF(C)                                                                                                         \
  do {                                                                                                                   \
    if (z_f16) ln_fwd_full_kernel<C, true><<<grid, THREADS, 0, stream>>>((const bf16*)z, gamma, beta, (bf16*)y, (bf16*)y_res, stats, cls_out, cls_stride > 0 ? cls_stride : 1, T, eps); \
    else ln_fwd_full_kernel<C, false><<<grid, THREADS, 0, stream>>>((const bf16*)z, gamma, beta, (bf16*)y, (bf16*)y_res, stats, cls_out, cls_stride > 0 ? cls_stride : 1, T, eps); \
  } while (0)
    DISPATCH_MAXC(H, CALLF);
#undef CALLF
    DPRB_LAUNCH_CHECK();
    return 0;
  }
#define CALL(C)                                                                                                          \
  do {                                                                                                                   \
    if (z_f16) ln_fwd_kernel<C, false, true><<<grid, THREADS, 0, stream>>>((const bf16*)z, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, gamma, beta, (bf16*)y, (bf16*)y_res, stats, cls_out, cls_stride > 0 ? cls_stride : 1, T, H, eps, Drop{0u, 0u, 1.f, 1u}, 1); \
    else ln_fwd_kernel<C, false, false><<<grid, THREADS, 0, stream>>>((const bf16*)z, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, gamma, beta, (bf16*)y, (bf16*)y_res, stats, cls_out, cls_stride > 0 ? cls_stride : 1, T, H, eps, Drop{0u, 0u, 1.f, 1u}, 0); \
  } while (0)
  DISPATCH_MAXC(H, CALL);
#undef CALL
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_ln_bwd(const void* dy, const float* dy_cls, int cls_stride, const void* z, const float* stats,
                           const float* gamma, void* dz, float* dgamma, float* dbeta, float* dbias, int T, int H,
                           void* dzm, float dropout_p, uint64_t site_seed, int z_f16, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Drop drop = drop_from_site(dropout_p, site_seed);  // the caller passes the derived site seed
  if (!drop.on()) dzm = nullptr;
  if (int rc = check_h(H, "ln_bwd")) return rc;
  if (T == 0) return 0;
  DPRB_REQUIRE((dy != nullptr) != (dy_cls != nullptr), "ln_bwd: exactly one of dy / dy_cls must be given");
  DPRB_REQUIRE(dy_cls == nullptr || cls_stride > 0, "ln_bwd: cls_stride must be positive");
  DPRB_NUM_SMS(sms);
  const int grid = grid_for_rows(T, sms);
  const int maxc = (H + 255) / 256;
  if (dy != nullptr && H % 256 == 0 && !ln_generic_forced()) {   // dense upstream gradient, full-width rows: paired-column kernel
    size_t front = (size_t)WARPS * H * sizeof(float);
    const size_t ring_f = (size_t)WARPS * PF_DEPTH * (2 * maxc * 512 + 16);
    if (ring_f > front) front = ring_f;
    const size_t smem_f = front + (size_t)H * sizeof(float);
    static bool attr_f = false;
    if (!attr_f) {
#define SET_ATTR_F(C)                                                                                                                    \
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(ln_bwd_full_kernel<C, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 164 * 1024)); \
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(ln_bwd_full_kernel<C, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 164 * 1024));
      SET_ATTR_F(1) SET_ATTR_F(2) SET_ATTR_F(3) SET_ATTR_F(4)
#undef SET_ATTR_F
      attr_f = true;
    }
#define CALLF(C)                                                                                                         \
  do {                                                                                                                   \
    if (z_f16) ln_bwd_full_kernel<C, true><<<grid, THREADS, smem_f, stream>>>((const bf16*)dy, (const bf16*)z, stats, gamma, (bf16*)dz, dgamma, dbeta, dbias, T, (bf16*)dzm, drop); \
    else ln_bwd_full_kernel<C, false><<<grid, THREADS, smem_f, stream>>>((const bf16*)dy, (const bf16*)z, stats, gamma, (bf16*)dz, dgamma, dbeta, dbias, T, (bf16*)dzm, drop); \
  } while (0)
    DISPATCH_MAXC(H, CALLF);
#undef CALLF
    DPRB_LAUNCH_CHECK();
    return 0;
  }
  size_t smem = (size_t)WARPS * H * sizeof(float);
  const size_t ring = (size_t)WARPS * PF_DEPTH * (2 * maxc * 512 + 16);
  if (ring > smem) smem = ring;
  static bool attr = false;
  if (!attr) {
#define SET_ATTR(C)                                                                                                                       \
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(ln_bwd_kernel<C, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); \
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(ln_bwd_kernel<C, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    SET_ATTR(1) SET_ATTR(2) SET_ATTR(3) SET_ATTR(4)
#undef SET_ATTR
    attr = true;
  }
#define CALL(C)                                                                                                          \
  do {                                                                                                                   \
    if (z_f16) ln_bwd_kernel<C, false, true><<<grid, THREADS, smem, stream>>>((const bf16*)dy, dy_cls, cls_stride > 0 ? cls_stride : 1, (const bf16*)z, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stats, gamma, (bf16*)dz, nullptr, nullptr, nullptr, dgamma, dbeta, dbias, T, H, (bf16*)dzm, drop, 1); \
    else ln_bwd_kernel<C, false, false><<<grid, THREADS, smem, stream>>>((const bf16*)dy, dy_cls, cls_stride > 0 ? cls_stride : 1, (const bf16*)z, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stats, gamma, (bf16*)dz, nullptr, nullptr, nullptr, dgamma, dbeta, dbias, T, H, (bf16*)dzm, drop, 0); \
  } while (0)
  DISPATCH_MAXC(H, CALL);
#undef CALL
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_embed_ln_bwd(const void* dy, const int64_t* ids, const int64_t* type_ids, const int64_t* pos_ids,
                                 const float* word, const float* pos, const float* type, const float* gamma,
                                 const float* stats, float* dword, float* dpos, float* dtype, float* dgamma,
                                 float* dbeta, int T, int H, float dropout_p, uint64_t seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Drop drop = make_drop(dropout_p, seed, 0, DROP_SITE_EMBED);
  if (int rc = check_h(H, "embed_ln_bwd")) return rc;
  if (T == 0) return 0;
  DPRB_NUM_SMS(sms);
  const int grid = grid_for_rows(T, sms);
  const size_t smem = (size_t)WARPS * H * sizeof(float);
#define CALL(C) ln_bwd_kernel<C, true, false><<<grid, THREADS, smem, stream>>>((const bf16*)dy, nullptr, 1, nullptr, ids, type_ids, pos_ids, word, pos, type, stats, gamma, nullptr, dword, dpos, dtype, dgamma, dbeta, nullptr, T, H, nullptr, drop, 0)
  DISPATCH_MAXC(H, CALL);
#undef CALL
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" uint64_t dprb_dropout_site_seed(uint64_t dropout_seed, int layer, int site) {
  return drop_site_seed64(dropout_seed, layer, site);
}

// Test aid: materialise the keep mask keep[r * cols + c] of one dropout site (the kernels never store masks).
extern "C" int dprb_dropout_mask(uint8_t* out, int64_t rows, int cols, float p, uint64_t seed, int layer, int site,
                                 dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (rows <= 0 || cols <= 0) return 0;
  const Drop d = make_drop(p, seed, layer, site);
  const long long n = rows * cols;
  dropout_mask_kernel<<<(int)((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256), 256, 0, stream>>>(out, rows, cols, d);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_colsum_bf16(const void* x, int64_t ld, float* out, int T, int N, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(N % 8 == 0 && ld % 8 == 0, "colsum: N=%d and ld=%lld must be multiples of 8", N, (long long)ld);
  if (T == 0 || N == 0) return 0;
  DPRB_NUM_SMS(sms);
  const int col_blocks = (N + 255) / 256;
  int row_chunks = (sms * 4 + col_blocks - 1) / col_blocks;
  int rows_per_cta = (T + row_chunks - 1) / row_chunks;
  if (rows_per_cta < 64) rows_per_cta = 64;
  row_chunks = (T + rows_per_cta - 1) / rows_per_cta;
  dim3 grid(col_blocks, row_chunks);
  colsum_kernel<<<grid, THREADS, 0, stream>>>((const bf16*)x, ld, out, T, N, rows_per_cta);
  DPRB_LAUNCH_CHECK();
  return 0;
}

extern "C" int dprb_gelu_from_pre(const void* pre, void* out, int64_t n, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(n % 8 == 0 && ((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
               "gelu_from_pre: n %% 8 == 0 and 16-byte aligned buffers required");
  if (n == 0) return 0;
  DPRB_NUM_SMS(sms);
  const long long n8 = n / 8;
  const long long want = (n8 + 255) / 256;
  gelu_from_pre_kernel<<<(int)(want < (long long)sms * 8 ? want : (long long)sms * 8), 256, 0, stream>>>((const bf16*)pre, (bf16*)out, n8);
  DPRB_LAUNCH_CHECK();
  return 0;
}
