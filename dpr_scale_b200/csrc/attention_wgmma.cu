// Self-attention core on Hopper warpgroup MMA (wgmma) for head_dim 64 and S <= 256.
//
//   forward : one CTA (one warpgroup) = 64 query rows of one (sequence, head) problem.  Q, K, V arrive by TMA
//             (128B-swizzled); S = Q K^T (wgmma m64nNKk16, fp32 in registers) -> exact row softmax in registers
//             (a row lives in the 4 threads of a quad) -> P (bf16) stays in registers as the A operand of
//             O = P V (wgmma RS form, V read in place as an MN-major operand) -> O / l -> ctx.  LSE saved for backward.
//   backward, S <= 128 (attn_bwd_short): persistent CTAs, each looping over problems of one head with the next
//             problem's Q, K, V, dO in flight (double-buffered TMA).  Warpgroup w owns query rows 64w .. 64w+63 and the
//             whole key row: S = Q K^T and dP = dO V^T (wgmma) -> P = exp2(S - lse), D = sum P~ dP and
//             dS = P (m dP - D) / 8 in fp32 registers -> dQ = dS K (RS form, written once).  P~ and dS are staged as
//             bf16 [query][key] tiles; after a CTA barrier warpgroup w computes dV = P~^T dO and dK = dS^T Q for keys
//             64w .. 64w+63 (staged tiles as MN-major A).  The QKV bias gradient (column sums of the bf16 dQ, dK, dV)
//             is summed per CTA and added once per column at the end.
//   backward, 128 < S <= 256: one CTA = one problem, two warpgroups.  Each warpgroup owns 64-key blocks and walks the
//             query blocks: S^T = K Q^T and dP^T = V dO^T (wgmma) -> P^T = exp2(S^T - lse), dS^T = P^T (dP^T - D) / 8
//             in registers -> dV += P^T dO and dK += dS^T Q (RS form, accumulators stay in registers across query
//             blocks) -> dS^T staged in shared memory -> dQ_part = dS K (both operands MN-major) added into an fp32 dQ
//             accumulator in shared memory.  D_i = sum_j P_ij dP_ij is computed first, in fp32, by a row pass.
//
// Tiles are moved by TMA through 3-D tensor maps [nseq, S, columns]: rows >= S of a short sequence are zero-filled on
// load, so only stores need row predicates.
//
// Replaces BertSelfAttention.forward's scaled_dot_product_attention and its autograd backward.
#include "attention.cuh"
#include "dprb_internal.h"

#include <algorithm>

namespace dprb {
namespace {

template <int N>
__device__ __forceinline__ void mma_ss(float (&d)[N / 2], uint64_t a, uint64_t b, int acc) {
  if constexpr (N == 64) wgmma_m64n64_ss_bf16<0, 0>(d, a, b, acc);
  else if constexpr (N == 128) wgmma_m64n128_ss_bf16<0, 0>(d, a, b, acc);
  else wgmma_m64n256_ss_bf16<0, 0>(d, a, b, acc);
}

// ------------------------------------------------------------------------------------------ forward
template <int NK>
constexpr int fwd_smem() { return 64 * 128 + 2 * NK * 128 + NK * 4 + 16 + 1024; }

template <int NK, bool DROP>
__global__ void __launch_bounds__(128)
attn_fwd_wg_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv,
                   const int32_t* __restrict__ attn_mask, bf16* __restrict__ ctx, float* __restrict__ lse_out, int S,
                   int heads, Drop drop) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;                       // [64][64]
  uint8_t* sK = sQ + 64 * 128;              // [NK][64]
  uint8_t* sV = sK + NK * 128;              // [NK][64]
  float* sMask = reinterpret_cast<float*>(sV + NK * 128);   // [NK]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sMask + NK);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3;
  // 1-D grid, query blocks of one problem adjacent: gridDim.y (65 535) would cap nseq * heads
  const int nqb = (S + 63) / 64;
  const int prob = blockIdx.x / nqb, qb = blockIdx.x - prob * nqb;
  const int seq = prob / heads, h = prob - seq * heads;
  const int H = heads * 64;
  if (tid == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_kv);
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 64 * 128 + 2 * NK * 128);
    tma_load_3d(sQ, &tm_q, bar, h * 64, qb * 64, seq);
    tma_load_3d(sK, &tm_kv, bar, H + h * 64, 0, seq);
    tma_load_3d(sV, &tm_kv, bar, 2 * H + h * 64, 0, seq);
  }
  for (int j = tid; j < NK; j += 128) {
    const bool keep = j < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + j] != 0);
    sMask[j] = keep ? 0.f : -INFINITY;
  }
  __syncthreads();
  mbar_wait(bar, 0);

  // S = Q K^T
  float s[NK / 2];
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) mma_ss<NK>(s, desc_k(sQ) + k * KSTEP_K, desc_k(sK) + k * KSTEP_K, k > 0);
  wgmma_commit();
  wgmma_wait<0>();

  // row softmax: this thread holds rows lrow (h2 = 0) and lrow + 8 (h2 = 1), columns 8c + 2 q4 + {0, 1}
  const int lrow = warp * 16 + (lane >> 2);
  float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int c = 0; c < NK / 8; ++c) {
    const float2 mk = *reinterpret_cast<const float2*>(sMask + 8 * c + 2 * q4);
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      float& x = s[4 * c + 2 * h2];
      float& y = s[4 * c + 2 * h2 + 1];
      x = fmaf(x, ATTN_SCALE_LOG2, mk.x);
      y = fmaf(y, ATTN_SCALE_LOG2, mk.y);
      m[h2] = fmaxf(m[h2], fmaxf(x, y));
    }
  }
  float l[2] = {0.f, 0.f};
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    m[h2] = fmaxf(m[h2], __shfl_xor_sync(0xFFFFFFFFu, m[h2], 1));
    m[h2] = fmaxf(m[h2], __shfl_xor_sync(0xFFFFFFFFu, m[h2], 2));
  }
  const float e[2] = {m[0] == -INFINITY ? 0.f : m[0], m[1] == -INFINITY ? 0.f : m[1]};   // fully masked row guard
  uint32_t pk[NK / 4];
#pragma unroll
  for (int c = 0; c < NK / 8; ++c) {
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      float px = ex2_approx(s[4 * c + 2 * h2] - e[h2]);
      float py = ex2_approx(s[4 * c + 2 * h2 + 1] - e[h2]);
      l[h2] += px + py;
      if (DROP) {
        // attention-probability dropout: the row sum keeps the un-dropped value, only the P V operand is masked
        float m0, m1;
        drop.mul2((uint32_t)(prob * S + qb * 64 + lrow + 8 * h2), (uint32_t)(8 * c + 2 * q4), m0, m1);
        px *= m0; py *= m1;
      }
      pk[2 * c + h2] = pack_bf16x2(px, py);
    }
  }
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    l[h2] += __shfl_xor_sync(0xFFFFFFFFu, l[h2], 1);
    l[h2] += __shfl_xor_sync(0xFFFFFFFFu, l[h2], 2);
  }

  // O = P V: k16 step j takes accumulator columns 16j .. 16j+15 as the A fragment
  float o[32];
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < NK / 16; ++j) {
    const uint32_t a[4] = {pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]};
    wgmma_m64n64_rs_bf16<1>(o, a, desc_mn(sV) + j * KSTEP_MN, j > 0);
  }
  wgmma_commit();
  wgmma_wait<0>();

#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = qb * 64 + lrow + 8 * h2;
    if (row >= S) continue;
    if (lse_out != nullptr && q4 == 0) lse_out[(long long)prob * S + row] = m[h2] * ATTN_LN2 + __logf(l[h2]);
    const float inv = l[h2] > 0.f ? 1.f / l[h2] : 0.f;
    bf16* dst = ctx + ((long long)seq * S + row) * H + h * 64;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      *reinterpret_cast<uint32_t*>(dst + 8 * c + 2 * q4) = pack_bf16x2(o[4 * c + 2 * h2] * inv, o[4 * c + 2 * h2 + 1] * inv);
  }
}

// ------------------------------------------------------------------------------------------ backward, S <= 128
// Sums v over the 8 lanes of a warp that share lane & 3 (the rows of a wgmma accumulator fragment), reduce-scatter
// style: v[2c + e] belongs to column 8c + 2 (lane & 3) + e, and lane g * 4 + q4 returns the sums of columns
// 8g + 2 q4 + {0, 1}.  14 shuffles instead of 48, in a fixed order.
__device__ __forceinline__ float2 rowlane_sum16(const float (&v)[16], int lane) {
  const bool b2 = lane & 16, b1 = lane & 8, b0 = lane & 4;
  float w[8], x[4], y[2];
#pragma unroll
  for (int j = 0; j < 8; ++j) w[j] = (b2 ? v[8 + j] : v[j]) + __shfl_xor_sync(0xFFFFFFFFu, b2 ? v[j] : v[8 + j], 16);
#pragma unroll
  for (int j = 0; j < 4; ++j) x[j] = (b1 ? w[4 + j] : w[j]) + __shfl_xor_sync(0xFFFFFFFFu, b1 ? w[j] : w[4 + j], 8);
#pragma unroll
  for (int j = 0; j < 2; ++j) y[j] = (b0 ? x[2 + j] : x[j]) + __shfl_xor_sync(0xFFFFFFFFu, b0 ? x[j] : x[2 + j], 4);
  return make_float2(y[0], y[1]);
}

// Writes the 16 columns this thread holds of accumulator rows row0 and row0 + 8 (bf16, only rows < S) to dst + row * ld
// and, when sums is set, adds the bf16-rounded values' column sums over the warp's 16 rows into sbias[64].
__device__ __forceinline__ void store_rows_colsum(const float (&acc)[32], bf16* dst, long long ld, int row0, int S,
                                                  int q4, int lane, bool sums, float* sbias) {
  float cs[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) cs[i] = 0.f;
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = row0 + 8 * h2;
    if (row >= S) continue;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const uint32_t u = pack_bf16x2(acc[4 * c + 2 * h2], acc[4 * c + 2 * h2 + 1]);
      *reinterpret_cast<uint32_t*>(dst + row * ld + 8 * c + 2 * q4) = u;
      const float2 f = unpack_bf16x2(u);
      cs[2 * c] += f.x;
      cs[2 * c + 1] += f.y;
    }
  }
  if (sums) {
    const float2 t = rowlane_sum16(cs, lane);
    float2* p = reinterpret_cast<float2*>(sbias + 8 * (lane >> 2) + 2 * q4);
    *p = make_float2(p->x + t.x, p->y + t.y);
  }
}

// smem: 2 x (Q | dO | K | V, [NK][64] bf16 each) | P~ and dS staging ([NK / 64 slabs][NK queries][64 keys] bf16 each)
//       | key mask [2][NK] | column sums [warps][192] | 2 barriers
template <int NK>
constexpr int bwd_short_smem() { return 8 * NK * 128 + 2 * NK * NK * 2 + 2 * NK * 4 + (NK / 16) * 192 * 4 + 16 + 1024; }

template <int NK, bool DROP>
__global__ void __launch_bounds__(2 * NK, NK == 64 ? 2 : 1)
attn_bwd_short_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                      const int32_t* __restrict__ attn_mask, const float* __restrict__ lse_in, bf16* __restrict__ dqkv,
                      float* __restrict__ dbias, int nseq, int S, int heads, Drop drop) {
  constexpr int NT = 2 * NK, NWARP = NT / 32, OPS = NK * 128, BUF = 4 * OPS, STG = NK * NK * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sP = smem + 2 * BUF;                                   // slab kb at kb * NK * 128
  uint8_t* sdS = sP + STG;
  float* sMask = reinterpret_cast<float*>(sdS + STG);             // [2][NK]
  float* sBias = sMask + 2 * NK;                                  // [NWARP][192]: dQ | dK | dV columns of head h
  uint64_t* bar = reinterpret_cast<uint64_t*>(sBias + NWARP * 192);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3;
  const int wg = warp >> 2;                                       // query block (phase 1) and key block (phase 2)
  const int lrow = (warp & 3) * 16 + (lane >> 2);                 // accumulator row in the block (+8 for h2 = 1)
  // CTA -> (head, first sequence, sequence stride): one head per CTA keeps its bias columns to 192
  const int h = blockIdx.x % heads, stride = gridDim.x / heads;
  const int H = heads * 64;
  const bool sums = dbias != nullptr;

  auto load = [&](int seq, int b) {
    uint8_t* buf = smem + b * BUF;
    mbar_arrive_expect_tx(&bar[b], BUF);
    tma_load_3d(buf, &tm_qkv, &bar[b], h * 64, 0, seq);
    tma_load_3d(buf + OPS, &tm_do, &bar[b], h * 64, 0, seq);
    tma_load_3d(buf + 2 * OPS, &tm_qkv, &bar[b], H + h * 64, 0, seq);
    tma_load_3d(buf + 3 * OPS, &tm_qkv, &bar[b], 2 * H + h * 64, 0, seq);
  };
  auto fill_mask = [&](int seq, int b) {
    if (tid < NK) {
      const bool keep = tid < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + tid] != 0);
      sMask[b * NK + tid] = keep ? 0.f : -INFINITY;
    }
  };

  const int seq0 = blockIdx.x / heads;
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  for (int i = tid; i < NWARP * 192; i += NT) sBias[i] = 0.f;
  if (seq0 < nseq) fill_mask(seq0, 0);
  __syncthreads();
  if (tid == 0 && seq0 < nseq) load(seq0, 0);

  int it = 0;
  for (int seq = seq0; seq < nseq; seq += stride, ++it) {
    const int b = it & 1;
    const int prob = seq * heads + h;
    // the other buffer and mask slot were last read in the previous iteration, which ended with a CTA barrier
    if (seq + stride < nseq) {
      if (tid == 0) load(seq + stride, b ^ 1);
      fill_mask(seq + stride, b ^ 1);
    }
    const uint8_t* sQ = smem + b * BUF;
    const uint8_t* sdO = sQ + OPS;
    const uint8_t* sK = sQ + 2 * OPS;
    const uint8_t* sV = sQ + 3 * OPS;
    const float* mask = sMask + b * NK;
    const int r0 = wg * 64 + lrow;                                // query rows r0, r0 + 8
    float ls[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2)                                // rows >= S: lse = +inf, so P = 0
      ls[h2] = r0 + 8 * h2 < S ? lse_in[(long long)prob * S + r0 + 8 * h2] * ATTN_LOG2E : INFINITY;
    mbar_wait(&bar[b], (it >> 1) & 1);

    // ---- phase 1: S = Q K^T, dP = dO V^T for this warpgroup's 64 queries x NK keys
    float s[NK / 2], dp[NK / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) mma_ss<NK>(s, desc_k(sQ + wg * 8192) + k * KSTEP_K, desc_k(sK) + k * KSTEP_K, k > 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) mma_ss<NK>(dp, desc_k(sdO + wg * 8192) + k * KSTEP_K, desc_k(sV) + k * KSTEP_K, k > 0);
    wgmma_commit();
    wgmma_wait<0>();

    // P (kept in s), the dropout-masked dP (kept in dp), P~ = P m staged, D = sum P~ dP; the multipliers are the
    // forward's: row prob * S + query, column pair 8c + 2 q4
    float D[2] = {0.f, 0.f};
#pragma unroll
    for (int c = 0; c < NK / 8; ++c) {
      const float2 mk = *reinterpret_cast<const float2*>(mask + 8 * c + 2 * q4);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int i = 4 * c + 2 * h2, r = r0 + 8 * h2;
        const float px = ex2_approx(fmaf(s[i], ATTN_SCALE_LOG2, mk.x) - ls[h2]);
        const float py = ex2_approx(fmaf(s[i + 1], ATTN_SCALE_LOG2, mk.y) - ls[h2]);
        float m0 = 1.f, m1 = 1.f;
        if (DROP) {
          drop.mul2((uint32_t)(prob * S + r), (uint32_t)(8 * c + 2 * q4), m0, m1);
          dp[i] *= m0;
          dp[i + 1] *= m1;
        }
        s[i] = px;
        s[i + 1] = py;
        D[h2] = fmaf(px, dp[i], fmaf(py, dp[i + 1], D[h2]));
        *reinterpret_cast<uint32_t*>(sP + (c >> 3) * (NK * 128) + r * 128 + (((c & 7) ^ (r & 7)) << 4) + q4 * 4) =
            pack_bf16x2(px * m0, py * m1);
      }
    }
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      D[h2] += __shfl_xor_sync(0xFFFFFFFFu, D[h2], 1);
      D[h2] += __shfl_xor_sync(0xFFFFFFFFu, D[h2], 2);
    }
    uint32_t ds[NK / 4];
#pragma unroll
    for (int c = 0; c < NK / 8; ++c) {
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int i = 4 * c + 2 * h2, r = r0 + 8 * h2;
        ds[2 * c + h2] = pack_bf16x2(s[i] * (dp[i] - D[h2]) * 0.125f, s[i + 1] * (dp[i + 1] - D[h2]) * 0.125f);
        *reinterpret_cast<uint32_t*>(sdS + (c >> 3) * (NK * 128) + r * 128 + (((c & 7) ^ (r & 7)) << 4) + q4 * 4) =
            ds[2 * c + h2];
      }
    }
    // dQ = dS K: dS straight from registers, K read in place as the MN-major B
    float dq[32];
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < NK / 16; ++j) {
      const uint32_t a[4] = {ds[4 * j], ds[4 * j + 1], ds[4 * j + 2], ds[4 * j + 3]};
      wgmma_m64n64_rs_bf16<1>(dq, a, desc_mn(sK) + j * KSTEP_MN, j > 0);
    }
    wgmma_commit();
    fence_proxy_async_smem();
    __syncthreads();                                              // both warpgroups' P~ and dS are staged

    // ---- phase 2: dV = P~^T dO and dK = dS^T Q for keys 64 wg .. 64 wg + 63, reduced over all NK queries
    float dv[32], dk[32];
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < NK / 16; ++j)
      wgmma_m64n64_ss_bf16<1, 1>(dv, desc_mn(sP + wg * (NK * 128)) + j * KSTEP_MN, desc_mn(sdO) + j * KSTEP_MN, j > 0);
#pragma unroll
    for (int j = 0; j < NK / 16; ++j)
      wgmma_m64n64_ss_bf16<1, 1>(dk, desc_mn(sdS + wg * (NK * 128)) + j * KSTEP_MN, desc_mn(sQ) + j * KSTEP_MN, j > 0);
    wgmma_commit();
    bf16* out = dqkv + (long long)seq * S * 3 * H + h * 64;
    wgmma_wait<1>();
    store_rows_colsum(dq, out, 3LL * H, wg * 64 + lrow, S, q4, lane, sums, sBias + warp * 192);
    wgmma_wait<0>();
    store_rows_colsum(dk, out + H, 3LL * H, wg * 64 + lrow, S, q4, lane, sums, sBias + warp * 192 + 64);
    store_rows_colsum(dv, out + 2 * H, 3LL * H, wg * 64 + lrow, S, q4, lane, sums, sBias + warp * 192 + 128);
    __syncthreads();                                              // staging, this buffer and its mask slot are free
  }
  if (sums && it > 0) {
    for (int t = tid; t < 192; t += NT) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < NWARP; ++w) v += sBias[w * 192 + t];
      atomicAdd(dbias + (t >> 6) * H + h * 64 + (t & 63), v);
    }
  }
}

// ------------------------------------------------------------------------------------------ backward, 128 < S <= 256
// smem: Q | dO | K | V ([NK][64] bf16 each) | dQ accumulator [NK][64] fp32 | dS^T staging [2 warpgroups][64][64] bf16
//       | lse2 [NK] | D [NK] | key mask [NK] | barrier
template <int NK>
constexpr int bwd_smem() { return 4 * NK * 128 + NK * 256 + 2 * 8192 + 3 * NK * 4 + 16 + 1024; }

template <int NK, bool DROP>
__global__ void __launch_bounds__(256, 1)
attn_bwd_wg_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                   const int32_t* __restrict__ attn_mask, const float* __restrict__ lse_in, bf16* __restrict__ dqkv, int S,
                   int heads, Drop drop) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sdO = sQ + NK * 128;
  uint8_t* sK = sdO + NK * 128;
  uint8_t* sV = sK + NK * 128;
  float* sdQ = reinterpret_cast<float*>(sV + NK * 128);          // [NK][64]
  uint8_t* sStage = reinterpret_cast<uint8_t*>(sdQ + NK * 64);   // [2][64][64] bf16, swizzled
  float* sLse = reinterpret_cast<float*>(sStage + 2 * 8192);     // [NK] lse * log2(e), +inf beyond S
  float* sD = sLse + NK;                                         // [NK]
  float* sMask = sD + NK;                                        // [NK]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sMask + NK);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3;
  const int wg = warp >> 2;
  const int prob = blockIdx.x, seq = prob / heads, h = prob - seq * heads;
  const int H = heads * 64;
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 4 * NK * 128);
    tma_load_3d(sQ, &tm_qkv, bar, h * 64, 0, seq);
    tma_load_3d(sdO, &tm_do, bar, h * 64, 0, seq);
    tma_load_3d(sK, &tm_qkv, bar, H + h * 64, 0, seq);
    tma_load_3d(sV, &tm_qkv, bar, 2 * H + h * 64, 0, seq);
  }
  for (int i = tid; i < NK * 64; i += 256) sdQ[i] = 0.f;
  for (int j = tid; j < NK; j += 256) {
    const bool keep = j < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + j] != 0);
    sMask[j] = keep ? 0.f : -INFINITY;
    sLse[j] = j < S ? lse_in[(long long)prob * S + j] * ATTN_LOG2E : INFINITY;   // rows beyond S: P = 0
    sD[j] = 0.f;
  }
  __syncthreads();
  mbar_wait(bar, 0);

  const int nblk = (S + 63) / 64;
  const int lrow = (warp & 3) * 16 + (lane >> 2);     // accumulator row inside a 64-row block (+8 for h2 = 1)
  // D_i = sum_j P_ij dP_ij in fp32 (dropout: the masked P and dP): warpgroup wg takes query blocks wg, wg + 2, ...
  // and walks the keys in 64-wide chunks (rows = queries here, so key pairs are the dropout hash's column pairs)
  for (int qb = wg; qb < nblk; qb += 2) {
    float Dr[2] = {0.f, 0.f};
    const float ls[2] = {sLse[qb * 64 + lrow], sLse[qb * 64 + lrow + 8]};
    for (int kc = 0; kc < nblk; ++kc) {
      float sc[32], dp[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(sc, desc_k(sQ + qb * 8192) + k * KSTEP_K, desc_k(sK + kc * 8192) + k * KSTEP_K, k > 0);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(dp, desc_k(sdO + qb * 8192) + k * KSTEP_K, desc_k(sV + kc * 8192) + k * KSTEP_K, k > 0);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int kcol = kc * 64 + 8 * c + 2 * q4;
        const float2 mk = *reinterpret_cast<const float2*>(sMask + kcol);
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int i = 4 * c + 2 * h2;
          float px = ex2_approx(fmaf(sc[i], ATTN_SCALE_LOG2, mk.x) - ls[h2]);
          float py = ex2_approx(fmaf(sc[i + 1], ATTN_SCALE_LOG2, mk.y) - ls[h2]);
          if (DROP) {
            float m0, m1;
            drop.mul2((uint32_t)(prob * S + qb * 64 + lrow + 8 * h2), (uint32_t)kcol, m0, m1);
            px *= m0; py *= m1;
          }
          Dr[h2] = fmaf(px, dp[i], fmaf(py, dp[i + 1], Dr[h2]));
        }
      }
    }
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      Dr[h2] += __shfl_xor_sync(0xFFFFFFFFu, Dr[h2], 1);
      Dr[h2] += __shfl_xor_sync(0xFFFFFFFFu, Dr[h2], 2);
      if (q4 == 0) sD[qb * 64 + lrow + 8 * h2] = Dr[h2];
    }
  }
  __syncthreads();

  uint8_t* stage = sStage + wg * 8192;
  for (int kb = wg; kb < nblk; kb += 2) {
    float dv[32], dk[32];
    const uint64_t dK_kb = desc_k(sK + kb * 64 * 128), dV_kb = desc_k(sV + kb * 64 * 128);
    const float mk[2] = {sMask[kb * 64 + lrow], sMask[kb * 64 + lrow + 8]};
    for (int qb = 0; qb < nblk; ++qb) {
      float st[32], dpt[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(st, dK_kb + k * KSTEP_K, desc_k(sQ + qb * 8192) + k * KSTEP_K, k > 0);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(dpt, dV_kb + k * KSTEP_K, desc_k(sdO + qb * 8192) + k * KSTEP_K, k > 0);
      wgmma_commit();
      wgmma_wait<0>();
      // element (key kr, query qc): P = exp2(s * scale + mask[kr] - lse2[qc]); dS = P (dP_m - D[qc]) / 8
      uint32_t pd[16], ds[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int qc = qb * 64 + 8 * c + 2 * q4;
        const float2 ls = *reinterpret_cast<const float2*>(sLse + qc);
        const float2 Dq = *reinterpret_cast<const float2*>(sD + qc);
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int i = 4 * c + 2 * h2;
          const float px = ex2_approx(fmaf(st[i], ATTN_SCALE_LOG2, mk[h2]) - ls.x);
          const float py = ex2_approx(fmaf(st[i + 1], ATTN_SCALE_LOG2, mk[h2]) - ls.y);
          float mx = 1.f, my = 1.f;
          if (DROP) {
            const uint32_t kr = (uint32_t)(kb * 64 + lrow + 8 * h2);
            mx = drop_one(drop, (uint32_t)(prob * S + qc), kr);
            my = drop_one(drop, (uint32_t)(prob * S + qc + 1), kr);
          }
          pd[2 * c + h2] = pack_bf16x2(px * mx, py * my);
          ds[2 * c + h2] = pack_bf16x2(px * fmaf(dpt[i], mx, -Dq.x) * 0.125f, py * fmaf(dpt[i + 1], my, -Dq.y) * 0.125f);
        }
      }
      // dS^T block -> staging tile [64 keys][64 queries] (128B swizzle), read back as the MN-major A of dQ = dS K
      named_bar_sync(1 + wg, 128);                     // the previous dQ MMA of this warpgroup has read the stage
#pragma unroll
      for (int c = 0; c < 8; ++c) {
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int r = lrow + 8 * h2;
          *reinterpret_cast<uint32_t*>(stage + r * 128 + ((c ^ (r & 7)) << 4) + q4 * 4) = ds[2 * c + h2];
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t a[4] = {pd[4 * j], pd[4 * j + 1], pd[4 * j + 2], pd[4 * j + 3]};
        wgmma_m64n64_rs_bf16<1>(dv, a, desc_mn(sdO + qb * 8192) + j * KSTEP_MN, qb > 0 || j > 0);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t a[4] = {ds[4 * j], ds[4 * j + 1], ds[4 * j + 2], ds[4 * j + 3]};
        wgmma_m64n64_rs_bf16<1>(dk, a, desc_mn(sQ + qb * 8192) + j * KSTEP_MN, qb > 0 || j > 0);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        wgmma_m64n64_ss_bf16<1, 1>(dq, desc_mn(stage) + j * KSTEP_MN, desc_mn(sK + kb * 8192) + j * KSTEP_MN, j > 0);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < 8; ++c) {
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          float* dst = sdQ + (qb * 64 + lrow + 8 * h2) * 64 + 8 * c + 2 * q4;
          atomicAdd(dst, dq[4 * c + 2 * h2]);
          atomicAdd(dst + 1, dq[4 * c + 2 * h2 + 1]);
        }
      }
    }
    // dK, dV of this key block
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      const int row = kb * 64 + lrow + 8 * h2;
      if (row >= S) continue;
      bf16* base = dqkv + ((long long)seq * S + row) * 3 * H + h * 64 + 2 * q4;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        *reinterpret_cast<uint32_t*>(base + H + 8 * c) = pack_bf16x2(dk[4 * c + 2 * h2], dk[4 * c + 2 * h2 + 1]);
        *reinterpret_cast<uint32_t*>(base + 2 * H + 8 * c) = pack_bf16x2(dv[4 * c + 2 * h2], dv[4 * c + 2 * h2 + 1]);
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < S * 32; i += 256) {
    const int r = i >> 5, c2 = (i & 31) * 2;
    *reinterpret_cast<uint32_t*>(dqkv + ((long long)seq * S + r) * 3 * H + h * 64 + c2) =
        pack_bf16x2(sdQ[r * 64 + c2], sdQ[r * 64 + c2 + 1]);
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------ host
int make_tmap3(CUtensorMap* out, const void* base, int nseq, int S, long long cols, int box_rows) {
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && cols % 8 == 0, "attention operand misaligned");
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)S, (cuuint64_t)nseq};
  const cuuint64_t strides[2] = {(cuuint64_t)cols * 2, (cuuint64_t)S * cols * 2};
  const cuuint32_t box[3] = {64u, (cuuint32_t)box_rows, 1u};
  return encode_tmap(out, "attention", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

namespace {

template <int NK>
int fwd_launch(const CUtensorMap& tq, const CUtensorMap& tkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq,
               int S, int heads, const Drop& drop, cudaStream_t stream) {
  constexpr int smem = fwd_smem<NK>();
  static bool attr = false;
  if (!attr) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_wg_kernel<NK, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_wg_kernel<NK, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const long long grid = (long long)((S + 63) / 64) * nseq * heads;
  DPRB_REQUIRE(grid < (1LL << 31), "attn_fwd: grid too large");
  if (drop.on()) attn_fwd_wg_kernel<NK, true><<<(unsigned)grid, 128, smem, stream>>>(tq, tkv, attn_mask, (bf16*)ctx, lse, S, heads, drop);
  else attn_fwd_wg_kernel<NK, false><<<(unsigned)grid, 128, smem, stream>>>(tq, tkv, attn_mask, (bf16*)ctx, lse, S, heads, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}

// 128 < S <= 256
int bwd_launch(const CUtensorMap& tq, const CUtensorMap& tdo, const int32_t* attn_mask, const float* lse, void* dqkv,
               int nseq, int S, int heads, const Drop& drop, cudaStream_t stream) {
  constexpr int smem = bwd_smem<256>();
  static_assert(smem <= 227 * 1024, "attention backward: shared memory budget exceeded");
  static bool attr = false;
  if (!attr) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_wg_kernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_wg_kernel<256, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const int grid = nseq * heads;
  if (drop.on())
    attn_bwd_wg_kernel<256, true><<<grid, 256, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, S, heads, drop);
  else
    attn_bwd_wg_kernel<256, false><<<grid, 256, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, S, heads, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}

// S <= 128: as many CTAs as fit on the device at once (a multiple of heads), each looping over sequences
template <int NK>
int bwd_short_launch(const CUtensorMap& tq, const CUtensorMap& tdo, const int32_t* attn_mask, const float* lse,
                     void* dqkv, float* dbias, int nseq, int S, int heads, const Drop& drop, cudaStream_t stream) {
  constexpr int smem = bwd_short_smem<NK>();
  static_assert(smem <= 227 * 1024, "attention backward: shared memory budget exceeded");
  static int per_sm = 0;
  if (per_sm == 0) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_short_kernel<NK, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_short_kernel<NK, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int n = 0;
    DPRB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_bwd_short_kernel<NK, true>, 2 * NK, smem));
    DPRB_REQUIRE(n > 0, "attn_bwd: the S <= %d kernel does not fit on an SM", NK);
    per_sm = n;
  }
  DPRB_NUM_SMS(sms);
  const int per_head = std::max(1, std::min(nseq, per_sm * sms / heads));
  const int grid = per_head * heads;
  if (drop.on())
    attn_bwd_short_kernel<NK, true><<<grid, 2 * NK, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, dbias, nseq,
                                                                    S, heads, drop);
  else
    attn_bwd_short_kernel<NK, false><<<grid, 2 * NK, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, dbias, nseq,
                                                                     S, heads, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int pad_keys(int S) { return S <= 64 ? 64 : (S <= 128 ? 128 : 256); }

}  // namespace

int attn_fwd_wg(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                float dropout_p, unsigned long long site_seed, cudaStream_t stream) {
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int H = heads * 64, NK = pad_keys(S);
  CUtensorMap tq, tkv;
  if (int rc = make_tmap3(&tq, qkv, nseq, S, 3LL * H, 64)) return rc;
  if (int rc = make_tmap3(&tkv, qkv, nseq, S, 3LL * H, NK)) return rc;
  if (NK == 64) return fwd_launch<64>(tq, tkv, attn_mask, ctx, lse, nseq, S, heads, drop, stream);
  if (NK == 128) return fwd_launch<128>(tq, tkv, attn_mask, ctx, lse, nseq, S, heads, drop, stream);
  return fwd_launch<256>(tq, tkv, attn_mask, ctx, lse, nseq, S, heads, drop, stream);
}

int attn_bwd_wg(const void* qkv, const int32_t* attn_mask, const float* lse, const void* dctx,
                void* dqkv, float* dbias, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                cudaStream_t stream) {
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int H = heads * 64, NK = pad_keys(S);
  DPRB_REQUIRE(lse != nullptr, "attn_bwd: lse from the forward is required");
  CUtensorMap tq, tdo;
  if (int rc = make_tmap3(&tq, qkv, nseq, S, 3LL * H, NK)) return rc;
  if (int rc = make_tmap3(&tdo, dctx, nseq, S, H, NK)) return rc;
  if (NK == 64) return bwd_short_launch<64>(tq, tdo, attn_mask, lse, dqkv, dbias, nseq, S, heads, drop, stream);
  if (NK == 128) return bwd_short_launch<128>(tq, tdo, attn_mask, lse, dqkv, dbias, nseq, S, heads, drop, stream);
  if (int rc = bwd_launch(tq, tdo, attn_mask, lse, dqkv, nseq, S, heads, drop, stream)) return rc;
  // the QKV bias gradient: column sums of the bf16 dQ / dK / dV
  return dbias != nullptr ? dprb_colsum_bf16(dqkv, 3LL * H, dbias, nseq * S, 3 * H, stream) : 0;
}

}  // namespace dprb
