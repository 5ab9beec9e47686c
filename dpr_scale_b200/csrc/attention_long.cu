// Self-attention core on wgmma for head_dim 64 and 256 < S <= 512 (S <= 256 runs attention_wgmma.cu).
//
//   forward : one CTA = 128 query rows (two warpgroups of 64) of one (sequence, head) problem.  Q and the problem's
//             K / V arrive by TMA in 128-key blocks, one mbarrier per block, so the first block is being computed
//             while the others land.  Per key block: S = Q K^T (wgmma m64n128k16 SS) -> online softmax in the exp2
//             domain (running row max and sum, O rescaled when the max grows) -> P (bf16) stays in registers as the A
//             operand of O += P V (RS form, V read in place as an MN-major operand).  O / l -> ctx, lse in natural log.
//   backward: two kernels, no atomics and no workspace, so the result is deterministic.
//             dK/dV: one CTA = 128 keys (64 per warpgroup).  The tile's K / V are loaded once; Q and dO come in
//             64-row blocks (one mbarrier each).  S^T = K Q^T, dP^T = V dO^T -> P^T = exp2(S^T - lse),
//             dS^T = P^T (dP^T - D) / 8 -> dV += P^T dO, dK += dS^T Q (RS form, accumulators in registers).
//             dQ: one CTA = 128 query rows.  K / V come in 64-key blocks; S = Q K^T, dP = dO V^T -> dS in registers
//             -> dQ += dS K (RS form, K read as the MN-major operand).
//             D_i = sum_j P_ij dP_ij is taken as rowsum(dO_i * ctx_i) in fp32 (equal in exact arithmetic, dropout
//             included: ctx carries the applied mask), computed by each kernel for the rows it needs.
//
// Attention-probability dropout uses the same (row = prob * S + query, column = key) keys as the S <= 256 kernels, so
// dprb_dropout_mask(..., site 1) describes the applied mask bit for bit.  Keys j >= S and attn_mask == 0 get -inf.
// Tensor maps are the 3-D [nseq, S, columns] maps of make_tmap3: rows >= S are zero-filled on load.
#include "attention.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int LMAX = 512;          // longest sequence these kernels take
constexpr int TILE = 128;          // query rows (forward, dQ) or keys (dK/dV) per CTA: 64 per warpgroup
constexpr int FBK = 128;           // forward key block
constexpr int BBK = 64;            // backward key / query block

// forward smem: Q [128][64] | K [512][64] | V [512][64] bf16 | key mask [512] | barriers (Q + one per key block)
constexpr int fwd_long_smem() { return TILE * 128 + 2 * LMAX * 128 + LMAX * 4 + (1 + LMAX / FBK) * 8 + 1024; }
// dK/dV smem: K [128][64] | V [128][64] | Q [512][64] | dO [512][64] bf16 | lse2 [512] | D [512] | barriers
constexpr int dkdv_long_smem() { return 2 * TILE * 128 + 2 * LMAX * 128 + 2 * LMAX * 4 + (1 + LMAX / BBK) * 8 + 1024; }
// dQ smem: Q [128][64] | dO [128][64] | K [512][64] | V [512][64] bf16 | key mask [512] | lse2 [128] | D [128] | barriers
constexpr int dq_long_smem() {
  return 2 * TILE * 128 + 2 * LMAX * 128 + LMAX * 4 + 2 * TILE * 4 + (1 + LMAX / BBK) * 8 + 1024;
}
static_assert(fwd_long_smem() <= 227 * 1024, "long attention forward: shared memory budget exceeded");
static_assert(dkdv_long_smem() <= 227 * 1024, "long attention dK/dV: shared memory budget exceeded");
static_assert(dq_long_smem() <= 227 * 1024, "long attention dQ: shared memory budget exceeded");

// D_i = rowsum(dO_i * ctx_i) in fp32 and lse_i * log2(e) for rows r0 .. r0 + n - 1 of one problem (n a multiple of
// 32; rows >= S get D = 0, lse2 = +inf so that P = 0).  Eight threads per row, 16-byte loads; 256 threads.
__device__ __forceinline__ void rows_d_lse(const bf16* __restrict__ dctx, const bf16* __restrict__ ctx,
                                           const float* __restrict__ lse, float* sD, float* sLse, int r0, int n,
                                           int seq, int prob, int S, int H, int h, int tid) {
  const int seg = tid & 7;
  for (int r = tid >> 3; r < n; r += 32) {
    const int row = r0 + r;
    float acc = 0.f;
    if (row < S) {
      const long long off = ((long long)seq * S + row) * H + h * 64 + seg * 8;
      const uint4 a = *reinterpret_cast<const uint4*>(dctx + off);
      const uint4 b = *reinterpret_cast<const uint4*>(ctx + off);
      const uint32_t* pa = &a.x;
      const uint32_t* pb = &b.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 x = unpack_bf16x2(pa[k]), y = unpack_bf16x2(pb[k]);
        acc = fmaf(x.x, y.x, fmaf(x.y, y.y, acc));
      }
    }
    acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
    acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 2);
    acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 4);
    if (seg == 0) {
      sD[r] = acc;
      sLse[r] = row < S ? lse[(long long)prob * S + row] * ATTN_LOG2E : INFINITY;
    }
  }
}

// ------------------------------------------------------------------------------------------ forward
template <bool DROP>
__global__ void __launch_bounds__(256, 1)
attn_fwd_long_kernel(const __grid_constant__ CUtensorMap tm_qkv, const int32_t* __restrict__ attn_mask,
                     bf16* __restrict__ ctx, float* __restrict__ lse_out, int S, int heads, int ntiles, Drop drop) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = align1024(smem_raw);               // [128][64]
  uint8_t* sK = sQ + TILE * 128;                   // [512][64]
  uint8_t* sV = sK + LMAX * 128;                   // [512][64]
  float* sMask = reinterpret_cast<float*>(sV + LMAX * 128);   // [512]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sMask + LMAX);  // [0]: Q, [1 + kb]: key block kb

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3, wg = warp >> 2;
  const int prob = blockIdx.x / ntiles, qt = blockIdx.x - prob * ntiles;
  const int seq = prob / heads, h = prob - seq * heads, H = heads * 64;
  const int nkb = (S + FBK - 1) / FBK;
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv);
    for (int i = 0; i <= nkb; ++i) mbar_init(bar + i, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, TILE * 128);
    tma_load_3d(sQ, &tm_qkv, bar, h * 64, qt * TILE, seq);
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_arrive_expect_tx(bar + 1 + kb, 2 * FBK * 128);
      tma_load_3d(sK + kb * FBK * 128, &tm_qkv, bar + 1 + kb, H + h * 64, kb * FBK, seq);
      tma_load_3d(sV + kb * FBK * 128, &tm_qkv, bar + 1 + kb, 2 * H + h * 64, kb * FBK, seq);
    }
  }
  for (int j = tid; j < nkb * FBK; j += 256) {
    const bool keep = j < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + j] != 0);
    sMask[j] = keep ? 0.f : -INFINITY;
  }
  __syncthreads();
  mbar_wait(bar, 0);

  // this thread holds rows lrow (h2 = 0) and lrow + 8 (h2 = 1) of its warpgroup's 64, columns 8c + 2 q4 + {0, 1}
  const uint8_t* sQw = sQ + wg * 64 * 128;
  const int lrow = (warp & 3) * 16 + (lane >> 2);
  const int qrow0 = qt * TILE + wg * 64 + lrow;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;

  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(bar + 1 + kb, 0);
    const uint8_t* sKb = sK + kb * FBK * 128;
    float s[FBK / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n128_ss_bf16<0, 0>(s, desc_k(sQw) + k * KSTEP_K, desc_k(sKb) + k * KSTEP_K, k > 0);
    wgmma_commit();
    wgmma_wait<0>();

    float mb[2] = {m[0], m[1]};
#pragma unroll
    for (int c = 0; c < FBK / 8; ++c) {
      const float2 mk = *reinterpret_cast<const float2*>(sMask + kb * FBK + 8 * c + 2 * q4);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        float& x = s[4 * c + 2 * h2];
        float& y = s[4 * c + 2 * h2 + 1];
        x = fmaf(x, ATTN_SCALE_LOG2, mk.x);
        y = fmaf(y, ATTN_SCALE_LOG2, mk.y);
        mb[h2] = fmaxf(mb[h2], fmaxf(x, y));
      }
    }
    float e[2];
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      mb[h2] = fmaxf(mb[h2], __shfl_xor_sync(0xFFFFFFFFu, mb[h2], 1));
      mb[h2] = fmaxf(mb[h2], __shfl_xor_sync(0xFFFFFFFFu, mb[h2], 2));
      e[h2] = mb[h2] == -INFINITY ? 0.f : mb[h2];          // no unmasked key yet: keep exponents finite
      const float alpha = ex2_approx(m[h2] - e[h2]);       // 0 while the row had no unmasked key (l, O are 0)
      m[h2] = mb[h2];
      l[h2] *= alpha;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        o[4 * c + 2 * h2] *= alpha;
        o[4 * c + 2 * h2 + 1] *= alpha;
      }
    }
    uint32_t pk[FBK / 4];
#pragma unroll
    for (int c = 0; c < FBK / 8; ++c) {
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        float px = ex2_approx(s[4 * c + 2 * h2] - e[h2]);
        float py = ex2_approx(s[4 * c + 2 * h2 + 1] - e[h2]);
        l[h2] += px + py;
        if (DROP) {
          // the row sum keeps the un-dropped value, only the P V operand is masked
          float m0, m1;
          drop.mul2((uint32_t)(prob * S + qrow0 + 8 * h2), (uint32_t)(kb * FBK + 8 * c + 2 * q4), m0, m1);
          px *= m0; py *= m1;
        }
        pk[2 * c + h2] = pack_bf16x2(px, py);
      }
    }
    // O += P V: k16 step j takes accumulator columns 16j .. 16j+15 as the A fragment
    const uint8_t* sVb = sV + kb * FBK * 128;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < FBK / 16; ++j) {
      const uint32_t a[4] = {pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]};
      wgmma_m64n64_rs_bf16<1>(o, a, desc_mn(sVb) + j * KSTEP_MN, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }

#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    l[h2] += __shfl_xor_sync(0xFFFFFFFFu, l[h2], 1);
    l[h2] += __shfl_xor_sync(0xFFFFFFFFu, l[h2], 2);
    const int row = qrow0 + 8 * h2;
    if (row >= S) continue;
    if (lse_out != nullptr && q4 == 0) lse_out[(long long)prob * S + row] = m[h2] * ATTN_LN2 + __logf(l[h2]);
    const float inv = l[h2] > 0.f ? 1.f / l[h2] : 0.f;
    bf16* dst = ctx + ((long long)seq * S + row) * H + h * 64;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      *reinterpret_cast<uint32_t*>(dst + 8 * c + 2 * q4) = pack_bf16x2(o[4 * c + 2 * h2] * inv, o[4 * c + 2 * h2 + 1] * inv);
  }
}

// ------------------------------------------------------------------------------------------ backward: dK, dV
template <bool DROP>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dkdv_long_kernel(const __grid_constant__ CUtensorMap tm_qkv128, const __grid_constant__ CUtensorMap tm_qkv64,
                          const __grid_constant__ CUtensorMap tm_do64, const int32_t* __restrict__ attn_mask,
                          const bf16* __restrict__ ctx, const bf16* __restrict__ dctx, const float* __restrict__ lse_in,
                          bf16* __restrict__ dqkv, int S, int heads, int ntiles, Drop drop) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sK = align1024(smem_raw);               // [128][64] keys of this tile
  uint8_t* sV = sK + TILE * 128;                   // [128][64]
  uint8_t* sQ = sV + TILE * 128;                   // [512][64]
  uint8_t* sdO = sQ + LMAX * 128;                  // [512][64]
  float* sLse = reinterpret_cast<float*>(sdO + LMAX * 128);   // [512] lse * log2(e), +inf beyond S
  float* sD = sLse + LMAX;                                    // [512]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sD + LMAX);     // [0]: K/V, [1 + qb]: query block qb

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3, wg = warp >> 2;
  const int prob = blockIdx.x / ntiles, kt = blockIdx.x - prob * ntiles;
  const int seq = prob / heads, h = prob - seq * heads, H = heads * 64;
  const int nqb = (S + BBK - 1) / BBK;
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv128);
    tma_prefetch_desc(&tm_qkv64);
    tma_prefetch_desc(&tm_do64);
    for (int i = 0; i <= nqb; ++i) mbar_init(bar + i, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 2 * TILE * 128);
    tma_load_3d(sK, &tm_qkv128, bar, H + h * 64, kt * TILE, seq);
    tma_load_3d(sV, &tm_qkv128, bar, 2 * H + h * 64, kt * TILE, seq);
    for (int qb = 0; qb < nqb; ++qb) {
      mbar_arrive_expect_tx(bar + 1 + qb, 2 * BBK * 128);
      tma_load_3d(sQ + qb * BBK * 128, &tm_qkv64, bar + 1 + qb, h * 64, qb * BBK, seq);
      tma_load_3d(sdO + qb * BBK * 128, &tm_do64, bar + 1 + qb, h * 64, qb * BBK, seq);
    }
  }
  rows_d_lse(dctx, ctx, lse_in, sD, sLse, 0, nqb * BBK, seq, prob, S, H, h, tid);
  __syncthreads();
  mbar_wait(bar, 0);

  const int lrow = (warp & 3) * 16 + (lane >> 2);     // accumulator row inside the warpgroup's 64 keys (+8: h2 = 1)
  const int kr0 = kt * TILE + wg * 64 + lrow;
  float mk[2];
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int kr = kr0 + 8 * h2;
    const bool keep = kr < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + kr] != 0);
    mk[h2] = keep ? 0.f : -INFINITY;
  }
  const uint64_t dK = desc_k(sK + wg * 64 * 128), dV = desc_k(sV + wg * 64 * 128);
  float dv[32], dk[32];
  for (int qb = 0; qb < nqb; ++qb) {
    mbar_wait(bar + 1 + qb, 0);
    const uint8_t* sQb = sQ + qb * BBK * 128;
    const uint8_t* sdOb = sdO + qb * BBK * 128;
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(st, dK + k * KSTEP_K, desc_k(sQb) + k * KSTEP_K, k > 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(dpt, dV + k * KSTEP_K, desc_k(sdOb) + k * KSTEP_K, k > 0);
    wgmma_commit();
    wgmma_wait<0>();
    // element (key kr, query qc): P = exp2(s * scale + mask[kr] - lse2[qc]); dS = P (dP_m - D[qc]) / 8
    uint32_t pd[16], ds[16];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int qc = qb * BBK + 8 * c + 2 * q4;
      const float2 ls = *reinterpret_cast<const float2*>(sLse + qc);
      const float2 Dq = *reinterpret_cast<const float2*>(sD + qc);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int i = 4 * c + 2 * h2;
        const float px = ex2_approx(fmaf(st[i], ATTN_SCALE_LOG2, mk[h2]) - ls.x);
        const float py = ex2_approx(fmaf(st[i + 1], ATTN_SCALE_LOG2, mk[h2]) - ls.y);
        float mx = 1.f, my = 1.f;
        if (DROP) {
          const uint32_t kr = (uint32_t)(kr0 + 8 * h2);
          mx = drop_one(drop, (uint32_t)(prob * S + qc), kr);
          my = drop_one(drop, (uint32_t)(prob * S + qc + 1), kr);
        }
        pd[2 * c + h2] = pack_bf16x2(px * mx, py * my);
        ds[2 * c + h2] = pack_bf16x2(px * fmaf(dpt[i], mx, -Dq.x) * 0.125f, py * fmaf(dpt[i + 1], my, -Dq.y) * 0.125f);
      }
    }
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t a[4] = {pd[4 * j], pd[4 * j + 1], pd[4 * j + 2], pd[4 * j + 3]};
      wgmma_m64n64_rs_bf16<1>(dv, a, desc_mn(sdOb) + j * KSTEP_MN, qb > 0 || j > 0);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t a[4] = {ds[4 * j], ds[4 * j + 1], ds[4 * j + 2], ds[4 * j + 3]};
      wgmma_m64n64_rs_bf16<1>(dk, a, desc_mn(sQb) + j * KSTEP_MN, qb > 0 || j > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = kr0 + 8 * h2;
    if (row >= S) continue;
    bf16* base = dqkv + ((long long)seq * S + row) * 3 * H + h * 64 + 2 * q4;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      *reinterpret_cast<uint32_t*>(base + H + 8 * c) = pack_bf16x2(dk[4 * c + 2 * h2], dk[4 * c + 2 * h2 + 1]);
      *reinterpret_cast<uint32_t*>(base + 2 * H + 8 * c) = pack_bf16x2(dv[4 * c + 2 * h2], dv[4 * c + 2 * h2 + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------ backward: dQ
template <bool DROP>
__global__ void __launch_bounds__(256, 1)
attn_bwd_dq_long_kernel(const __grid_constant__ CUtensorMap tm_qkv128, const __grid_constant__ CUtensorMap tm_qkv64,
                        const __grid_constant__ CUtensorMap tm_do128, const int32_t* __restrict__ attn_mask,
                        const bf16* __restrict__ ctx, const bf16* __restrict__ dctx, const float* __restrict__ lse_in,
                        bf16* __restrict__ dqkv, int S, int heads, int ntiles, Drop drop) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = align1024(smem_raw);               // [128][64] query rows of this tile
  uint8_t* sdO = sQ + TILE * 128;                  // [128][64]
  uint8_t* sK = sdO + TILE * 128;                  // [512][64]
  uint8_t* sV = sK + LMAX * 128;                   // [512][64]
  float* sMask = reinterpret_cast<float*>(sV + LMAX * 128);   // [512]
  float* sLse = sMask + LMAX;                                 // [128]
  float* sD = sLse + TILE;                                    // [128]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sD + TILE);     // [0]: Q/dO, [1 + kb]: key block kb

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3, wg = warp >> 2;
  const int prob = blockIdx.x / ntiles, qt = blockIdx.x - prob * ntiles;
  const int seq = prob / heads, h = prob - seq * heads, H = heads * 64;
  const int nkb = (S + BBK - 1) / BBK;
  if (tid == 0) {
    tma_prefetch_desc(&tm_qkv128);
    tma_prefetch_desc(&tm_qkv64);
    tma_prefetch_desc(&tm_do128);
    for (int i = 0; i <= nkb; ++i) mbar_init(bar + i, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 2 * TILE * 128);
    tma_load_3d(sQ, &tm_qkv128, bar, h * 64, qt * TILE, seq);
    tma_load_3d(sdO, &tm_do128, bar, h * 64, qt * TILE, seq);
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_arrive_expect_tx(bar + 1 + kb, 2 * BBK * 128);
      tma_load_3d(sK + kb * BBK * 128, &tm_qkv64, bar + 1 + kb, H + h * 64, kb * BBK, seq);
      tma_load_3d(sV + kb * BBK * 128, &tm_qkv64, bar + 1 + kb, 2 * H + h * 64, kb * BBK, seq);
    }
  }
  for (int j = tid; j < nkb * BBK; j += 256) {
    const bool keep = j < S && (attn_mask == nullptr || attn_mask[(long long)seq * S + j] != 0);
    sMask[j] = keep ? 0.f : -INFINITY;
  }
  rows_d_lse(dctx, ctx, lse_in, sD, sLse, qt * TILE, TILE, seq, prob, S, H, h, tid);
  __syncthreads();
  mbar_wait(bar, 0);

  const int lrow = (warp & 3) * 16 + (lane >> 2);
  const int qrow0 = qt * TILE + wg * 64 + lrow;
  const float ls[2] = {sLse[wg * 64 + lrow], sLse[wg * 64 + lrow + 8]};
  const float Dq[2] = {sD[wg * 64 + lrow], sD[wg * 64 + lrow + 8]};
  const uint64_t dQw = desc_k(sQ + wg * 64 * 128), ddOw = desc_k(sdO + wg * 64 * 128);
  float dq[32];
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(bar + 1 + kb, 0);
    const uint8_t* sKb = sK + kb * BBK * 128;
    const uint8_t* sVb = sV + kb * BBK * 128;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(s, dQw + k * KSTEP_K, desc_k(sKb) + k * KSTEP_K, k > 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64_ss_bf16<0, 0>(dp, ddOw + k * KSTEP_K, desc_k(sVb) + k * KSTEP_K, k > 0);
    wgmma_commit();
    wgmma_wait<0>();
    // element (query qrow, key kcol): P = exp2(s * scale + mask[kcol] - lse2[qrow]); dS = P (dP_m - D[qrow]) / 8
    uint32_t ds[16];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int kcol = kb * BBK + 8 * c + 2 * q4;
      const float2 mk = *reinterpret_cast<const float2*>(sMask + kcol);
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int i = 4 * c + 2 * h2;
        const float px = ex2_approx(fmaf(s[i], ATTN_SCALE_LOG2, mk.x) - ls[h2]);
        const float py = ex2_approx(fmaf(s[i + 1], ATTN_SCALE_LOG2, mk.y) - ls[h2]);
        float mx = 1.f, my = 1.f;
        if (DROP) drop.mul2((uint32_t)(prob * S + qrow0 + 8 * h2), (uint32_t)kcol, mx, my);
        ds[2 * c + h2] = pack_bf16x2(px * fmaf(dp[i], mx, -Dq[h2]) * 0.125f, py * fmaf(dp[i + 1], my, -Dq[h2]) * 0.125f);
      }
    }
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t a[4] = {ds[4 * j], ds[4 * j + 1], ds[4 * j + 2], ds[4 * j + 3]};
      wgmma_m64n64_rs_bf16<1>(dq, a, desc_mn(sKb) + j * KSTEP_MN, kb > 0 || j > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int row = qrow0 + 8 * h2;
    if (row >= S) continue;
    bf16* base = dqkv + ((long long)seq * S + row) * 3 * H + h * 64 + 2 * q4;
#pragma unroll
    for (int c = 0; c < 8; ++c)
      *reinterpret_cast<uint32_t*>(base + 8 * c) = pack_bf16x2(dq[4 * c + 2 * h2], dq[4 * c + 2 * h2 + 1]);
  }
}

template <typename K>
int set_smem(K kernel, int bytes) {
  DPRB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------ host
int attn_fwd_long(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                  float dropout_p, unsigned long long site_seed, cudaStream_t stream) {
  DPRB_REQUIRE(S > 0 && S <= LMAX, "attn_fwd_long: sequence length %d unsupported", S);
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int H = heads * 64;
  CUtensorMap tm;
  if (int rc = make_tmap3(&tm, qkv, nseq, S, 3LL * H, TILE)) return rc;
  constexpr int smem = fwd_long_smem();
  static bool attr = false;
  if (!attr) {
    if (int rc = set_smem(attn_fwd_long_kernel<false>, smem)) return rc;
    if (int rc = set_smem(attn_fwd_long_kernel<true>, smem)) return rc;
    attr = true;
  }
  const int ntiles = (S + TILE - 1) / TILE;
  const long long grid = (long long)ntiles * nseq * heads;
  DPRB_REQUIRE(grid < (1LL << 31), "attn_fwd_long: grid too large");
  if (drop.on())
    attn_fwd_long_kernel<true><<<(unsigned)grid, 256, smem, stream>>>(tm, attn_mask, (bf16*)ctx, lse, S, heads, ntiles, drop);
  else
    attn_fwd_long_kernel<false><<<(unsigned)grid, 256, smem, stream>>>(tm, attn_mask, (bf16*)ctx, lse, S, heads, ntiles, drop);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int attn_bwd_long(const void* qkv, const int32_t* attn_mask, const void* ctx, const float* lse, const void* dctx,
                  void* dqkv, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                  cudaStream_t stream) {
  DPRB_REQUIRE(S > 0 && S <= LMAX, "attn_bwd_long: sequence length %d unsupported", S);
  DPRB_REQUIRE(lse != nullptr && ctx != nullptr, "attn_bwd: lse and ctx from the forward are required");
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(ctx) & 15) == 0 && (reinterpret_cast<uintptr_t>(dctx) & 15) == 0,
               "attn_bwd: ctx / dctx misaligned");
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int H = heads * 64;
  CUtensorMap tq128, tq64, tdo128, tdo64;
  if (int rc = make_tmap3(&tq128, qkv, nseq, S, 3LL * H, TILE)) return rc;
  if (int rc = make_tmap3(&tq64, qkv, nseq, S, 3LL * H, BBK)) return rc;
  if (int rc = make_tmap3(&tdo128, dctx, nseq, S, H, TILE)) return rc;
  if (int rc = make_tmap3(&tdo64, dctx, nseq, S, H, BBK)) return rc;
  constexpr int smem_kv = dkdv_long_smem(), smem_q = dq_long_smem();
  static bool attr = false;
  if (!attr) {
    if (int rc = set_smem(attn_bwd_dkdv_long_kernel<false>, smem_kv)) return rc;
    if (int rc = set_smem(attn_bwd_dkdv_long_kernel<true>, smem_kv)) return rc;
    if (int rc = set_smem(attn_bwd_dq_long_kernel<false>, smem_q)) return rc;
    if (int rc = set_smem(attn_bwd_dq_long_kernel<true>, smem_q)) return rc;
    attr = true;
  }
  const int ntiles = (S + TILE - 1) / TILE;
  const long long grid = (long long)ntiles * nseq * heads;
  DPRB_REQUIRE(grid < (1LL << 31), "attn_bwd_long: grid too large");
  const bf16 *c = (const bf16*)ctx, *dc = (const bf16*)dctx;
  bf16* d = (bf16*)dqkv;
  if (drop.on()) {
    attn_bwd_dkdv_long_kernel<true><<<(unsigned)grid, 256, smem_kv, stream>>>(tq128, tq64, tdo64, attn_mask, c, dc, lse, d, S, heads, ntiles, drop);
    DPRB_LAUNCH_CHECK();
    attn_bwd_dq_long_kernel<true><<<(unsigned)grid, 256, smem_q, stream>>>(tq128, tq64, tdo128, attn_mask, c, dc, lse, d, S, heads, ntiles, drop);
  } else {
    attn_bwd_dkdv_long_kernel<false><<<(unsigned)grid, 256, smem_kv, stream>>>(tq128, tq64, tdo64, attn_mask, c, dc, lse, d, S, heads, ntiles, drop);
    DPRB_LAUNCH_CHECK();
    attn_bwd_dq_long_kernel<false><<<(unsigned)grid, 256, smem_q, stream>>>(tq128, tq64, tdo128, attn_mask, c, dc, lse, d, S, heads, ntiles, drop);
  }
  DPRB_LAUNCH_CHECK();
  return 0;
}

}  // namespace dprb
