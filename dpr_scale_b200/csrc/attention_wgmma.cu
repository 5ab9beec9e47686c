// Self-attention core on Hopper warpgroup MMA (wgmma) for head_dim 64 and S <= 256.
//
//   forward : one CTA (one warpgroup) = 64 query rows of one (sequence, head) problem.  Q, K, V arrive by TMA
//             (128B-swizzled); S = Q K^T (wgmma m64nNKk16, fp32 in registers) -> exact row softmax in registers
//             (a row lives in the 4 threads of a quad) -> P (bf16) stays in registers as the A operand of
//             O = P V (wgmma RS form, V read in place as an MN-major operand) -> O / l -> ctx.  LSE saved for backward.
//   backward: one CTA = one problem, two warpgroups.  Each warpgroup owns 64-key blocks and walks the query blocks:
//             S^T = K Q^T and dP^T = V dO^T (wgmma) -> P^T = exp2(S^T - lse), dS^T = P^T (dP^T - D) / 8 in registers
//             -> dV += P^T dO and dK += dS^T Q (RS form, accumulators stay in registers across query blocks)
//             -> dS^T staged in shared memory -> dQ_part = dS K (both operands MN-major) added into an fp32 dQ
//             accumulator in shared memory.  D_i = sum_j P_ij dP_ij is computed first, in fp32, by a row pass.
//
// Tiles are moved by TMA through 3-D tensor maps [nseq, S, columns]: rows >= S of a short sequence are zero-filled on
// load, so only stores need row predicates.
//
// Replaces BertSelfAttention.forward's scaled_dot_product_attention and its autograd backward.
#include "attention.cuh"
#include "dprb_internal.h"

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

// ------------------------------------------------------------------------------------------ backward
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

template <int NK>
int bwd_launch(const CUtensorMap& tq, const CUtensorMap& tdo, const int32_t* attn_mask, const float* lse, void* dqkv,
               int nseq, int S, int heads, const Drop& drop, cudaStream_t stream) {
  constexpr int smem = bwd_smem<NK>();
  static_assert(smem <= 227 * 1024, "attention backward: shared memory budget exceeded");
  static bool attr = false;
  if (!attr) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_wg_kernel<NK, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_wg_kernel<NK, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const int grid = nseq * heads;
  if (drop.on())
    attn_bwd_wg_kernel<NK, true><<<grid, 256, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, S, heads, drop);
  else
    attn_bwd_wg_kernel<NK, false><<<grid, 256, smem, stream>>>(tq, tdo, attn_mask, lse, (bf16*)dqkv, S, heads, drop);
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
                void* dqkv, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                cudaStream_t stream) {
  const Drop drop = drop_from_site(dropout_p, site_seed);
  const int H = heads * 64, NK = pad_keys(S);
  DPRB_REQUIRE(lse != nullptr, "attn_bwd: lse from the forward is required");
  CUtensorMap tq, tdo;
  if (int rc = make_tmap3(&tq, qkv, nseq, S, 3LL * H, NK)) return rc;
  if (int rc = make_tmap3(&tdo, dctx, nseq, S, H, NK)) return rc;
  if (NK == 64) return bwd_launch<64>(tq, tdo, attn_mask, lse, dqkv, nseq, S, heads, drop, stream);
  if (NK == 128) return bwd_launch<128>(tq, tdo, attn_mask, lse, dqkv, nseq, S, heads, drop, stream);
  return bwd_launch<256>(tq, tdo, attn_mask, lse, dqkv, nseq, S, heads, drop, stream);
}

}  // namespace dprb
