// bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring (mbarrier pipeline) -> wgmma (fp32 accumulators in
// registers) -> epilogue with the fused bias / bias+GELU / bias+residual / dGELU / fp32 split-K accumulate variants
// the encoder needs.
//
// Persistent: one CTA per SM walks the work units (output tile, K split) in a static stride order.  A unit is a
// 128x256 tile: warpgroups 1 and 2 own rows [0, 64) and [64, 128) (wgmma m64n256k16, 128 fp32 accumulators per
// thread), warpgroup 0 is the TMA producer (one thread issues, setmaxnreg hands its registers to the consumers).  The
// 3-stage ring of 48 KB runs across unit boundaries, so the producer loads the next unit's first k-blocks while the
// consumers run the current unit's epilogue.  16-bit outputs go through a per-warpgroup staging slab in shared memory
// laid out as the TMA box (four 64-column, 128B-swizzled subtiles): the fragment-layout results are written there and
// one thread issues TMA stores, so the warpgroup goes straight back to the next unit's MMAs while the tile drains.  The
// aux operand (residual, gelu'(pre) or pre-activation) is TMA-loaded into the same slab by the producer during the
// unit's mainloop, once the previous unit's stores have read it.  fp32 outputs (split-K partial sums) stay
// fragment-layout red.global.add.v2.f32 / st.global straight from the registers.
//
// Replaces, on the reference path, every torch.nn.Linear call inside HF BertLayer (QKV, attention output,
// intermediate, output) and their autograd backward (dgrad / wgrad).
//
// D[M,N] = epi( sum_k A(m,k) * B(n,k) ).  Each operand may be K-major (row = MN index, K contiguous)
// or MN-major (row = K index, MN contiguous); the latter lets dgrad read W[N_out,K_in] and wgrad
// read dY[T,N_out] / X[T,K_in] in place, with no transposed copies.
#include <cstdlib>
#include <vector>
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int STAGES = 3;
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB
constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 2;   // 32 KB
constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
constexpr int NUM_CONSUMERS = 2;                      // warpgroups
constexpr int NUM_THREADS = (NUM_CONSUMERS + 1) * 128; // + the producer warpgroup
constexpr int WG_ROWS = BLOCK_M / NUM_CONSUMERS;      // 64
// Staging slab of one consumer warpgroup: 64 rows x 256 16-bit columns as four TMA boxes of 64 columns (128 B per row).
constexpr int SUB_COLS = 64;
constexpr int SUB_BYTES = WG_ROWS * SUB_COLS * 2;   // 8 KB
constexpr int STG_BYTES = WG_ROWS * BLOCK_N * 2;    // 32 KB
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + NUM_CONSUMERS * STG_BYTES + 1024 /*align slack*/ + 128 /*barriers*/;
static_assert(SMEM_BYTES <= 227 * 1024, "ring + staging must fit one CTA per SM");
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + NUM_CONSUMERS * 128 * CONSUMER_REGS <= 65536, "register file");

struct GemmParams {
  int M, N, K;
  int num_m_blocks, num_n_blocks;
  int k_blocks_total, k_blocks_per_split, splits;
  int units;           // num_m_blocks * num_n_blocks * splits
  int epilogue;
  void* D;
  long long ldd;
  const float* bias;   // [N] fp32 or null
  int has_aux;         // EPI_BIAS_RESIDUAL / EPI_DGELU / EPI_DGELU_PRE: the aux tile is TMA-loaded into the slab
  int has_out2;        // EPI_BIAS_GELU: a second output (gelu'(pre) or pre) goes to the out2 map
  float alpha;         // scale applied to the accumulator before the epilogue
  float* colsum;       // optional: colsum[n] += sum_m D(m, n) of the bf16-rounded output (bias gradients)
  Drop drop;           // EPI_BIAS_RESIDUAL only: D = dropout(acc + bias) + aux  (hidden dropout before the residual)
  int aux_f16, out_f16;  // aux / D hold fp16 instead of bf16 (the encoder's fp16 residual stream)
  int save_pre;          // EPI_BIAS_GELU: out2 receives the pre-activation itself instead of gelu'(pre) (lean activations)
};

// Work unit u -> tile origin and k-block range.  Units of one split are consecutive and tiles run N-fastest, so the
// ~one wave of units in flight at a time covers a band of A rows against all of B (the encoder's B is at most 4.7 MB,
// so it stays in L2); the wgrad splits in flight share one K slice of both operands.
struct Unit {
  int m0, n0, kb0, kb1;
};
__device__ __forceinline__ Unit unit_at(const GemmParams& p, int u) {
  const int tiles = p.num_m_blocks * p.num_n_blocks;
  const int tile = u % tiles, split = u / tiles;
  Unit w;
  w.m0 = (tile / p.num_n_blocks) * BLOCK_M;
  w.n0 = (tile % p.num_n_blocks) * BLOCK_N;
  w.kb0 = split * p.k_blocks_per_split;
  w.kb1 = min(w.kb0 + p.k_blocks_per_split, p.k_blocks_total);
  return w;
}

__device__ __forceinline__ void red_add_v2_f32(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
// barrier of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

template <int A_MN, int B_MN, int F16>
__device__ __forceinline__ void mma_kblock(float (&acc)[128], uint32_t sa, uint32_t sb, int accumulate_first) {
  // K-major SW128: 8-row groups 1024 B apart; a k16 step is +32 B inside the swizzle row.
  // MN-major SW128: 64-element MN atoms BLOCK_K*128 B apart (LBO), 8-deep K groups 1024 B apart; a k16 step is
  // +16 rows of 128 B.
  const uint64_t da = make_wgmma_desc_sw128(sa, A_MN ? BLOCK_K * 128 : 16, 1024);
  const uint64_t db = make_wgmma_desc_sw128(sb, B_MN ? BLOCK_K * 128 : 16, 1024);
  constexpr uint32_t A_KSTEP = (A_MN ? 16 * 128 : 32) >> 4;
  constexpr uint32_t B_KSTEP = (B_MN ? 16 * 128 : 32) >> 4;
#pragma unroll
  for (int k = 0; k < BLOCK_K / 16; ++k) {
    const int accum = (k > 0 || accumulate_first) ? 1 : 0;
    if (F16) wgmma_m64n256_ss_f16<A_MN, B_MN>(acc, da + k * A_KSTEP, db + k * B_KSTEP, accum);
    else wgmma_m64n256_ss_bf16<A_MN, B_MN>(acc, da + k * A_KSTEP, db + k * B_KSTEP, accum);
  }
}

__device__ __forceinline__ uint32_t pack_out(float a, float b, bool f16) { return f16 ? pack_f16x2(a, b) : pack_bf16x2(a, b); }

// Staging slab addressing.  Subtile c / 8 holds columns [64 (c / 8), +64) as 64 rows of 128 B, 128B-swizzled the way
// TMA reads and writes it: 16-byte chunk j of row r sits at chunk j ^ (r & 7).  The 8 rows one fragment store touches
// thus land in 8 different chunks, on 32 distinct banks.  A thread's pairs sit in rows lr and lr + 8, which share
// r & 7, so one base address per thread (row lr, its swizzled chunk 0, byte 4q) gives every pair with an XOR and an
// immediate offset.  32-bit shared addresses keep that to one register: with generic pointers the compiler hoists all
// 64 pair addresses out of the tile loop and spills them.
__device__ __forceinline__ uint32_t slab_base(const uint8_t* stg, int lr, int q) {
  return smem_u32(stg) + lr * 128 + ((lr & 7) << 4) + 4 * q;
}
// the pair (row lr + 8h, columns 8c + 2q, +1)
__device__ __forceinline__ uint32_t slab_pair(uint32_t base, int c, int h) {
  return (base ^ ((c & 7) << 4)) + (c >> 3) * SUB_BYTES + h * 8 * 128;
}
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
// Subtiles of the 64-row slab at (row0, n0) that hold any in-bounds element.  TMA clips the rest of a partial box on
// store and zero-fills it on load.
__device__ __forceinline__ int slab_boxes(int row0, int n0, int M, int N) {
  return row0 < M ? min(BLOCK_N / SUB_COLS, (N - n0 + SUB_COLS - 1) / SUB_COLS) : 0;
}
// One thread: TMA-store the slab as one bulk group.  The caller has fenced its writes to the async proxy and synced.
__device__ __forceinline__ void slab_tma_store(const CUtensorMap* m, const uint8_t* stg, int row0, int n0, int M, int N) {
  const int boxes = slab_boxes(row0, n0, M, N);
  for (int s = 0; s < boxes; ++s) tma_store_2d(m, smem_u32(stg + s * SUB_BYTES), n0 + s * SUB_COLS, row0);
  tma_store_commit();
}

// fp32 output straight from the fragment registers: split-K partial sums (red.global.add) or a plain store + bias
template <bool ATOMIC>
__device__ __forceinline__ void epilogue_f32(const GemmParams& p, const float (&acc)[128], int row0, int n0, int lr, int q) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + lr + 8 * h;
    if (row >= p.M) continue;
    float* drow = reinterpret_cast<float*>(p.D) + (long long)row * p.ldd;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      const int col = n0 + 8 * c + 2 * q;
      const float x = acc[4 * c + 2 * h] * p.alpha, y = acc[4 * c + 2 * h + 1] * p.alpha;
      if (ATOMIC) {
        if (col + 1 < p.N) red_add_v2_f32(drow + col, x, y);
        else if (col < p.N) atomicAdd(drow + col, x);
      } else {
        if (col < p.N) drow[col] = x + (p.bias != nullptr ? __ldg(p.bias + col) : 0.f);
        if (col + 1 < p.N) drow[col + 1] = y + (p.bias != nullptr ? __ldg(p.bias + col + 1) : 0.f);
      }
    }
  }
}

// 16-bit epilogues: the fragment-layout results go to the warpgroup's staging slab (which holds aux, if any, on entry).
// One instantiation per (epilogue, dropout, column sums), picked once per tile: the fully unrolled loop of each stays
// a short straight run of code, where one loop branching on all of them per element pair spans ~170 KB of SASS and
// misses the instruction cache on every tile.  EPI_BIAS_GELU leaves out2's values in acc.
template <int EP, bool DROP, bool COLSUM>
__device__ __forceinline__ void epilogue16(const GemmParams& p, float (&acc)[128], uint32_t slab, int row0, int n0, int lr,
                                           int q, int lane) {
  const bool out_f16 = p.out_f16 != 0, aux_f16 = p.aux_f16 != 0;
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    const int col = n0 + 8 * c + 2 * q;
    float2 b = make_float2(0.f, 0.f);
    if (p.bias != nullptr) {
      if (col + 1 < p.N) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
      else if (col < p.N) b.x = __ldg(p.bias + col);
    }
    float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + lr + 8 * h;
      const uint32_t sp = slab_pair(slab, c, h);
      float2 v = ffma2(make_float2(acc[4 * c + 2 * h], acc[4 * c + 2 * h + 1]), make_float2(p.alpha, p.alpha), b);
      if constexpr (EP == DPRB_EPI_BIAS_GELU) {
        float2 g, d;
        gelu_and_grad2(v, g, d);
        if (p.save_pre) d = v;        // lean activations: keep pre, rebuild gelu / gelu' in backward
        sts32(sp, pack_bf16x2(g.x, g.y));
        acc[4 * c + 2 * h] = d.x;
        acc[4 * c + 2 * h + 1] = d.y;
        continue;
      }
      if constexpr (DROP) {
        float m0f, m1f;
        p.drop.mul2((uint32_t)row, (uint32_t)col, m0f, m1f);
        v.x *= m0f; v.y *= m1f;
      }
      if constexpr (EP == DPRB_EPI_BIAS_RESIDUAL) {
        const float2 a = unpack_16x2(lds32(sp), aux_f16);
        v.x += a.x; v.y += a.y;
      } else if constexpr (EP == DPRB_EPI_DGELU) {
        const float2 a = unpack_bf16x2(lds32(sp));   // aux holds gelu'(pre) written by the forward epilogue
        v.x *= a.x; v.y *= a.y;
      } else if constexpr (EP == DPRB_EPI_DGELU_PRE) {
        float2 g, d;                           // aux holds the pre-activation: derivative rebuilt (same fitted function)
        gelu_and_grad2(unpack_bf16x2(lds32(sp)), g, d);
        v.x *= d.x; v.y *= d.y;
      }
      const uint32_t o = pack_out(v.x, v.y, out_f16);
      sts32(sp, o);
      if (COLSUM && row < p.M && col < p.N) {   // bias gradient: sums of the bf16-rounded output
        const float2 f = unpack_bf16x2(o);
        cs0 += f.x;
        if (col + 1 < p.N) cs1 += f.y;
      }
    }
    if (COLSUM) {
      // lanes with the same q hold the same columns: reduce over the 8 row groups of the warp
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        cs0 += __shfl_xor_sync(0xFFFFFFFFu, cs0, o);
        cs1 += __shfl_xor_sync(0xFFFFFFFFu, cs1, o);
      }
      if (lane < 4) {
        if (col < p.N) atomicAdd(p.colsum + col, cs0);
        if (col + 1 < p.N) atomicAdd(p.colsum + col + 1, cs1);
      }
    }
  }
}

template <int A_MN, int B_MN, int F16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_aux,
                 const __grid_constant__ CUtensorMap tmap_out2, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B needs 1024-byte aligned tiles
  uint8_t* smem = align1024(smem_raw);
  uint8_t* staging = smem + STAGES * STAGE_BYTES;                                     // [NUM_CONSUMERS][STG_BYTES]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + NUM_CONSUMERS * STG_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                                // [STAGES]
  uint64_t* aux_full = empty_bar + STAGES;                                                // [NUM_CONSUMERS]
  uint64_t* slab_empty = aux_full + NUM_CONSUMERS;                                        // [NUM_CONSUMERS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool out16 = p.epilogue != DPRB_EPI_F32_ATOMIC_ADD && p.epilogue != DPRB_EPI_F32_STORE;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (out16) tma_prefetch_desc(&tmap_d);
    if (p.has_aux) tma_prefetch_desc(&tmap_aux);
    if (p.has_out2) tma_prefetch_desc(&tmap_out2);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);                   // producer arrive (+ transaction bytes)
      mbar_init(&empty_bar[i], NUM_CONSUMERS * 4);  // one arrive per consumer warp
    }
    for (int i = 0; i < NUM_CONSUMERS; ++i) {
      mbar_init(&aux_full[i], 1);                   // producer arrive (+ transaction bytes)
      mbar_init(&slab_empty[i], 1);                 // the warpgroup's storing thread, once its stores have read the slab
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================ TMA producer ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0, uphase = 0;
      for (int u = blockIdx.x; u < p.units; u += gridDim.x, uphase ^= 1) {
        const Unit w = unit_at(p, u);
        // The aux tile goes in after this unit's first k-blocks are queued: the consumers free the slab at their second
        // k-block, so waiting for it here never leaves the ring empty.
        const int aux_kb = min(w.kb0 + 2, w.kb1 - 1);
        for (int kb = w.kb0; kb < w.kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_TILE_BYTES;
          if (A_MN == 0) {
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, w.m0);
          } else {
#pragma unroll
            for (int i = 0; i < BLOCK_M / 64; ++i) tma_load_2d(sa + i * (BLOCK_K * 128), &tmap_a, &full_bar[stage], w.m0 + i * 64, kb * BLOCK_K);
          }
          if (B_MN == 0) {
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, w.n0);
          } else {
#pragma unroll
            for (int i = 0; i < BLOCK_N / 64; ++i) tma_load_2d(sb + i * (BLOCK_K * 128), &tmap_b, &full_bar[stage], w.n0 + i * 64, kb * BLOCK_K);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (p.has_aux && kb == aux_kb) {
            for (int g = 0; g < NUM_CONSUMERS; ++g) {
              const int row0 = w.m0 + g * WG_ROWS;
              const int boxes = slab_boxes(row0, w.n0, p.M, p.N);
              uint8_t* slab = staging + g * STG_BYTES;
              mbar_wait(&slab_empty[g], uphase);
              mbar_arrive_expect_tx(&aux_full[g], boxes * SUB_BYTES);
              for (int s = 0; s < boxes; ++s)
                tma_load_2d(slab + s * SUB_BYTES, &tmap_aux, &aux_full[g], w.n0 + s * SUB_COLS, row0);
            }
          }
        }
      }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = (warp >> 2) - 1;
  const int t = threadIdx.x - 128 * (wg + 1);
  uint8_t* stg = staging + wg * STG_BYTES;
  // this warpgroup's 64 rows of the A tile: K-major +64 rows of 128 B, MN-major the second 64-wide MN atom
  const uint32_t a_off = (uint32_t)wg * (A_MN ? BLOCK_K * 128 : 64 * 128);
  // fragment coordinates: the thread holds slab rows lr (d[4c], d[4c+1]) and lr + 8 (d[4c+2], d[4c+3]) at columns
  // 8c + 2q, +1
  const int q = lane & 3;
  const int lr = (warp & 3) * 16 + (lane >> 2);
  const uint32_t slab = slab_base(stg, lr, q);
  const int ep = p.epilogue;

  float acc[128];
  int stage = 0;
  uint32_t phase = 0, uphase = 0;
  for (int u = blockIdx.x; u < p.units; u += gridDim.x, uphase ^= 1) {
    const Unit w = unit_at(p, u);
    {
      int prev = -1;
      // thread 0 hands the slab to the producer's aux load here, a full mainloop after the last unit's stores
      const int release_kb = min(w.kb0 + 1, w.kb1 - 1);
      for (int kb = w.kb0; kb < w.kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + a_off;
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES + A_TILE_BYTES);
        wgmma_fence();
        mma_kblock<A_MN, B_MN, F16>(acc, sa, sb, kb > w.kb0);
        wgmma_commit();
        // keep one k-block of MMAs in flight; the one before it has retired and its stage can be refilled
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        if (p.has_aux && kb == release_kb && t == 0) {
          tma_store_wait_read();
          mbar_arrive(&slab_empty[wg]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }

    // ================================ epilogue ================================
    const int row0 = w.m0 + wg * WG_ROWS;   // first global row of this warpgroup's slab
    switch (ep) {
      case DPRB_EPI_F32_ATOMIC_ADD: epilogue_f32<true>(p, acc, row0, w.n0, lr, q); continue;
      case DPRB_EPI_F32_STORE: epilogue_f32<false>(p, acc, row0, w.n0, lr, q); continue;
      default: break;
    }
    if (p.has_aux) mbar_wait(&aux_full[wg], uphase);   // the producer loaded it after the slab was released above
    else if (t == 0) tma_store_wait_read();            // the previous unit's stores have read the slab
    // also reconverges the warpgroup after the waits: the column-sum shuffles then need no divergence fallback
    wg_bar(wg);
    const bool cs = p.colsum != nullptr, drop = p.drop.on();
    switch (ep) {
      case DPRB_EPI_BIAS:
        if (cs) epilogue16<DPRB_EPI_BIAS, false, true>(p, acc, slab, row0, w.n0, lr, q, lane);
        else epilogue16<DPRB_EPI_BIAS, false, false>(p, acc, slab, row0, w.n0, lr, q, lane);
        break;
      case DPRB_EPI_BIAS_GELU: epilogue16<DPRB_EPI_BIAS_GELU, false, false>(p, acc, slab, row0, w.n0, lr, q, lane); break;
      case DPRB_EPI_BIAS_RESIDUAL:
        if (drop) {
          if (cs) epilogue16<DPRB_EPI_BIAS_RESIDUAL, true, true>(p, acc, slab, row0, w.n0, lr, q, lane);
          else epilogue16<DPRB_EPI_BIAS_RESIDUAL, true, false>(p, acc, slab, row0, w.n0, lr, q, lane);
        } else {
          if (cs) epilogue16<DPRB_EPI_BIAS_RESIDUAL, false, true>(p, acc, slab, row0, w.n0, lr, q, lane);
          else epilogue16<DPRB_EPI_BIAS_RESIDUAL, false, false>(p, acc, slab, row0, w.n0, lr, q, lane);
        }
        break;
      case DPRB_EPI_DGELU:
        if (cs) epilogue16<DPRB_EPI_DGELU, false, true>(p, acc, slab, row0, w.n0, lr, q, lane);
        else epilogue16<DPRB_EPI_DGELU, false, false>(p, acc, slab, row0, w.n0, lr, q, lane);
        break;
      default:
        if (cs) epilogue16<DPRB_EPI_DGELU_PRE, false, true>(p, acc, slab, row0, w.n0, lr, q, lane);
        else epilogue16<DPRB_EPI_DGELU_PRE, false, false>(p, acc, slab, row0, w.n0, lr, q, lane);
        break;
    }
    fence_proxy_async_smem();   // make the slab writes visible to the TMA store
    wg_bar(wg);
    if (t == 0) slab_tma_store(&tmap_d, stg, row0, w.n0, p.M, p.N);
    if (p.has_out2) {
      // one slab for both outputs: out2 waits until D's stores have read it
      if (t == 0) tma_store_wait_read();
      wg_bar(wg);
#pragma unroll
      for (int c = 0; c < 32; ++c)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          sts32(slab_pair(slab, c, h), pack_bf16x2(acc[4 * c + 2 * h], acc[4 * c + 2 * h + 1]));
      fence_proxy_async_smem();
      wg_bar(wg);
      if (t == 0) slab_tma_store(&tmap_out2, stg, row0, w.n0, p.M, p.N);
    }
  }
  if (t == 0) tma_store_wait_all();   // the slab must outlive the stores that read it
}

// ---------------------------------------------------------------- host side
// Row-major 16-bit matrix [rows, cols] with leading dimension ld (elements); box = [box_rows, 64 cols], 128B swizzle.
// Encoded as BFLOAT16 for fp16 operands too: TMA only moves the bytes.
int make_tmap(CUtensorMap* out, const void* base, long long rows, long long cols, long long ld, int box_rows) {
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "gemm operand base %p not 16-byte aligned", base);
  DPRB_REQUIRE((ld * 2) % 16 == 0, "gemm operand leading dimension %lld not a multiple of 8 elements", ld);
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  return encode_tmap(out, "gemm", CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// ---- optional live profiling: CUDA events around every GEMM launch (bench.py's roofline leg) ----
struct GemmProfile {
  bool enabled = false;
  std::vector<cudaEvent_t> ev;   // pairs
  std::vector<double> flops;
  size_t used = 0;
};
GemmProfile g_prof;

int choose_splits(int tiles, int k_blocks, int sms) {
  // One CTA per SM walks ceil(tiles*s/sms) units of ceil(k_blocks/s) k-blocks each; every unit also pays about 4
  // k-blocks' worth for its fp32 atomic epilogue (a 128x256 tile = 128 KB of red.global.add), which keeps s from
  // growing for a marginally better fit.  Minimise that makespan, keeping >= 4 k-blocks per split.
  int best = 1;
  double best_cost = 1e30;
  for (int s = 1; s <= 32; ++s) {
    if (k_blocks / s < 4 && s > 1) break;
    const int rounds = (tiles * s + sms - 1) / sms;
    const double cost = (double)rounds * ((k_blocks + s - 1) / s + 4);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
  }
  return best;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int64_t lda, int64_t ldb,
                              int64_t ldd, int a_mn_major, int b_mn_major, int epilogue, const float* bias,
                              const void* aux, int64_t ld_aux, void* out2, float alpha, int splits, float* colsum,
                              float dropout_p, uint64_t drop_site_seed, dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  const int dt_flags = epilogue & ~0xFF;   // DPRB_GEMM_{A,B,AUX,OUT}_F16, DPRB_GEMM_SAVE_PRE
  epilogue &= 0xFF;
  const int a_f16 = (dt_flags & DPRB_GEMM_A_F16) != 0, b_f16 = (dt_flags & DPRB_GEMM_B_F16) != 0;
  const int aux_f16 = (dt_flags & DPRB_GEMM_AUX_F16) != 0, out_f16 = (dt_flags & DPRB_GEMM_OUT_F16) != 0;
  DPRB_REQUIRE(epilogue >= 0 && epilogue < DPRB_EPI_COUNT, "gemm: bad epilogue %d", epilogue);
  DPRB_REQUIRE(!(aux_f16 || out_f16) || epilogue == DPRB_EPI_BIAS || epilogue == DPRB_EPI_BIAS_RESIDUAL,
               "gemm: fp16 aux / output is implemented for the BIAS and BIAS_RESIDUAL epilogues only");
  DPRB_REQUIRE(a_f16 == b_f16, "gemm: wgmma takes no fp16 x bf16 operand pair: give "
               "DPRB_GEMM_A_F16 and DPRB_GEMM_B_F16 together or not at all");
  DPRB_REQUIRE(!out_f16 || colsum == nullptr, "gemm: colsum reads a bf16 slab (not available with fp16 output)");
  const bool f32_out = (epilogue == DPRB_EPI_F32_ATOMIC_ADD || epilogue == DPRB_EPI_F32_STORE);
  DPRB_REQUIRE(f32_out || (ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0),
               "gemm: bf16 output must be 16-byte aligned with ldd %% 8 == 0 (ldd=%lld)", (long long)ldd);
  DPRB_REQUIRE(!f32_out || (ldd % 4 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0),
               "gemm: fp32 output must be 16-byte aligned with ldd %% 4 == 0 (ldd=%lld)", (long long)ldd);
  const bool has_aux = epilogue == DPRB_EPI_BIAS_RESIDUAL || epilogue == DPRB_EPI_DGELU || epilogue == DPRB_EPI_DGELU_PRE;
  if (has_aux)
    DPRB_REQUIRE(aux != nullptr && ld_aux % 8 == 0 && (reinterpret_cast<uintptr_t>(aux) & 15) == 0,
                 "gemm: epilogue %d needs a 16-byte aligned aux with ld %% 8 == 0", epilogue);
  if (bias != nullptr) DPRB_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15) == 0, "gemm: bias not 16B aligned");

  DPRB_REQUIRE(colsum == nullptr || (!f32_out && epilogue != DPRB_EPI_BIAS_GELU),
               "gemm: colsum is supported for the BIAS / BIAS_RESIDUAL / DGELU epilogues only");

  const bool has_out2 = epilogue == DPRB_EPI_BIAS_GELU && out2 != nullptr;
  if (has_out2)
    DPRB_REQUIRE((reinterpret_cast<uintptr_t>(out2) & 15) == 0, "gemm: out2 not 16-byte aligned");

  // 16-bit outputs, aux and out2 move as 64-row x 64-column boxes: one per subtile of a warpgroup's staging slab
  CUtensorMap ta, tb, td{}, tx{}, to2{};
  int rc;
  if (!a_mn_major) rc = make_tmap(&ta, A, M, K, lda, BLOCK_M); else rc = make_tmap(&ta, A, K, M, lda, BLOCK_K);
  if (rc) return rc;
  if (!b_mn_major) rc = make_tmap(&tb, B, N, K, ldb, BLOCK_N); else rc = make_tmap(&tb, B, K, N, ldb, BLOCK_K);
  if (rc) return rc;
  if (!f32_out && (rc = make_tmap(&td, D, M, N, ldd, WG_ROWS))) return rc;
  if (has_aux && (rc = make_tmap(&tx, aux, M, N, ld_aux, WG_ROWS))) return rc;
  if (has_out2 && (rc = make_tmap(&to2, out2, M, N, ldd, WG_ROWS))) return rc;

  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.num_m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  p.num_n_blocks = (N + BLOCK_N - 1) / BLOCK_N;
  p.k_blocks_total = (K + BLOCK_K - 1) / BLOCK_K;
  DPRB_NUM_SMS(sms);
  const int tiles = p.num_m_blocks * p.num_n_blocks;
  if (epilogue != DPRB_EPI_F32_ATOMIC_ADD) splits = 1;
  else if (splits <= 0) splits = choose_splits(tiles, p.k_blocks_total, sms);
  if (splits > p.k_blocks_total) splits = p.k_blocks_total;
  p.k_blocks_per_split = (p.k_blocks_total + splits - 1) / splits;
  p.splits = (p.k_blocks_total + p.k_blocks_per_split - 1) / p.k_blocks_per_split;
  p.epilogue = epilogue;
  p.D = D; p.ldd = ldd; p.bias = bias; p.has_aux = has_aux; p.has_out2 = has_out2; p.alpha = alpha;
  p.colsum = colsum;
  p.aux_f16 = aux_f16; p.out_f16 = out_f16;
  p.save_pre = (dt_flags & DPRB_GEMM_SAVE_PRE) != 0;
  p.drop = drop_from_site(epilogue == DPRB_EPI_BIAS_RESIDUAL ? dropout_p : 0.f, drop_site_seed);

  p.units = tiles * p.splits;
  const int grid = p.units < sms ? p.units : sms;   // persistent: one CTA per SM
  static bool attr_set = false;
  if (!attr_set) {
#define DPRB_SET_ATTR(...) DPRB_CHECK_CUDA(cudaFuncSetAttribute(__VA_ARGS__, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    DPRB_SET_ATTR(gemm_bf16_kernel<0, 0, 0>) DPRB_SET_ATTR(gemm_bf16_kernel<0, 1, 0>)
    DPRB_SET_ATTR(gemm_bf16_kernel<1, 0, 0>) DPRB_SET_ATTR(gemm_bf16_kernel<1, 1, 0>)
    DPRB_SET_ATTR(gemm_bf16_kernel<0, 0, 1>) DPRB_SET_ATTR(gemm_bf16_kernel<0, 1, 1>)
    DPRB_SET_ATTR(gemm_bf16_kernel<1, 0, 1>) DPRB_SET_ATTR(gemm_bf16_kernel<1, 1, 1>)
#undef DPRB_SET_ATTR
    attr_set = true;
  }
  auto launch = [&](auto kern) -> int {
    const bool prof = g_prof.enabled && g_prof.used + 2 <= g_prof.ev.size();
    if (prof) DPRB_CHECK_CUDA(cudaEventRecord(g_prof.ev[g_prof.used], stream));
    kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ta, tb, td, tx, to2, p);
    DPRB_LAUNCH_CHECK();
    if (prof) {
      DPRB_CHECK_CUDA(cudaEventRecord(g_prof.ev[g_prof.used + 1], stream));
      g_prof.flops.push_back(2.0 * (double)M * (double)N * (double)K);
      g_prof.used += 2;
    }
    return 0;
  };
  const int key = (a_mn_major ? 4 : 0) | (b_mn_major ? 2 : 0) | (a_f16 ? 1 : 0);
  switch (key) {
    case 0: return launch(gemm_bf16_kernel<0, 0, 0>);
    case 1: return launch(gemm_bf16_kernel<0, 0, 1>);
    case 2: return launch(gemm_bf16_kernel<0, 1, 0>);
    case 3: return launch(gemm_bf16_kernel<0, 1, 1>);
    case 4: return launch(gemm_bf16_kernel<1, 0, 0>);
    case 5: return launch(gemm_bf16_kernel<1, 0, 1>);
    case 6: return launch(gemm_bf16_kernel<1, 1, 0>);
    default: return launch(gemm_bf16_kernel<1, 1, 1>);
  }
}

extern "C" int dprb_gemm_profile_enable(int enable, int max_launches) {
  if (enable) {
    const size_t want = (size_t)max_launches * 2;
    while (g_prof.ev.size() < want) {
      cudaEvent_t e;
      DPRB_CHECK_CUDA(cudaEventCreate(&e));
      g_prof.ev.push_back(e);
    }
    g_prof.used = 0;
    g_prof.flops.clear();
  }
  g_prof.enabled = enable != 0;
  return 0;
}

// Sums the recorded launch durations (synchronises on each end event). Outputs: total ms, total FLOPs, launches.
extern "C" int dprb_gemm_profile_read(double* total_ms, double* total_flops, int64_t* launches) {
  double ms = 0.0, fl = 0.0;
  for (size_t i = 0; i + 1 < g_prof.used; i += 2) {
    DPRB_CHECK_CUDA(cudaEventSynchronize(g_prof.ev[i + 1]));
    float t = 0.f;
    DPRB_CHECK_CUDA(cudaEventElapsedTime(&t, g_prof.ev[i], g_prof.ev[i + 1]));
    ms += t;
    fl += g_prof.flops[i / 2];
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = (int64_t)(g_prof.used / 2);
  return 0;
}
