// Brute-force inner-product search with a running top-k, for sm_90a.
//
// Replaces search_index() of the reference (dpr_scale/run_retrieval_pytorch.py):
//     scores = einsum('ik,jk->ij', queries.half(), corpus)          # [Q, N] fp16, materialised
//     sort_scores, sort_candidates = torch.topk(scores, k)          # several more passes over [Q, N]
// and the per-shard merge (concat shard results, topk, gather).
//
// Design: the [Q, N] score matrix never exists.  The corpus ([N, d] fp16/bf16, K-major, resident in HBM) is
// streamed ONCE per block of <= 128 queries through a TMA -> wgmma pipeline (two m64n128k16 per k16 step, fp32
// accumulators staged in shared memory as a [128 query][128 row] tile).  Thread i of the filter warpgroup owns
// query i: it keeps that query's current bar in a register, tests the max of each 32-score chunk against it, and
// appends the (rare) scores above the bar to a private candidate queue.  The bar is the larger of the query's own
// k-th best (a full queue is cut back to its best k by the whole warp: exact bisection on (score, ~row) keys) and
// a cross-partition bound (min over partitions of their m-th best, m = ceil(k / partitions)), which rises much
// faster and keeps the queues a few entries long.  The corpus stream costs 2*d bytes per corpus row per query
// block.  A second small kernel merges the per-CTA queues of every
// query (exact selection + bitonic sort).
//
// Ranking is by fp32-accumulated score, ties broken towards the lower index (torch.topk leaves tie order
// unspecified).  Results are exact for the fp32 scores: no approximation, no score quantisation.
#include <cstdint>
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {

namespace {

typedef unsigned long long u64;

constexpr int QT = 128;       // queries per CTA = filter threads
constexpr int CT = 128;       // corpus rows per tile = wgmma N
constexpr int BK = 64;        // 64 x 2 B = one 128-byte swizzle row
constexpr int UK = 16;
constexpr int STAGES = 4;
constexpr int A_BYTES = QT * BK * 2;   // 16 KB
constexpr int B_BYTES = CT * BK * 2;   // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int ACC_LD = CT + 4;         // fp32 score tile [QT][ACC_LD] (padded: conflict-free row reads)
constexpr int THREADS = 256;           // warp 0 TMA, warps 4-7 (warpgroup 1) wgmma + filter
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + QT * ACC_LD * 4 + 1024 + 256;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");
constexpr int MAX_QTILES = 8;          // query tiles per launch (they share the corpus stream through L2)

constexpr int SEL_THREADS = 1024;
constexpr int SEL_SMEM_KEYS = 22528;   // 176 KB of candidates staged in shared memory

struct SearchParams {
  long long N;          // corpus rows
  int Q;                // queries in this launch (<= gridDim.y * 128)
  int d;
  int k;
  int kblocks;          // ceil(d / 64)
  long long tiles;      // ceil(N / 128)
  long long tiles_per_part;
  u64* queues;          // [gridDim.x][gridDim.y * 128][CAP]
  int* counts;          // [gridDim.x][gridDim.y * 128]
  uint32_t* bounds;     // [gridDim.x][gridDim.y * 128] ordered-uint of each partition's m-th best score (0 = none yet)
  int m_track;          // m = ceil(k / partitions) if <= 8, else 0 (cross-partition bound disabled)
  int f16;              // operands are fp16 (else bf16)
  int rank_f16;         // rank by the fp16-ROUNDED score: the reference's einsum on fp16 tensors returns fp16
                        // (run_retrieval_pytorch.py:150-151), so its topk orders fp16 values; ties go to the lower row id
};

__device__ __forceinline__ uint32_t ord_u32(float v) {   // monotone float -> unsigned
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_u32(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}
__device__ __forceinline__ u64 make_key(float v, uint32_t idx) {
  if (v == 0.0f) v = 0.0f;   // -0 and +0 are equal scores: one key, so the tie goes to the lower index
  return ((u64)ord_u32(v) << 32) | (u64)(~idx);        // larger key = better score, then lower index
}
__device__ __forceinline__ float key_score(u64 key) { return unord_u32((uint32_t)(key >> 32)); }
__device__ __forceinline__ uint32_t key_index(u64 key) { return ~(uint32_t)key; }

// Warp-collective: every lane owns one queue (myq, cnt, thr).  Queues with more than `limit` entries are cut back
// to their best k entries; thr becomes the k-th best score.  Exact: bisection over the 64 key bits finds the k-th
// largest key P (keys are unique), then the entries >= P are packed to the front.
template <int EPL>
__device__ __forceinline__ void compact_queues(u64* myq, uint32_t& cnt, float& thr, const uint32_t k,
                                               const uint32_t limit, const int lane) {
  uint32_t need = __ballot_sync(0xFFFFFFFFu, cnt > limit);
  while (need) {
    const int src = __ffs(need) - 1;
    need &= need - 1;
    u64* qb = reinterpret_cast<u64*>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<u64>(myq), src));
    const uint32_t n = __shfl_sync(0xFFFFFFFFu, cnt, src);
    __syncwarp();
    u64 key[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const uint32_t slot = e * 32 + lane;
      key[e] = slot < n ? qb[slot] : 0ull;
    }
    // k-th largest key P: bisection on the 32 score bits, then (only if the k-th score is tied) on the id bits
    uint32_t Ph = 0;
#pragma unroll 1
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t t = Ph | (1u << bit);
      uint32_t c = 0;
#pragma unroll
      for (int e = 0; e < EPL; ++e) c += (uint32_t)(key[e] >> 32) >= t ? 1u : 0u;
      c = __reduce_add_sync(0xFFFFFFFFu, c);
      if (c >= k) Ph = t;
    }
    uint32_t above = 0, tied = 0;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const uint32_t h = (uint32_t)(key[e] >> 32);
      above += h > Ph ? 1u : 0u;
      tied += (h == Ph && key[e] != 0ull) ? 1u : 0u;
    }
    above = __reduce_add_sync(0xFFFFFFFFu, above);
    tied = __reduce_add_sync(0xFFFFFFFFu, tied);
    uint32_t Pl = 0;
    if (above < k && tied > k - above) {          // warp-uniform: more rows share the k-th score than fit
      const uint32_t want = k - above;
#pragma unroll 1
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t t = Pl | (1u << bit);
        uint32_t c = 0;
#pragma unroll
        for (int e = 0; e < EPL; ++e)
          c += ((uint32_t)(key[e] >> 32) == Ph && (uint32_t)key[e] >= t) ? 1u : 0u;
        c = __reduce_add_sync(0xFFFFFFFFu, c);
        if (c >= want) Pl = t;
      }
    }
    const u64 P = ((u64)Ph << 32) | (u64)Pl;
    __syncwarp();
    uint32_t base = 0;
    const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
    for (int e = 0; e < EPL; ++e) {
      const bool keep = key[e] != 0ull && key[e] >= P;
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, keep);
      if (keep) qb[base + __popc(bal & lt)] = key[e];
      base += __popc(bal);
    }
    __syncwarp();
    if (lane == src) {
      cnt = base;
      if (base >= k) thr = key_score(P);
    }
  }
}

template <int EPL>
__global__ void __launch_bounds__(THREADS, 1)
search_topk_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_c,
                   const SearchParams p) {
  constexpr uint32_t CAP = 32 * EPL;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_BYTES;
  float* sAcc = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [QT][ACC_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sAcc + QT * ACC_LD);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long t0 = (long long)blockIdx.x * p.tiles_per_part;
  const long long t1 = min(t0 + p.tiles_per_part, p.tiles);
  const int q0 = blockIdx.y * QT;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_c);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);   // one arrive per filter warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ---------------- TMA producer: query tile (L2-resident) + corpus tile (HBM stream) per k-block
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = t0; t < t1; ++t) {
        const int row0 = (int)(t * CT);
        for (int kb = 0; kb < p.kblocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(smem_a + stage * A_BYTES, &tm_q, &full_bar[stage], kb * BK, q0);
          tma_load_2d(smem_b + stage * B_BYTES, &tm_c, &full_bar[stage], kb * BK, row0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ---------------- wgmma + threshold filter: thread <-> query
    const int quarter = warp & 3;
    const int qslot = blockIdx.y * QT + quarter * 32 + lane;         // < gridDim.y * 128
    const int qpad = gridDim.y * QT;
    u64* myq = p.queues + ((size_t)blockIdx.x * qpad + qslot) * CAP;
    const bool active = qslot < p.Q;
    float thr = active ? -INFINITY : INFINITY;
    uint32_t cnt = 0;
    const uint32_t k = (uint32_t)p.k;
    // Cross-partition bound: every partition publishes its m-th best score for this query (m = ceil(k / partitions));
    // all partitions hold >= m rows at or above the minimum G of those, i.e. >= k rows in total, so rows scoring
    // below G cannot be in the top-k.  G rises like the best of n rows, long before the local k-th best does, which
    // keeps the queues short (usually no compaction at all).  t0_..t7_ = this partition's 8 best scores so far.
    const bool track = active && p.m_track > 0;
    const float top_init = track ? -INFINITY : INFINITY;
    float t0_ = top_init, t1_ = top_init, t2_ = top_init, t3_ = top_init, t4_ = top_init, t5_ = top_init,
          t6_ = top_init, t7_ = top_init;                              // descending
    uint32_t* my_bound = p.bounds + (size_t)blockIdx.x * qpad + qslot;
    const uint32_t* q_bounds = p.bounds + qslot;
    float lowbar = fminf(thr, t7_);
    int stage = 0;
    uint32_t phase = 0;
    long long done = 0;
    const float* arow = sAcc + (quarter * 32 + lane) * ACC_LD;
    for (long long t = t0; t < t1; ++t) {
      {
        float d0[64], d1[64];      // query rows [0, 64) and [64, 128) of the tile
        for (int kb = 0; kb < p.kblocks; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint64_t a_desc = make_wgmma_desc_sw128(smem_u32(smem_a + stage * A_BYTES), 16, 1024);
          const uint64_t b_desc = make_wgmma_desc_sw128(smem_u32(smem_b + stage * B_BYTES), 16, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k) {
            const int accum = (kb > 0 || k > 0) ? 1 : 0;
            if (p.f16) {
              wgmma_m64n128_ss_f16<0, 0>(d0, a_desc + 2 * k, b_desc + 2 * k, accum);
              wgmma_m64n128_ss_f16<0, 0>(d1, a_desc + 64 * 8 + 2 * k, b_desc + 2 * k, accum);   // +64 rows of 128 B
            } else {
              wgmma_m64n128_ss_bf16<0, 0>(d0, a_desc + 2 * k, b_desc + 2 * k, accum);
              wgmma_m64n128_ss_bf16<0, 0>(d1, a_desc + 64 * 8 + 2 * k, b_desc + 2 * k, accum);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        // the previous tile's rows have all been read (barrier at the end of the loop body)
        store_acc_128x128<ACC_LD>(sAcc, d0, d1, quarter, lane);
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      const long long rem = p.N - t * CT;
      const int ncols = rem < CT ? (int)rem : CT;
      const uint32_t idx0 = (uint32_t)(t * CT);
#pragma unroll 1
      for (int c = 0; c < CT / 32; ++c) {
        if (c * 32 >= ncols) break;
        if (__any_sync(0xFFFFFFFFu, cnt > CAP - 32)) {
          compact_queues<EPL>(myq, cnt, thr, k, CAP - 32, lane);
          lowbar = fminf(thr, t7_);
        }
        uint32_t r[32];
#pragma unroll
        for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(r + j) = *reinterpret_cast<const float4*>(arow + c * 32 + j);
        const uint32_t ib = idx0 + c * 32;
        const int nvalid = ncols - c * 32;          // >= 32 except in the ragged last tile
        // one test per 32 scores: in steady state almost no chunk holds a score above the bar
        float cmax = __uint_as_float(r[0]);
#pragma unroll
        for (int j = 1; j < 32; ++j) cmax = fmaxf(cmax, __uint_as_float(r[j]));
        if (p.rank_f16) cmax = __half2float(__float2half_rn(cmax));   // rounding is monotone: max commutes with it
        if (cmax >= lowbar) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float v = __uint_as_float(r[j]);
            if (p.rank_f16) v = __half2float(__float2half_rn(v));
            if (v >= lowbar && j < nvalid) {
              if (v >= thr) myq[cnt++] = make_key(v, ib + j);
              if (v > t7_) {
                float x = v, y;                                            // insert, dropping the old 8th best
                y = fminf(t0_, x); t0_ = fmaxf(t0_, x); x = y;
                y = fminf(t1_, x); t1_ = fmaxf(t1_, x); x = y;
                y = fminf(t2_, x); t2_ = fmaxf(t2_, x); x = y;
                y = fminf(t3_, x); t3_ = fmaxf(t3_, x); x = y;
                y = fminf(t4_, x); t4_ = fmaxf(t4_, x); x = y;
                y = fminf(t5_, x); t5_ = fmaxf(t5_, x); x = y;
                y = fminf(t6_, x); t6_ = fmaxf(t6_, x); x = y;
                t7_ = fmaxf(t7_, x);
              }
              lowbar = fminf(thr, t7_);
            }
          }
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");   // the tile is read: the next one may overwrite it
      ++done;
      if (p.m_track > 0 && ((done & (done - 1)) == 0 || (done & 31) == 0)) {
        const int mt = p.m_track;
        const float mine = mt == 1 ? t0_ : mt == 2 ? t1_ : mt == 3 ? t2_ : mt == 4 ? t3_ : mt == 5 ? t4_
                         : mt == 6 ? t5_ : mt == 7 ? t6_ : t7_;
        if (track) __stcg(my_bound, ord_u32(mine));
        uint32_t g = 0xFFFFFFFFu;
        for (int part = 0; part < (int)gridDim.x; ++part) g = min(g, __ldcg(q_bounds + (size_t)part * qpad));
        if (track && g > ord_u32(thr)) {
          thr = unord_u32(g);
          lowbar = fminf(thr, t7_);
          // drop queued rows that fell below the new bound (thread-private pass; keeps the final lists short)
          const u64 floor_key = (u64)g << 32;
          uint32_t w = 0;
          for (uint32_t i = 0; i < cnt; ++i) {
            const u64 key = myq[i];
            if (key >= floor_key) myq[w++] = key;
          }
          cnt = w;
        }
      }
    }
    // leave at most k candidates per queue for the merge
    if (__any_sync(0xFFFFFFFFu, cnt > k)) compact_queues<EPL>(myq, cnt, thr, k, k, lane);
    p.counts[(size_t)blockIdx.x * qpad + qslot] = (int)cnt;
  }

}

// One CTA per query: gather the candidate lists, select the k best keys exactly, sort them, write scores / indices.
// list l of query q: lists + l * list_stride + q * query_stride, length counts[l * count_stride + q] (or fixed).
struct SelectParams {
  const u64* lists;
  const int* counts;
  int num_lists;
  long long list_stride, query_stride, count_stride;
  int fixed_count;
  int k, kpad;
  long long index_offset;
  float* out_scores;      // [Q, k]
  long long* out_index;   // [Q, k]
  const long long* gather;   // optional [Q, gather_stride]: out_index = gather[q][key index] instead of the key index
  long long gather_stride;
  u64* scratch;           // [Q, scratch_per_query] or null (used when the candidates do not fit shared memory)
  long long scratch_per_query;
};

__global__ void __launch_bounds__(SEL_THREADS, 1) select_topk_kernel(const SelectParams p) {
  extern __shared__ uint8_t sel_smem[];
  u64* s_keys = reinterpret_cast<u64*>(sel_smem);                    // [SEL_SMEM_KEYS]
  u64* s_out = s_keys + SEL_SMEM_KEYS;                                // [kpad <= 1024]
  int* s_off = reinterpret_cast<int*>(s_out + 1024);                  // [num_lists + 1]   (<= 1024 + 1)
  __shared__ uint32_t s_cnt[64];
  __shared__ uint32_t s_nout;
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (int l = tid; l < p.num_lists; l += SEL_THREADS)
    s_off[l + 1] = p.counts != nullptr ? p.counts[(long long)l * p.count_stride + q] : p.fixed_count;
  if (tid < 64) s_cnt[tid] = 0;
  if (tid == 0) { s_off[0] = 0; s_nout = 0; }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int l = 0; l < p.num_lists; ++l) { const int c = s_off[l + 1]; s_off[l] = run; run += c; }
    s_off[p.num_lists] = run;
  }
  __syncthreads();
  const int total = s_off[p.num_lists];
  u64* cand = total <= SEL_SMEM_KEYS ? s_keys : p.scratch + (long long)q * p.scratch_per_query;
  for (int l = warp; l < p.num_lists; l += SEL_THREADS / 32) {
    const u64* src = p.lists + (long long)l * p.list_stride + (long long)q * p.query_stride;
    const int o = s_off[l], n = s_off[l + 1] - o;
    for (int i = lane; i < n; i += 32) cand[o + i] = src[i];
  }
  __syncthreads();

  const uint32_t k = (uint32_t)min(p.k, total);
  u64 P = 0;
  for (int bit = 63; bit >= 0; --bit) {
    const u64 t = P | (1ull << bit);
    uint32_t c = 0;
    for (int i = tid; i < total; i += SEL_THREADS) c += cand[i] >= t ? 1u : 0u;
    c = __reduce_add_sync(0xFFFFFFFFu, c);
    if (lane == 0 && c) atomicAdd(&s_cnt[63 - bit], c);
    __syncthreads();
    if (s_cnt[63 - bit] >= k) P = t;
  }
  for (int i = tid; i < p.kpad; i += SEL_THREADS) s_out[i] = 0ull;
  __syncthreads();
  for (int i = tid; i < total; i += SEL_THREADS) {
    const u64 key = cand[i];
    if (key >= P && key != 0ull) {
      const uint32_t pos = atomicAdd(&s_nout, 1u);
      if (pos < (uint32_t)p.kpad) s_out[pos] = key;
    }
  }
  // bitonic sort, descending
  for (int size = 2; size <= p.kpad; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      if (tid < p.kpad) {
        const int j = tid ^ stride;
        if (j > tid) {
          const bool up = (tid & size) == 0;
          const u64 a = s_out[tid], b = s_out[j];
          if ((a < b) == up) { s_out[tid] = b; s_out[j] = a; }
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < p.k; i += SEL_THREADS) {
    const u64 key = s_out[i];
    const bool ok = key != 0ull;
    p.out_scores[(long long)q * p.k + i] = ok ? key_score(key) : -INFINITY;
    long long id = -1ll;
    if (ok) {
      id = (long long)key_index(key);
      id = p.gather != nullptr ? p.gather[(long long)q * p.gather_stride + id] : id + p.index_offset;
    }
    p.out_index[(long long)q * p.k + i] = id;
  }
}

// key index = position inside the query's concatenated list (ties resolve towards the earlier shard / rank)
__global__ void pack_keys_kernel(const float* __restrict__ scores, u64* keys, long long n, int total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = make_key(scores[i], (uint32_t)(i % total));
}

// row-major 16-bit matrix [rows, d]; box = [box_rows, 64 cols]; rows / cols past the end read as zero
int make_tmap(CUtensorMap* out, const void* base, long long rows, int d, int box_rows, int dtype) {
  const cuuint64_t dims[2] = {(cuuint64_t)d, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)d * 2};
  const cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  return encode_tmap(out, "search", dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                     base, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

int cap_for_k(int k) { return k <= 256 ? 512 : 2048; }

struct WsLayout {
  u64* queues;
  int* counts;
  uint32_t* bounds;
  u64* scratch;           // null when every query's candidates fit the selection kernel's shared memory
  long long scratch_per_query, total;
};
WsLayout ws_layout(void* base, long long Q, int k, int sms) {
  const long long slots = (long long)sms * QT;                      // parts * qtiles * 128 <= sms * 128 per launch
  Carve c(base);
  WsLayout w;
  w.queues = (u64*)c.take(slots * cap_for_k(k) * (long long)sizeof(u64));
  w.counts = (int*)c.take(slots * (long long)sizeof(int));
  w.bounds = (uint32_t*)c.take(slots * (long long)sizeof(uint32_t));
  w.scratch_per_query = (long long)sms * k;                         // parts <= sms lists of <= k keys
  const long long qb = Q < (long long)MAX_QTILES * QT ? Q : (long long)MAX_QTILES * QT;
  w.scratch = w.scratch_per_query > SEL_SMEM_KEYS ? (u64*)c.take(qb * w.scratch_per_query * (long long)sizeof(u64))
                                                  : nullptr;
  w.total = c.off;
  return w;
}

int launch_select(const SelectParams& sp, long long Q, cudaStream_t stream) {
  static bool attr_set = false;
  const int smem = SEL_SMEM_KEYS * 8 + 1024 * 8 + (1024 + 8) * 4;
  if (!attr_set) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(select_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  select_topk_kernel<<<(unsigned)Q, SEL_THREADS, smem, stream>>>(sp);
  DPRB_LAUNCH_CHECK();
  return 0;
}

int kpad_for(int k) {
  int kp = 2;
  while (kp < k) kp <<= 1;
  return kp;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int64_t dprb_search_workspace_bytes(int64_t Q, int k) {
  const int sms = num_sms();
  return sms > 0 ? ws_layout(nullptr, Q, k, sms).total : -1;
}

extern "C" int dprb_search_topk(const void* queries, const void* corpus, int dtype, int64_t Q, int64_t N, int d, int k,
                                int64_t index_offset, float* out_scores, int64_t* out_index_, void* workspace,
                                int64_t workspace_bytes, dprb_stream_t stream_) {
  long long* out_index = reinterpret_cast<long long*>(out_index_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(Q > 0 && N > 0 && d > 0, "search: empty problem Q=%lld N=%lld d=%d", (long long)Q, (long long)N, d);
  const int rank_f16 = (dtype & DPRB_SEARCH_RANK_FP16) != 0;
  dtype &= 0xFF;
  DPRB_REQUIRE(dtype == 0 || dtype == 1, "search: dtype must be 0 (fp16) or 1 (bf16), got %d", dtype);
  DPRB_REQUIRE(k >= 1 && k <= 1024, "search: k=%d outside [1, 1024]", k);
  DPRB_REQUIRE(N >= k, "search: k=%d exceeds the %lld corpus rows (torch.topk raises here too)", k, (long long)N);
  DPRB_REQUIRE(N < 0x7FFFFF00ll, "search: %lld corpus rows exceed the 31-bit TMA row coordinate; split into shards",
               (long long)N);
  DPRB_REQUIRE(d % 8 == 0, "search: d=%d must be a multiple of 8 (16-byte rows for TMA)", d);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(queries) & 15) == 0 && (reinterpret_cast<uintptr_t>(corpus) & 15) == 0,
               "search: operands must be 16-byte aligned");
  DPRB_NUM_SMS(sms);
  const WsLayout w = ws_layout(workspace, Q, k, sms);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= w.total,
               "search: workspace %lld B < required %lld B", (long long)workspace_bytes, w.total);

  static bool attr_set = false;
  if (!attr_set) {
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(search_topk_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    DPRB_CHECK_CUDA(cudaFuncSetAttribute(search_topk_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  const int cap = cap_for_k(k);
  const long long tiles = (N + CT - 1) / CT;
  CUtensorMap tc;
  if (int rc = make_tmap(&tc, corpus, N, d, CT, dtype)) return rc;
  const long long qtiles_total = (Q + QT - 1) / QT;
  for (long long qt0 = 0; qt0 < qtiles_total; qt0 += MAX_QTILES) {
    const int nb = (int)((qtiles_total - qt0) < MAX_QTILES ? (qtiles_total - qt0) : MAX_QTILES);
    const long long qbase = qt0 * QT;
    const int Qb = (int)((Q - qbase) < (long long)nb * QT ? (Q - qbase) : (long long)nb * QT);
    long long parts = sms / nb;
    if (parts > tiles) parts = tiles;
    if (parts < 1) parts = 1;
    const long long tpp = (tiles + parts - 1) / parts;
    parts = (tiles + tpp - 1) / tpp;                                  // no empty partitions
    CUtensorMap tq;
    const uint8_t* qptr = static_cast<const uint8_t*>(queries) + (size_t)qbase * d * 2;
    if (int rc = make_tmap(&tq, qptr, Qb, d, QT, dtype)) return rc;
    SearchParams sp;
    sp.N = N; sp.Q = Qb; sp.d = d; sp.k = k; sp.kblocks = (d + BK - 1) / BK;
    sp.tiles = tiles; sp.tiles_per_part = tpp; sp.queues = w.queues; sp.counts = w.counts;
    sp.f16 = dtype == 0 ? 1 : 0;
    sp.rank_f16 = rank_f16;
    const long long m = (k + parts - 1) / parts;
    sp.bounds = w.bounds;
    sp.m_track = m <= 8 ? (int)m : 0;
    if (sp.m_track > 0)
      DPRB_CHECK_CUDA(cudaMemsetAsync(w.bounds, 0, (size_t)parts * nb * QT * sizeof(uint32_t), stream));
    dim3 grid((unsigned)parts, (unsigned)nb);
    if (cap == 512) search_topk_kernel<16><<<grid, THREADS, SMEM_BYTES, stream>>>(tq, tc, sp);
    else search_topk_kernel<64><<<grid, THREADS, SMEM_BYTES, stream>>>(tq, tc, sp);
    DPRB_LAUNCH_CHECK();
    SelectParams sl;
    const long long qpad = (long long)nb * QT;
    sl.lists = w.queues; sl.counts = w.counts; sl.num_lists = (int)parts;
    sl.list_stride = qpad * cap; sl.query_stride = cap; sl.count_stride = qpad; sl.fixed_count = 0;
    sl.k = k; sl.kpad = kpad_for(k); sl.index_offset = index_offset;
    sl.out_scores = out_scores + qbase * k; sl.out_index = out_index + qbase * k;
    sl.scratch = w.scratch; sl.scratch_per_query = w.scratch_per_query;
    sl.gather = nullptr; sl.gather_stride = 0;
    if (int rc = launch_select(sl, Qb, stream)) return rc;
  }
  return 0;
}

extern "C" int64_t dprb_topk_merge_workspace_bytes(int64_t Q, int total) {
  Carve c(nullptr);
  c.take(Q * total * (long long)sizeof(u64));
  return c.off;
}

extern "C" int dprb_topk_merge(const float* scores, const int64_t* index_, int64_t Q, int total, int k,
                               float* out_scores, int64_t* out_index_, void* workspace, int64_t workspace_bytes,
                               dprb_stream_t stream_) {
  const long long* index = reinterpret_cast<const long long*>(index_);
  long long* out_index = reinterpret_cast<long long*>(out_index_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(Q > 0 && total > 0, "topk_merge: empty problem Q=%lld total=%d", (long long)Q, total);
  DPRB_REQUIRE(k >= 1 && k <= 1024 && k <= total, "topk_merge: k=%d outside [1, min(1024, %d)]", k, total);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= dprb_topk_merge_workspace_bytes(Q, total),
               "topk_merge: workspace %lld B < required %lld B", (long long)workspace_bytes,
               (long long)dprb_topk_merge_workspace_bytes(Q, total));
  u64* keys = static_cast<u64*>(workspace);
  const long long n = Q * total;
  pack_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(scores, keys, n, total);
  DPRB_LAUNCH_CHECK();
  SelectParams sl;
  sl.lists = keys; sl.counts = nullptr; sl.num_lists = 1; sl.list_stride = 0; sl.query_stride = total;
  sl.count_stride = 0; sl.fixed_count = total; sl.k = k; sl.kpad = kpad_for(k); sl.index_offset = 0;
  sl.out_scores = out_scores; sl.out_index = out_index;
  // candidates beyond the shared-memory staging area are selected in place from the packed keys (read-only use)
  sl.scratch = keys; sl.scratch_per_query = total;
  sl.gather = index; sl.gather_stride = total;
  return launch_select(sl, Q, stream);
}
