// Retrieval from a COIL / CITADEL expert index, forward only: for every query of a block and every passage row d,
//
//   score(q, d) = cls_q . cls_d                                                     (only with CLS operands)
//               + sum over the query's entries (x, u) of max(0, max over d's index entries (x, v) of u . v)
//
// (the max over an empty set is 0), then the k best rows of each query, ties towards the lower row.  This is the
// stage that consumes the files GenerateMultiVecEmbeddingsTask writes (the reference's CITADELRetrievalTask searches
// them with an inverted vector index that is not part of its tree).
//
// Index (device, built once by the caller): entries sorted by expert, and inside an expert by passage row, so one
// passage's entries of an expert are contiguous (a "run"); payload fp16 [E, ldp].  Posting tiles partition the entries
// without splitting a run (a tile may be longer than one 128-entry chunk; the segmented max carries across chunks).
// The CLS vectors are a second section [N, ldc] whose "tiles" are 128 consecutive rows, with one entry per row and no
// clamp.
//
// Work: a group is <= 64 query rows of one expert (query entries grouped by expert) or 64 queries' CLS vectors, paired
// with every tile of that expert (or every CLS tile); item i of the launch is (group, tile) by a binary search over the
// groups' inclusive prefix sums of tile counts.  Persistent CTAs of one warpgroup take items from an atomic counter.
// Per 128-entry chunk of the tile: cp.async stages of 64 query rows x 64 columns and 128 entries x 64 columns, stored
// 128B-swizzled, two stages in flight; wgmma m64n128k16 (fp16 operands, fp32 accumulators, only the k16 steps that hold
// columns below the width); the fp32 tile goes to shared memory (aliasing the stages) and each of 64 threads walks its
// query row in entry order with a running max, flushing it at every change of passage row.
//
// Accumulation: the flushed term (clamped at 0 for expert entries) is rounded once to int64 fixed point at 2^-32 and
// added into acc[q, d] with a 64-bit integer atomicAdd.  Integer addition is associative, so the sums, and therefore the
// results, do not depend on the order of the atomics: bitwise repeatable, and a query's results do not depend on the
// other queries of its block.  The host bounds every query's sum of |terms| below 2^30 before the launch.
//
// Selection: the k best rows of every query from the accumulator (fixed_select.cu).
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int THREADS = 128;                       // one warpgroup
constexpr int QG = 64;                             // query rows per group (wgmma M)
constexpr int TN = 128;                            // index entries per chunk (wgmma N)
constexpr int BK = 64;                             // columns per stage: one 128-byte swizzle row of fp16
constexpr int A_BYTES = QG * BK * 2;               // 8 KB
constexpr int B_BYTES = TN * BK * 2;               // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int STAGES = 2;
constexpr int S_LD = TN + 4;                       // fp32 score tile [QG][S_LD]
constexpr int TILE_BYTES = QG * S_LD * 4;
constexpr int MAIN_BYTES = STAGES * STAGE_BYTES > TILE_BYTES ? STAGES * STAGE_BYTES : TILE_BYTES;
constexpr int SMEM_BYTES = MAIN_BYTES + (TN + 1) * 4 + QG * 4 + 1024;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget exceeded");
constexpr int MAX_P = 1024;
constexpr float FIX_SCALE = 4294967296.f;          // 2^32

struct SearchParams {
  const __half* pay[2];      // [E, ld0] index payload, [N, ld1] CLS
  const __half* qpay[2];     // [Eq, ld0] query payload, [Qb, ld1] query CLS
  int ld[2], K[2];
  const int32_t* row;        // [E] passage row of each entry
  const int32_t* tile_bounds;  // [T + 1] entry ranges of the index tiles
  const int4* groups;        // [G] (section, first query row, query rows, first tile)
  const int32_t* item_end;   // [G] inclusive prefix sums of the groups' tile counts
  const int32_t* q_seq;      // [Eq] query (in the block) of each query entry
  int G, items;
  long long N;
  unsigned long long* acc;   // [Qb, N] fixed point, 2^-32
  int* counter;
};

// rows [0, rows) of a K-major fp16 matrix (stride ld elements, width K), columns [c0, c0 + 64), into a 128B-swizzled
// [nrows][64] tile; everything beyond `rows` or K is zero
template <int NROWS>
__device__ __forceinline__ void load_tile(uint8_t* dst, const __half* src, long long row0, int rows, int ld, int K,
                                          int c0) {
#pragma unroll
  for (int i = threadIdx.x; i < NROWS * 8; i += THREADS) {
    const int r = i >> 3, c = i & 7;
    const int col = c0 + c * 8;
    const bool ok = r < rows && col < K;
    const __half* g = ok ? src + (row0 + r) * (long long)ld + col : src;
    cp_async_16_zfill(dst + r * 128 + ((c ^ (r & 7)) << 4), g, ok);
  }
}

__global__ void __launch_bounds__(THREADS)
expert_search_kernel(const SearchParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  float* sS = reinterpret_cast<float*>(smem);                              // [QG][S_LD], aliases the stages
  int* sDoc = reinterpret_cast<int*>(smem + MAIN_BYTES);                    // [TN + 1]: rows of the chunk, then next
  int* sQ = sDoc + TN + 1;                                                  // [QG] query of each group row
  __shared__ int s_item;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (;;) {
    if (tid == 0) s_item = atomicAdd(p.counter, 1);
    __syncthreads();
    const int item = s_item;
    if (item >= p.items) break;
    int lo = 0, hi = p.G - 1;                                               // first group with item_end > item
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(p.item_end + mid) > item) hi = mid; else lo = mid + 1;
    }
    const int4 g = __ldg(p.groups + lo);
    const int t = item - (lo > 0 ? __ldg(p.item_end + lo - 1) : 0);
    const int sec = g.x, qlo = g.y, qcnt = g.z;
    long long e0, e1;
    if (sec == 0) {
      e0 = __ldg(p.tile_bounds + g.w + t);
      e1 = __ldg(p.tile_bounds + g.w + t + 1);
    } else {
      e0 = (long long)t * TN;
      e1 = min(e0 + TN, p.N);
    }
    const int K = sec == 0 ? p.K[0] : p.K[1], ld = sec == 0 ? p.ld[0] : p.ld[1];   // no dynamic param indexing
    const __half* A = sec == 0 ? p.qpay[0] : p.qpay[1];
    const __half* B = sec == 0 ? p.pay[0] : p.pay[1];
    if (tid < QG) sQ[tid] = tid < qcnt ? (sec == 0 ? __ldg(p.q_seq + qlo + tid) : qlo + tid) : -1;
    const int kblocks = (K + BK - 1) / BK;
    float m = -INFINITY;                                                    // threads < QG: running max of the row
    for (long long c0 = e0; c0 < e1; c0 += TN) {
      const int ncols = (int)min((long long)TN, e1 - c0);
      float acc[64];
      load_tile<QG>(smem, A, qlo, qcnt, ld, K, 0);
      load_tile<TN>(smem + A_BYTES, B, c0, ncols, ld, K, 0);
      cp_async_commit();
      for (int kb = 0; kb < kblocks; ++kb) {
        if (kb + 1 < kblocks) {
          uint8_t* st = smem + ((kb + 1) & 1) * STAGE_BYTES;
          load_tile<QG>(st, A, qlo, qcnt, ld, K, (kb + 1) * BK);
          load_tile<TN>(st + A_BYTES, B, c0, ncols, ld, K, (kb + 1) * BK);
          cp_async_commit();
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        fence_proxy_async_smem();
        __syncthreads();
        const uint32_t base = smem_u32(smem + (kb & 1) * STAGE_BYTES);
        const uint64_t da = make_wgmma_desc_sw128(base, 16, 1024);
        const uint64_t db = make_wgmma_desc_sw128(base + A_BYTES, 16, 1024);
        const int ksteps = min(BK / 16, (K - kb * BK + 15) / 16);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          if (k < ksteps) wgmma_m64n128_ss_f16<0, 0>(acc, da + 2 * k, db + 2 * k, (kb > 0 || k > 0) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        __syncthreads();                                                    // the stage may be refilled
      }
      {                                                                     // registers -> [QG][S_LD]
        const int r0 = warp * 16 + (lane >> 2), q4 = lane & 3;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          float* a0 = sS + r0 * S_LD + 8 * c + 2 * q4;
          *reinterpret_cast<float2*>(a0) = make_float2(acc[4 * c], acc[4 * c + 1]);
          *reinterpret_cast<float2*>(a0 + 8 * S_LD) = make_float2(acc[4 * c + 2], acc[4 * c + 3]);
        }
      }
      for (int j = tid; j <= ncols; j += THREADS) {
        const long long e = c0 + j;
        int d = -1;
        if (e < e1) d = sec == 0 ? __ldg(p.row + e) : (int)e;
        sDoc[j] = d;
      }
      __syncthreads();
      if (tid < QG) {
        const int qi = sQ[tid];
        const float* srow = sS + tid * S_LD;
        unsigned long long* arow = qi >= 0 ? p.acc + (long long)qi * p.N : nullptr;
        int d = sDoc[0];
        for (int j = 0; j < ncols; ++j) {
          m = fmaxf(m, srow[j]);
          const int nd = sDoc[j + 1];
          if (nd != d) {                                                    // the run of row d ends here
            const float v = sec == 0 ? fmaxf(m, 0.f) : m;
            const long long f = __float2ll_rn(v * FIX_SCALE);
            if (arow != nullptr && f != 0) atomicAdd(arow + d, (unsigned long long)f);
            m = -INFINITY;
            d = nd;
          }
        }
      }
      __syncthreads();                                                      // sS / sDoc are rewritten next chunk
    }
  }
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_expert_search_block_queries(int64_t N) { return fixed_acc_block_queries(N); }

extern "C" int64_t dprb_expert_search_workspace_bytes(int64_t N, int Qb) { return fixed_acc_workspace_bytes(N, Qb); }

extern "C" int dprb_expert_search(const void* payload, const int32_t* row, const int32_t* tile_bounds, int64_t E, int T,
                                  int P, int ldp, const void* cls, int Pc, int ldc, const int64_t* row_ids_, int64_t N,
                                  const void* q_payload, const int32_t* q_seq, int64_t Eq, const void* q_cls, int Qb,
                                  const int32_t* groups, const int32_t* item_end, int G, int items, int k,
                                  float* out_scores, int64_t* out_ids_, void* workspace, int64_t workspace_bytes,
                                  dprb_stream_t stream_) {
  const long long* row_ids = reinterpret_cast<const long long*>(row_ids_);
  long long* out_ids = reinterpret_cast<long long*>(out_ids_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(P % 8 == 0 && P >= 8 && P <= MAX_P && ldp >= P && ldp % 8 == 0,
               "expert_search: P=%d ldp=%d unsupported (P a multiple of 8, 8 .. %d; ldp >= P, a multiple of 8)", P,
               ldp, MAX_P);
  DPRB_REQUIRE(N >= 1 && N < (1LL << 31), "expert_search: N=%lld passages outside [1, 2^31)", (long long)N);
  DPRB_REQUIRE(E >= 0 && E < (1LL << 31) && Eq >= 0 && Eq < (1LL << 31),
               "expert_search: E=%lld index entries or Eq=%lld query entries outside [0, 2^31)", (long long)E,
               (long long)Eq);
  DPRB_REQUIRE(T >= 0 && G >= 0 && items >= 0 && (G > 0 || items == 0),
               "expert_search: T=%d tiles, G=%d groups, %d work items", T, G, items);
  DPRB_REQUIRE(k >= 1 && k <= 1024 && k <= N, "expert_search: k=%d outside [1, min(1024, N=%lld)]", k, (long long)N);
  DPRB_REQUIRE(Qb >= 1 && Qb <= dprb_expert_search_block_queries(N),
               "expert_search: Qb=%d queries per block outside [1, %d] (dprb_expert_search_block_queries)", Qb,
               dprb_expert_search_block_queries(N));
  DPRB_REQUIRE((cls == nullptr) == (q_cls == nullptr), "expert_search: give both CLS operands or neither");
  if (cls != nullptr)
    DPRB_REQUIRE(Pc % 8 == 0 && Pc >= 8 && Pc <= MAX_P && ldc >= Pc && ldc % 8 == 0,
                 "expert_search: Pc=%d ldc=%d unsupported (Pc a multiple of 8, 8 .. %d; ldc >= Pc, a multiple of 8)",
                 Pc, ldc, MAX_P);
  DPRB_REQUIRE(G == 0 || (groups != nullptr && item_end != nullptr), "expert_search: NULL group operand");
  DPRB_REQUIRE(Eq == 0 || (q_payload != nullptr && q_seq != nullptr && payload != nullptr && row != nullptr &&
                           tile_bounds != nullptr),
               "expert_search: NULL index or query operand");
  DPRB_REQUIRE(out_scores != nullptr && out_ids != nullptr, "expert_search: NULL output");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(payload) | reinterpret_cast<uintptr_t>(q_payload) |
                 reinterpret_cast<uintptr_t>(cls) | reinterpret_cast<uintptr_t>(q_cls)) & 15) == 0,
               "expert_search: payloads must be 16-byte aligned");
  const long long need = dprb_expert_search_workspace_bytes(N, Qb);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
               "expert_search: workspace of %lld bytes (256-byte aligned), %lld needed", (long long)workspace_bytes, need);
  DPRB_NUM_SMS(sms);

  FixedAcc fa;
  if (const int rc = fixed_acc_init(workspace, N, Qb, &fa, stream)) return rc;
  if (items > 0) {
    static bool attr_done = false;
    if (!attr_done) {
      DPRB_CHECK_CUDA(cudaFuncSetAttribute(expert_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           SMEM_BYTES));
      attr_done = true;
    }
    int per_sm = 0;
    DPRB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, expert_search_kernel, THREADS, SMEM_BYTES));
    if (per_sm < 1) per_sm = 1;
    SearchParams sp;
    sp.pay[0] = static_cast<const __half*>(payload);
    sp.pay[1] = static_cast<const __half*>(cls);
    sp.qpay[0] = static_cast<const __half*>(q_payload);
    sp.qpay[1] = static_cast<const __half*>(q_cls);
    sp.ld[0] = ldp; sp.ld[1] = ldc; sp.K[0] = P; sp.K[1] = Pc;
    sp.row = row; sp.tile_bounds = tile_bounds;
    sp.groups = reinterpret_cast<const int4*>(groups);
    sp.item_end = item_end; sp.q_seq = q_seq;
    sp.G = G; sp.items = items; sp.N = N; sp.acc = fa.acc; sp.counter = fa.counter;
    const long long want = (long long)sms * per_sm;
    const int grid = (int)(items < want ? items : want);
    expert_search_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(sp);
    DPRB_LAUNCH_CHECK();
  }
  return fixed_acc_select(fa.acc, N, Qb, k, row_ids, out_scores, out_ids, stream);
}
