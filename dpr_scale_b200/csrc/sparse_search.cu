// Retrieval from a sparse vocabulary index (SPLADE), forward only: for every query of a block and every passage row d,
//
//   score(q, d) = sum over q's entries (t, w_q) of sum over d's postings (t, w_p) of w_q * w_p
//
// then the k best rows of each query, ties towards the lower row.
//
// Index (device, built once by the caller): postings sorted by term and, inside a term, by passage row; row int32 and
// weight fp16 [nnz], term_ptr int64 [V + 1].  Both posting arrays hold a multiple of 8 entries and are 16-byte aligned,
// so a lane reads 8 postings with two 16-byte loads of rows and one of weights.  A term's postings are cut into tiles of
// TILE entries, so one very common term does not serialize the launch.
//
// Work: item i of the launch is (query entry e, tile j of e's term), found by a binary search over the entries'
// inclusive prefix sums of tile counts.  Persistent CTAs of 8 warps; each warp takes items from an atomic counter and
// its lanes stream the tile's postings 8 at a time (one 256-posting span per warp step, coalesced).
//
// Accumulation: w_q * w_p is formed in fp32, rounded once to int64 fixed point at 2^-32 and added into acc[q, row] with
// a 64-bit integer atomicAdd.  Integer addition is associative, so the results are bitwise repeatable and a query's
// results do not depend on the other queries of its block.  The host bounds every query's sum of |terms| below 2^30.
//
// Selection: the k best rows of every query from the accumulator (fixed_select.cu).
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int THREADS = 256;
constexpr int TILE = DPRB_SPARSE_SEARCH_TILE;      // postings per work item
constexpr float FIX_SCALE = 4294967296.f;          // 2^32
static_assert(TILE % 256 == 0, "a tile is whole warp steps of 8 postings per lane");

struct SparseParams {
  const int32_t* row;          // [nnz, padded to 8] passage row of each posting
  const __half* weight;        // [nnz, padded to 8]
  const long long* term_ptr;   // [V + 1]
  const int32_t* q_term;       // [Eq] term of each query entry
  const float* q_weight;       // [Eq]
  const int32_t* q_seq;        // [Eq] query (in the block) of each entry
  const int32_t* item_end;     // [Eq] inclusive prefix sums of the entries' tile counts
  int Eq, items;
  long long N;
  unsigned long long* acc;     // [Qb, N] fixed point, 2^-32
  int* counter;
};

__global__ void __launch_bounds__(THREADS)
sparse_search_kernel(const SparseParams p) {
  const int lane = threadIdx.x & 31;
  for (;;) {
    // unsigned: every warp takes one item past the end, so the counter may pass 2^31 - 1 when items is close to it
    unsigned next = 0;
    if (lane == 0) next = atomicAdd(reinterpret_cast<unsigned*>(p.counter), 1u);
    next = __shfl_sync(0xffffffffu, next, 0);
    if (next >= (unsigned)p.items) break;
    const int item = (int)next;
    int lo = 0, hi = p.Eq - 1;                                              // first entry with item_end > item
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(p.item_end + mid) > item) hi = mid; else lo = mid + 1;
    }
    const int t = item - (lo > 0 ? __ldg(p.item_end + lo - 1) : 0);
    const int term = __ldg(p.q_term + lo);
    const float wq = __ldg(p.q_weight + lo);
    unsigned long long* arow = p.acc + (long long)__ldg(p.q_seq + lo) * p.N;
    const long long p0 = __ldg(p.term_ptr + term) + (long long)t * TILE;
    const long long p1 = min(p0 + TILE, __ldg(p.term_ptr + term + 1));
    for (long long g = (p0 & ~7LL) + 8 * lane; g < p1; g += 256) {
      const int4 r0 = __ldg(reinterpret_cast<const int4*>(p.row + g));
      const int4 r1 = __ldg(reinterpret_cast<const int4*>(p.row + g + 4));
      const uint4 wv = __ldg(reinterpret_cast<const uint4*>(p.weight + g));
      const int r[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
      const __half* w = reinterpret_cast<const __half*>(&wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (g + j < p0 || g + j >= p1) continue;
        const long long f = __float2ll_rn(wq * __half2float(w[j]) * FIX_SCALE);
        if (f != 0) atomicAdd(arow + r[j], (unsigned long long)f);
      }
    }
  }
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int dprb_sparse_search_block_queries(int64_t N) { return fixed_acc_block_queries(N); }

extern "C" int64_t dprb_sparse_search_workspace_bytes(int64_t N, int Qb) { return fixed_acc_workspace_bytes(N, Qb); }

extern "C" int dprb_sparse_search(const int32_t* row, const void* weight, const int64_t* term_ptr_, int64_t nnz, int V,
                                  const int64_t* row_ids_, int64_t N, const int32_t* q_term, const float* q_weight,
                                  const int32_t* q_seq, const int32_t* item_end, int Eq, int items, int Qb, int k,
                                  float* out_scores, int64_t* out_ids_, void* workspace, int64_t workspace_bytes,
                                  dprb_stream_t stream_) {
  const long long* term_ptr = reinterpret_cast<const long long*>(term_ptr_);
  const long long* row_ids = reinterpret_cast<const long long*>(row_ids_);
  long long* out_ids = reinterpret_cast<long long*>(out_ids_);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DPRB_REQUIRE(N >= 1 && N < (1LL << 31), "sparse_search: N=%lld passages outside [1, 2^31)", (long long)N);
  DPRB_REQUIRE(V >= 1, "sparse_search: V=%d terms, at least 1 needed", V);
  DPRB_REQUIRE(nnz >= 0 && nnz < (1LL << 40), "sparse_search: nnz=%lld postings outside [0, 2^40)", (long long)nnz);
  DPRB_REQUIRE(Eq >= 0 && items >= 0 && (Eq > 0 || items == 0),
               "sparse_search: Eq=%d query entries, %d work items", Eq, items);
  DPRB_REQUIRE(k >= 1 && k <= 1024 && k <= N, "sparse_search: k=%d outside [1, min(1024, N=%lld)]", k, (long long)N);
  DPRB_REQUIRE(Qb >= 1 && Qb <= dprb_sparse_search_block_queries(N),
               "sparse_search: Qb=%d queries per block outside [1, %d] (dprb_sparse_search_block_queries)", Qb,
               dprb_sparse_search_block_queries(N));
  DPRB_REQUIRE(term_ptr != nullptr, "sparse_search: NULL term_ptr");
  DPRB_REQUIRE(nnz == 0 || (row != nullptr && weight != nullptr), "sparse_search: NULL posting operand");
  DPRB_REQUIRE(Eq == 0 || (q_term != nullptr && q_weight != nullptr && q_seq != nullptr && item_end != nullptr),
               "sparse_search: NULL query operand");
  DPRB_REQUIRE(out_scores != nullptr && out_ids != nullptr, "sparse_search: NULL output");
  DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(row) | reinterpret_cast<uintptr_t>(weight)) & 15) == 0,
               "sparse_search: posting arrays must be 16-byte aligned");
  const long long need = dprb_sparse_search_workspace_bytes(N, Qb);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
               "sparse_search: workspace of %lld bytes (256-byte aligned), %lld needed", (long long)workspace_bytes, need);
  DPRB_NUM_SMS(sms);

  FixedAcc fa;
  if (const int rc = fixed_acc_init(workspace, N, Qb, &fa, stream)) return rc;
  if (items > 0 && nnz > 0) {
    int per_sm = 0;
    DPRB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sparse_search_kernel, THREADS, 0));
    if (per_sm < 1) per_sm = 1;
    SparseParams sp;
    sp.row = row;
    sp.weight = static_cast<const __half*>(weight);
    sp.term_ptr = term_ptr;
    sp.q_term = q_term; sp.q_weight = q_weight; sp.q_seq = q_seq; sp.item_end = item_end;
    sp.Eq = Eq; sp.items = items; sp.N = N; sp.acc = fa.acc; sp.counter = fa.counter;
    const long long want = (long long)sms * per_sm;
    const long long blocks = (items + THREADS / 32 - 1) / (THREADS / 32);
    const int grid = (int)(blocks < want ? blocks : want);
    sparse_search_kernel<<<grid, THREADS, 0, stream>>>(sp);
    DPRB_LAUNCH_CHECK();
  }
  return fixed_acc_select(fa.acc, N, Qb, k, row_ids, out_scores, out_ids, stream);
}
