// Group the kept (token, expert) entries of one encoded COIL / CITADEL batch by expert, forward only:
//
//   entry i = (n, s, k), i = (n * S + s) * K + k, is kept when s >= 1, mask[n, s] != 0 and
//             w[i] > threshold                                  (the weight test is skipped in context-id mode)
//   kept entries are written sorted by expert (per-sequence mode: by (n, expert)), ties in (n, s, k) order, with
//   their expert, n, s, w[i] and payload w[i] * float(reps[n, s, :P])  (context-id mode: float(tokens[n, s]))
//
// Replaces the per-entry Python loops of GenerateMultiVecEmbeddingsTask._eval_step / test_epoch_end and
// GenerateMultiVecQueryEmbeddingsTask._eval_step (dpr_scale/task/citadel_eval_task.py:43-70, :95-102, :143-171),
// which append one list entry per kept entry to a dict keyed by expert.  Their iteration order is (n, s, k), so within
// an expert the entries stay in that order; (key, entry index) is unique and the output fully determined.
//
// Design: a stable LSD radix sort over 8-bit digits of the key, only over the bits the key needs (ceil(log2 V), plus
// ceil(log2 N) in per-sequence mode, where the sequence digits are sorted last).  Items are (expert, entry index)
// pairs.  Each pass is three launches over tiles of 1024 items: a per-tile 256-bin histogram (shared-memory counters;
// per-digit totals by integer atomics, so exact), one scan per digit row of the [256][tiles] histogram (digit base =
// sum of the smaller digits' totals), and a stable scatter: within a round of 256 items each warp ranks equal digits
// with __match_any_sync, earlier warps' counts come from shared memory, and a running per-digit offset carries over
// the tile's four rounds.  The keep rule is applied by the first pass, which reads the raw entries, so dropped
// entries are never moved.  The kept count lands in `count` after the first scan; later launches read it from there
// and tiles beyond it do nothing, so the host never waits.  A final gather writes the outputs: per-entry metadata one
// thread per entry, payload rows by groups of lanes (16-byte bf16 loads, fp32 products rounded once, coalesced
// 32-byte stores per lane).  Integer counting only, so the output is bitwise repeatable.
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {
namespace {

constexpr int THREADS = 256, ITEMS = 4, TILE = THREADS * ITEMS, WARPS = THREADS / 32;
constexpr int RADIX = 256;              // one histogram bin per thread of a tile
constexpr int MAX_PASSES = 7;           // 24 expert bits + 31 sequence bits, 8 per pass
constexpr int MAX_K = 8, MAX_S = 512, MAX_P = 1024;
static_assert(THREADS == RADIX, "the histogram and scatter kernels give each thread one digit");

struct GroupParams {
  const int32_t* ids;      // [N, S, K]
  const float* w;          // [N, S, K]
  const int32_t* mask;     // [N, S]
  const int32_t* tokens;   // [N, S] (context-id mode only)
  int N, S, K, SK;         // SK = S * K
  float threshold;
  int context_id;
  int total;               // N * S * K
  int tiles;               // ceil(total / TILE)
  int vpasses;             // passes over the expert id's digits; the sequence's follow
};

// (expert, entry index) of raw entry i when it is kept
__device__ __forceinline__ bool keep_entry(const GroupParams& p, int i, int2& item) {
  const int n = i / p.SK, rem = i - n * p.SK, s = rem / p.K;
  if (s == 0 || __ldg(p.mask + n * p.S + s) == 0) return false;
  if (!p.context_id && !(__ldg(p.w + i) > p.threshold)) return false;
  item = make_int2(__ldg(p.ids + i), i);
  return true;
}

__device__ __forceinline__ int digit_of(const GroupParams& p, int2 item, int pass) {
  const int key = pass < p.vpasses ? item.x : item.y / p.SK;
  const int shift = 8 * (pass < p.vpasses ? pass : pass - p.vpasses);
  return (key >> shift) & (RADIX - 1);
}

// the item at position pos of this pass's input (pass 0: raw entry pos); false when there is none or it is dropped
__device__ __forceinline__ bool load_item(const GroupParams& p, const int2* in, int n_items, int pass, long long pos,
                                          int2& item) {
  if (pos >= n_items) return false;
  if (pass == 0) return keep_entry(p, (int)pos, item);
  item = in[pos];
  return true;
}

// block-wide inclusive scan of one int per thread (THREADS threads); returns the block total in `sum`
__device__ __forceinline__ int block_incl_scan(int v, int& sum) {
  __shared__ int warp_tot[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) warp_tot[warp] = v;
  __syncthreads();
  int before = 0;
  sum = 0;
#pragma unroll
  for (int w = 0; w < WARPS; ++w) {
    const int t = warp_tot[w];
    if (w < warp) before += t;
    sum += t;
  }
  __syncthreads();                                   // warp_tot is reused by the next call
  return v + before;
}

__global__ void __launch_bounds__(THREADS)
group_hist_kernel(const GroupParams p, const int2* in, const int* count, int pass, int* hist, int* totals) {
  __shared__ int h[RADIX];
  const int t = threadIdx.x;
  h[t] = 0;
  __syncthreads();
  const int n_items = pass == 0 ? p.total : *count;
  const long long base = (long long)blockIdx.x * TILE;
#pragma unroll
  for (int j = 0; j < ITEMS; ++j) {
    int2 item;
    if (load_item(p, in, n_items, pass, base + j * THREADS + t, item)) atomicAdd(&h[digit_of(p, item, pass)], 1);
  }
  __syncthreads();
  const int c = h[t];
  hist[(long long)t * p.tiles + blockIdx.x] = c;
  if (c) atomicAdd(totals + pass * RADIX + t, c);
}

// block d: exclusive scan of histogram row d (one count per tile) plus the items of all smaller digits
__global__ void __launch_bounds__(THREADS)
group_scan_kernel(int* hist, const int* totals, int tiles, int pass, int* count) {
  __shared__ int s_base;
  const int d = blockIdx.x, t = threadIdx.x;
  const int tot = totals[pass * RADIX + t];
  int all;
  const int incl = block_incl_scan(tot, all);
  if (t == d) s_base = incl - tot;                   // items of the digits below d
  __syncthreads();
  int base = s_base;
  if (pass == 0 && d == 0 && t == 0) *count = all;
  int* row = hist + (long long)d * tiles;
  for (int r = 0; r < tiles; r += THREADS) {
    const int idx = r + t;
    const int x = idx < tiles ? row[idx] : 0;
    int sum;
    const int incl = block_incl_scan(x, sum);
    if (idx < tiles) row[idx] = base + incl - x;
    base += sum;
  }
}

__global__ void __launch_bounds__(THREADS)
group_scatter_kernel(const GroupParams p, const int2* in, const int* count, int pass, const int* hist, int2* out) {
  __shared__ int run[RADIX];
  __shared__ int wcnt[WARPS][RADIX];
  const int n_items = pass == 0 ? p.total : *count;
  const long long base = (long long)blockIdx.x * TILE;
  if (base >= n_items) return;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  run[t] = hist[(long long)t * p.tiles + blockIdx.x];
#pragma unroll
  for (int w = 0; w < WARPS; ++w) wcnt[w][t] = 0;
  __syncthreads();
  const unsigned lt_mask = (1u << lane) - 1u;
#pragma unroll 1
  for (int j = 0; j < ITEMS; ++j) {
    int2 item;
    const bool valid = load_item(p, in, n_items, pass, base + j * THREADS + t, item);
    const int dg = valid ? digit_of(p, item, pass) : RADIX;          // RADIX: groups the lanes without an item
    const unsigned peers = __match_any_sync(0xffffffffu, dg);
    const int rank = __popc(peers & lt_mask);
    if (valid && rank == 0) wcnt[warp][dg] = __popc(peers);
    __syncthreads();
    if (valid) {
      int off = run[dg] + rank;
      for (int w = 0; w < warp; ++w) off += wcnt[w][dg];
      out[off] = item;
    }
    __syncthreads();
    int s = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      s += wcnt[w][t];
      wcnt[w][t] = 0;
    }
    run[t] += s;
    __syncthreads();
  }
}

// G lanes per payload row (a power of two, at most 32, at most P / 8 chunks of 8 columns)
__global__ void __launch_bounds__(THREADS)
group_gather_kernel(const GroupParams p, const int2* items, const int* count, const bf16* reps, long long ldr, int P,
                    int G, int32_t* o_expert, int32_t* o_seq, int32_t* o_tok, float* o_w, float* o_payload) {
  const int E = *count;
  const long long tid = (long long)blockIdx.x * THREADS + threadIdx.x, nthreads = (long long)gridDim.x * THREADS;
  for (long long e = tid; e < E; e += nthreads) {
    const int2 it = items[e];
    const int n = it.y / p.SK, s = (it.y - n * p.SK) / p.K;
    o_expert[e] = it.x;
    o_seq[e] = n;
    o_tok[e] = s;
    o_w[e] = __ldg(p.w + it.y);
    if (p.context_id) o_payload[e] = (float)__ldg(p.tokens + n * p.S + s);
  }
  if (p.context_id) return;
  const int sub = threadIdx.x % G;
  const long long grp = tid / G, ngrp = nthreads / G;
  for (long long e = grp; e < E; e += ngrp) {
    const int i = items[e].y;
    const int n = i / p.SK, s = (i - n * p.SK) / p.K;
    const float wv = __ldg(p.w + i);
    const bf16* row = reps + ((long long)n * p.S + s) * ldr;
    float* orow = o_payload + e * P;
    for (int c = sub * 8; c < P; c += G * 8) {
      const uint4 u = ldg_nc_v4(row + c);
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c2 = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
      float4* o = reinterpret_cast<float4*>(orow + c);
      o[0] = make_float4(__fmul_rn(wv, a.x), __fmul_rn(wv, a.y), __fmul_rn(wv, b.x), __fmul_rn(wv, b.y));
      o[1] = make_float4(__fmul_rn(wv, c2.x), __fmul_rn(wv, c2.y), __fmul_rn(wv, d.x), __fmul_rn(wv, d.y));
    }
  }
}

int bits_for(long long v) {                             // bits needed to hold every value in [0, v)
  int b = 0;
  while ((1LL << b) < v) ++b;
  return b;
}

struct Layout {
  void *items_a, *items_b, *hist, *totals;
  long long bytes;
};

Layout carve(void* ws, long long total, int tiles) {
  Carve c(ws);
  Layout l;
  l.items_a = c.take(total * 8);
  l.items_b = c.take(total * 8);
  l.hist = c.take((long long)RADIX * tiles * 4);
  l.totals = c.take((long long)MAX_PASSES * RADIX * 4);
  l.bytes = c.off;
  return l;
}

}  // namespace
}  // namespace dprb

using namespace dprb;

extern "C" int64_t dprb_expert_group_workspace_bytes(int N, int S, int K) {
  if (N < 1 || S < 1 || K < 1) return 0;
  const long long total = (long long)N * S * K;
  if (total >= (1LL << 31)) return -1;
  return carve(nullptr, total, (int)((total + TILE - 1) / TILE)).bytes;
}

extern "C" int dprb_expert_group(const int32_t* ids, const float* w, const int32_t* mask, const int32_t* tokens,
                                 const void* reps, int64_t ldr, int N, int S, int K, int P, int V, float threshold,
                                 int flags, int32_t* count, int32_t* out_expert, int32_t* out_seq, int32_t* out_tok,
                                 float* out_w, float* out_payload, void* workspace, int64_t workspace_bytes,
                                 dprb_stream_t stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool ctx_id = (flags & DPRB_EXPERT_GROUP_CONTEXT_ID) != 0;
  const bool per_seq = (flags & DPRB_EXPERT_GROUP_PER_SEQUENCE) != 0;
  DPRB_REQUIRE((flags & ~(DPRB_EXPERT_GROUP_CONTEXT_ID | DPRB_EXPERT_GROUP_PER_SEQUENCE)) == 0,
               "expert_group: unknown flags 0x%x", flags);
  DPRB_REQUIRE(N >= 1 && K >= 1 && K <= MAX_K && S >= 2 && S <= MAX_S,
               "expert_group: N=%d S=%d K=%d unsupported (N >= 1, 2 <= S <= %d, 1 <= K <= %d)", N, S, K, MAX_S, MAX_K);
  const long long total = (long long)N * S * K;
  DPRB_REQUIRE(total < (1LL << 31), "expert_group: N*S*K=%lld entries reach 2^31", total);
  DPRB_REQUIRE(V >= 1 && V < (1 << 24), "expert_group: V=%d outside [1, 2^24)", V);
  DPRB_REQUIRE(ids != nullptr && w != nullptr && mask != nullptr && count != nullptr && out_expert != nullptr &&
               out_seq != nullptr && out_tok != nullptr && out_w != nullptr && out_payload != nullptr,
               "expert_group: NULL operand");
  if (ctx_id) {
    DPRB_REQUIRE(tokens != nullptr, "expert_group: context-id mode needs the token ids");
  } else {
    DPRB_REQUIRE(P % 8 == 0 && P >= 8 && P <= MAX_P, "expert_group: P=%d unsupported (multiple of 8, 8 .. %d)", P,
                 MAX_P);
    DPRB_REQUIRE(reps != nullptr && ldr >= P && ldr % 8 == 0, "expert_group: reps NULL or ldr=%lld (>= P=%d, multiple "
                 "of 8)", (long long)ldr, P);
    DPRB_REQUIRE(((reinterpret_cast<uintptr_t>(reps) | reinterpret_cast<uintptr_t>(out_payload)) & 15) == 0,
                 "expert_group: reps / payload must be 16-byte aligned");
  }
  const int tiles = (int)((total + TILE - 1) / TILE);
  const Layout l = carve(workspace, total, tiles);
  DPRB_REQUIRE(workspace != nullptr && workspace_bytes >= l.bytes,
               "expert_group: workspace of %lld bytes, %lld needed (dprb_expert_group_workspace_bytes)",
               (long long)workspace_bytes, l.bytes);
  DPRB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "expert_group: workspace must be 256-byte aligned");
  DPRB_NUM_SMS(sms);

  GroupParams p;
  p.ids = ids; p.w = w; p.mask = mask; p.tokens = tokens;
  p.N = N; p.S = S; p.K = K; p.SK = S * K;
  p.threshold = threshold;
  p.context_id = ctx_id ? 1 : 0;
  p.total = (int)total;
  p.tiles = tiles;
  p.vpasses = (bits_for(V) + 7) / 8;
  if (p.vpasses == 0) p.vpasses = 1;                 // the first pass also filters
  const int passes = p.vpasses + (per_seq ? (bits_for(N) + 7) / 8 : 0);

  int* hist = static_cast<int*>(l.hist);
  int* totals = static_cast<int*>(l.totals);
  DPRB_CHECK_CUDA(cudaMemsetAsync(totals, 0, (size_t)MAX_PASSES * RADIX * 4, stream));
  int2* src = static_cast<int2*>(l.items_b);
  int2* dst = static_cast<int2*>(l.items_a);
  for (int pass = 0; pass < passes; ++pass) {
    group_hist_kernel<<<tiles, THREADS, 0, stream>>>(p, src, count, pass, hist, totals);
    DPRB_LAUNCH_CHECK();
    group_scan_kernel<<<RADIX, THREADS, 0, stream>>>(hist, totals, tiles, pass, count);
    DPRB_LAUNCH_CHECK();
    group_scatter_kernel<<<tiles, THREADS, 0, stream>>>(p, src, count, pass, hist, dst);
    DPRB_LAUNCH_CHECK();
    int2* t = src; src = dst; dst = t;
  }
  int G = 1;
  if (!ctx_id)
    while (G < 32 && 2 * G <= P / 8) G *= 2;
  const long long want = ((total + THREADS - 1) / THREADS);
  const int grid = (int)(want < (long long)sms * 8 ? (want > 0 ? want : 1) : (long long)sms * 8);
  group_gather_kernel<<<grid, THREADS, 0, stream>>>(p, src, count, static_cast<const bf16*>(reps), ldr, P, G,
                                                    out_expert, out_seq, out_tok, out_w, out_payload);
  DPRB_LAUNCH_CHECK();
  return 0;
}
