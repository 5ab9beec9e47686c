// Internal C++ declarations shared by the kernel translation units of libdprb.so: only what one file calls in another
// and include/dprb.h does not declare.  Every dprb_* entry point is defined in the file that holds its kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/dprb.h"

namespace dprb {

// host.cu: a tiled tensor map of rank 2 or 3 (dims, box: innermost first; strides: bytes, rank - 1 of them), always
// 128B-swizzled, non-interleaved, out-of-bounds elements read as zero.  Binds the primary context to the calling
// thread first.  Returns 0, or an error code with the message set (`what` names the caller in it).
int encode_tmap(CUtensorMap* out, const char* what, CUtensorMapDataType dtype, int rank, const void* base,
                const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                CUtensorMapL2promotion l2);

// Bump allocator over a caller-owned workspace: every buffer starts 256-byte aligned.  With a null base it only
// measures (take returns null, off still grows), which is how the *_workspace_bytes functions size a workspace.
struct Carve {
  uint8_t* base;
  long long off;
  explicit Carve(void* b) : base(reinterpret_cast<uint8_t*>(b)), off(0) {}
  void* take(long long bytes) {
    void* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~255LL;
    return p;
  }
};

int attn_fwd_wg(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                float dropout_p, unsigned long long site_seed, cudaStream_t stream);
// adds the QKV bias gradient into dbias when it is given
int attn_bwd_wg(const void* qkv, const int32_t* attn_mask, const float* lse, const void* dctx,
                void* dqkv, float* dbias, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                cudaStream_t stream);

int add_rows_bf16(void* dst, const void* src, int nrows, int H, long long stride_rows, cudaStream_t stream);

// fixed_select.cu: the int64 fixed-point accumulator [Qb, N] at 2^-32 of the index searches, and its per-query top-k.
// fixed_acc_init carves the accumulator and a work counter from the workspace and zeroes both on the stream;
// fixed_acc_select writes the k best rows of every query (descending, ties towards the lower row), as row_ids[row].
struct FixedAcc {
  unsigned long long* acc;
  int* counter;
};
int fixed_acc_block_queries(long long N);
long long fixed_acc_workspace_bytes(long long N, int Qb);
int fixed_acc_init(void* workspace, long long N, int Qb, FixedAcc* out, cudaStream_t stream);
int fixed_acc_select(const unsigned long long* acc, long long N, int Qb, int k, const long long* row_ids,
                     float* out_scores, long long* out_ids, cudaStream_t stream);

}  // namespace dprb
