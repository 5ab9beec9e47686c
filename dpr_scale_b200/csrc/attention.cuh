// Helpers shared by the wgmma attention kernels (attention_wgmma.cu: S <= 256, attention_long.cu: 256 < S <= 512).
#pragma once
#include "common.cuh"

namespace dprb {

constexpr float ATTN_SCALE_LOG2 = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) in the exp2 domain
constexpr float ATTN_LOG2E = 1.4426950408889634f;
constexpr float ATTN_LN2 = 0.6931471805599453f;

// K-major operand: [rows][64] bf16, one swizzle atom wide, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t desc_k(const void* p) { return make_wgmma_desc_sw128(smem_u32(p), 16, 1024); }
// MN-major operand read from [K rows][64 MN] (a single 64-wide MN atom)
__device__ __forceinline__ uint64_t desc_mn(const void* p) { return make_wgmma_desc_sw128(smem_u32(p), 16, 1024); }
// descriptor steps of one k16 slice (16-byte units): K-major +32 B, MN-major +16 rows of 128 B
constexpr uint64_t KSTEP_K = 2, KSTEP_MN = 128;

// bf16 [nseq, S, cols] (row stride `cols` elements), box = [1, box_rows, 64 cols], 128B swizzle; rows >= S of a
// sequence are zero-filled on load
int make_tmap3(CUtensorMap* out, const void* base, int nseq, int S, long long cols, int box_rows);

int attn_fwd_long(const void* qkv, const int32_t* attn_mask, void* ctx, float* lse, int nseq, int S, int heads,
                  float dropout_p, unsigned long long site_seed, cudaStream_t stream);
int attn_bwd_long(const void* qkv, const int32_t* attn_mask, const void* ctx, const float* lse, const void* dctx,
                  void* dqkv, int nseq, int S, int heads, float dropout_p, unsigned long long site_seed,
                  cudaStream_t stream);

}  // namespace dprb
