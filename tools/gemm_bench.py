#!/usr/bin/env python3
"""Time the encoder's GEMM shapes/epilogues in isolation with CUDA events (inputs >> L2 each), each next to cuBLAS
(torch.matmul on the same bf16 operands into a bf16 output, no epilogue) as an in-call yardstick.
  python tools/gemm_bench.py [T]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dpr_scale_b200 import ops

T = int(sys.argv[1]) if len(sys.argv) > 1 else 131072
H, I = 768, 3072
dev = "cuda"
bf = torch.bfloat16


def run(name, M, N, K, a_mn, b_mn, epi, aux=False, out2=False, colsum=False, f32=False, drop=0.0, f16=False,
        aux_stride=1, iters=5):
    """f16: fp16 residual in and fp16 sum out (the encoder's residual stream); drop: hidden dropout before the residual;
    aux_stride: the aux rows are that many rows apart in a taller buffer (the pruned last layer reads CLS rows)."""
    A = torch.randn((K, M) if a_mn else (M, K), device=dev, dtype=bf)
    B = torch.randn((K, N) if b_mn else (N, K), device=dev, dtype=bf) * 0.02
    D = torch.zeros(M, N, device=dev, dtype=torch.float32 if f32 else (torch.float16 if f16 else bf))
    bias = torch.zeros(N, device=dev) if epi in (0, 1, 2) and not f32 else None
    ax = torch.randn(M * aux_stride, N, device=dev, dtype=torch.float16 if f16 else bf) if aux else None
    o2 = torch.empty(M, N, device=dev, dtype=bf) if out2 else None
    cs = torch.zeros(N, device=dev) if colsum else None
    lda = M if a_mn else K
    ldb = N if b_mn else K
    if f16:
        epi |= ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16
    f = lambda: ops.gemm(A, B, D, M, N, K, lda, ldb, N, a_mn, b_mn, epi, bias, ax, N * aux_stride if aux else 0, o2, 1.0,
                         0 if f32 else 1, cs, drop, 0x5EED if drop else 0)
    Am = A.T if a_mn else A          # [M, K] views of the same storage
    Bm = B if b_mn else B.T          # [K, N]
    C = torch.empty(M, N, device=dev, dtype=bf)
    ms = timed(f, iters)
    ms_cublas = timed(lambda: torch.matmul(Am, Bm, out=C), iters)
    tf = lambda t: 2.0 * M * N * K / t / 1e9
    print(f"{name:34s} M={M:7d} N={N:5d} K={K:7d}  {ms*1e3:9.1f} us  {tf(ms):8.1f} TF/s   cuBLAS {ms_cublas*1e3:9.1f} us "
          f"{tf(ms_cublas):8.1f} TF/s", flush=True)


def timed(f, iters):
    for _ in range(2):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


run("fwd qkv bias", T, 3 * H, H, 0, 0, 0)
run("fwd attn-out bias+res", T, H, H, 0, 0, 2, aux=True)
run("fwd ffn-in bias only", T, I, H, 0, 0, 0)
run("fwd ffn-in gelu (no pre)", T, I, H, 0, 0, 1)
run("fwd ffn-in gelu + pre", T, I, H, 0, 0, 1, out2=True)
run("fwd ffn-out bias+res", T, H, I, 0, 0, 2, aux=True)
# what the training step runs: fp16 residual stream, hidden dropout p = 0.1
run("fwd attn-out bias+res+drop", T, H, H, 0, 0, 2, aux=True, f16=True, drop=0.1)
run("fwd ffn-out bias+res+drop", T, H, I, 0, 0, 2, aux=True, f16=True, drop=0.1)
# pruned last layer: the CLS rows of T / 128 sequences, residual rows S * H apart
run("fwd pruned attn-out res, ld_aux=S*H", T // 128, H, H, 0, 0, 2, aux=True, f16=True, drop=0.1, aux_stride=128,
    iters=50)
run("dgrad w2 plain", T, I, H, 0, 1, 0)
run("dgrad w2 dgelu", T, I, H, 0, 1, 3, aux=True)
run("dgrad w2 dgelu+colsum", T, I, H, 0, 1, 3, aux=True, colsum=True)
run("dgrad w1 res", T, H, I, 0, 1, 2, aux=True)
run("dgrad wo", T, H, H, 0, 1, 0)
run("dgrad wqkv res", T, H, 3 * H, 0, 1, 2, aux=True)
run("wgrad w2", H, I, T, 1, 1, 4, f32=True)
run("wgrad w1", I, H, T, 1, 1, 4, f32=True)
run("wgrad wo", H, H, T, 1, 1, 4, f32=True)
run("wgrad wqkv", 3 * H, H, T, 1, 1, 4, f32=True)
run("q-enc fwd qkv", 16384, 3 * H, H, 0, 0, 0)
run("q-enc fwd ffn-in gelu+pre", 16384, I, H, 0, 0, 1, out2=True)
run("q-enc wgrad w1", I, H, 16384, 1, 1, 4, f32=True)
