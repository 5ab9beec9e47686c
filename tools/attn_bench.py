#!/usr/bin/env python3
"""Time attention fwd/bwd as the encoder calls them: python tools/attn_bench.py S heads [T ...] [--iters N]

Dropout 0.1 with a site seed and the QKV bias gradient (dbias) requested, as in a training step.  One line per
(pass, T): us per call and TFLOP/s.  FLOP counts per (sequence, head) problem: forward 2 products (Q K^T, P V),
backward 5 products (Q K^T, dO V^T, dQ = dS K, dK = dS^T Q, dV = P^T dO), each 2 * S^2 * 64.
"""
import argparse
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from dpr_scale_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("S", type=int)
ap.add_argument("heads", type=int)
ap.add_argument("T", type=int, nargs="*", default=[131072])
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--dropout", type=float, default=0.1)
args = ap.parse_args()
S, heads = args.S, args.heads
H = heads * 64
dev = "cuda"
bf = torch.bfloat16
SEED = 0x2F6A3C51


def timeit(name, T, f, flops):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    print(f"{name:9s} S={S} heads={heads} T={T} p={args.dropout}: {ms * 1e3:9.1f} us  {flops / ms / 1e9:7.1f} TFLOP/s",
          flush=True)


for T in args.T:
    g = torch.Generator(device=dev).manual_seed(T)
    nseq = T // S
    qkv = torch.randn(T, 3 * H, device=dev, dtype=bf, generator=g)
    dctx = torch.randn(T, H, device=dev, dtype=bf, generator=g)
    dqkv = torch.empty_like(qkv)
    dbias = torch.zeros(3 * H, device=dev, dtype=torch.float32)
    kw = dict(dropout_p=args.dropout, site_seed=SEED)
    ctx, lse = ops.attn_fwd(qkv, None, nseq, S, heads, **kw)
    prod = 2.0 * S * S * 64 * nseq * heads
    timeit("attn_fwd", T, lambda: ops.attn_fwd(qkv, None, nseq, S, heads, ctx=ctx, lse=lse, **kw), 2 * prod)
    timeit("attn_bwd", T, lambda: ops.attn_bwd(qkv, None, ctx, lse, dctx, nseq, S, heads, dbias=dbias, dqkv=dqkv, **kw),
           5 * prod)
    del qkv, dctx, dqkv, ctx, lse
