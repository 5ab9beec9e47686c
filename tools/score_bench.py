#!/usr/bin/env python3
"""Time the fused scoring + cross-entropy kernels at the 1-GPU (128 x 1024) and 8-GPU (1024 x 8192 global, 128 local
queries / 1024 local contexts) shapes of BASELINE.json configs[1] / configs[2], d = 768."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpr_scale_b200 import ops


def timeit(f, iters=20):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


_a = [int(x) for x in sys.argv[1:]]
SHAPES = [tuple(_a[i:i + 4]) for i in range(0, len(_a), 4)] or [(128, 1024, 128, 1024), (1024, 8192, 128, 1024)]
for Q, C, nq, nc in SHAPES:
    d = 768
    q, c = torch.randn(Q, d, device="cuda"), torch.randn(C, d, device="cuda")
    mask = torch.zeros(C, dtype=torch.uint8, device="cuda")
    labels = torch.randint(0, C, (Q,), device="cuda")
    _, _, _, ctx = ops.score_fwd(q, c, mask, labels, 1.0, False, None, (nq, nc))
    f = timeit(lambda: ops.score_fwd(q, c, mask, labels, 1.0, False, None, (nq, nc)))
    b = timeit(lambda: ops.score_bwd(ctx, 1.0, 1.0, 0, nq, 0, nc))
    print(f"Q={Q} C={C} tensor-core single pass (bf16x3: 2-part split, 3 products): fwd {f:8.1f} us ({2.0*Q*C*d/f/1e6:6.2f} TFLOP/s of fp32-equivalent "
          f"work, {6.0*Q*C*d/f/1e6:6.1f} executed)   bwd(recompute W + 6 GEMMs) {b:8.1f} us", flush=True)
