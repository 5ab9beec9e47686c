#!/usr/bin/env python3
"""Optimizer-step benchmark: the fused AdamW / LAMB / MADGRAD steps over two BERT-base arenas (the query and context
encoders of the default bi-encoder, ~109 M parameters each) against the same updates written as per-tensor torch loops,
and against torch.optim.AdamW(foreach=True).  Every variant includes the global-norm clip (2.0) and the bf16 shadow
refresh the encoders need after a step, so they do the same job.

Bytes per parameter (fp32 state, bf16 shadow, counted from what each fused step must move):
  clip sum of squares: read g (4);
  AdamW:   read p, g, m, v, write p, m, v, shadow                   -> 30 (+4 clip)
  LAMB:    pass 1 read p, g, m, v, write m, v; pass 2 read p, m, v, write p, shadow -> 42 (+4 clip)
  MADGRAD: read p, g, nu, s, x0, write p, nu, s, shadow             -> 34 (+4 clip)
GB/s is those bytes over the measured step time; frac_hbm compares it with the H100 SXM data-sheet 3.35 TB/s.
Times are CUDA-event times over many steps after warmup, on the card named in the output line with its power limit.
  python tools/optim_bench.py [--steps 50] [--warmup 5] [--torch-steps 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dpr_scale_b200 import ops  # noqa: E402
from dpr_scale_b200.models.hf_model import ParamLayout, _normalise_config  # noqa: E402

BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512)
HBM = 3.35e12
MAX_NORM, LR, WD = 2.0, 1e-4, 0.01
STEP_BYTES = {"adamw": 30 + 4, "lamb": 42 + 4, "madgrad": 34 + 4}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


class Arena:
    def __init__(self, layout, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        n = layout.total
        self.sizes = [math.prod(s) for _, s, _ in layout.entries]
        self.p = torch.randn(n, device="cuda", generator=g) * 0.02
        self.g = torch.randn(n, device="cuda", generator=g) * 1e-3
        self.a, self.b = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        self.x0 = self.p.clone()
        self.shadow = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        self.plan = ops.LambPlan(self.sizes, "cuda")

    def views(self, t):
        out, lo = [], 0
        for n in self.sizes:
            out.append(t[lo:lo + n])
            lo += n
        return out


def fused(kind, arenas, sumsq, step):
    sumsq.zero_()
    for A in arenas:
        ops.sumsq(A.g, sumsq)
    for A in arenas:
        if kind == "adamw":
            ops.adamw_step(A.p, A.g, A.a, A.b, A.shadow, LR, 0.9, 0.999, 1e-8, WD, step, 1.0, sumsq, MAX_NORM)
        elif kind == "lamb":
            ops.lamb_step(A.p, A.g, A.a, A.b, A.shadow, A.plan, LR, 0.9, 0.999, 1e-6, WD, 10.0, False, False, step,
                          1.0, sumsq, MAX_NORM)
        else:
            ops.madgrad_step(A.p, A.g, A.a, A.b, A.x0, A.shadow, LR, 0.9, WD, 1e-6, step - 1, 1.0, sumsq, MAX_NORM)


def per_tensor(kind, tensors, step):
    """The same update as per-tensor torch ops: [(p, g, a, b, x0)] views, then the shadow refresh per arena."""
    grads = [t[1] for t in tensors]
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g) for g in grads]))
    coef = torch.clamp(MAX_NORM / (total + 1e-6), max=1.0)
    lamb = (LR + 1e-6) * math.sqrt(step)
    for p, g, a, b, x0 in tensors:
        g = g * coef
        if kind == "adamw":
            p.mul_(1.0 - LR * WD)
            a.mul_(0.9).add_(g, alpha=0.1)
            b.mul_(0.999).addcmul_(g, g, value=0.001)
            p.addcdiv_(a, b.sqrt() / math.sqrt(1 - 0.999 ** step) + 1e-8, value=-LR / (1 - 0.9 ** step))
        elif kind == "lamb":
            a.mul_(0.9).add_(g, alpha=0.1)
            b.mul_(0.999).addcmul_(g, g, value=0.001)
            u = a / (b.sqrt() + 1e-6) + WD * p
            w, un = p.norm().clamp(0, 10.0), u.norm()
            trust = torch.where((w == 0) | (un == 0), torch.ones_like(w), w / un)
            p.sub_(u * (trust * LR))
        else:
            g = g + WD * p
            b.addcmul_(g, g, value=lamb)
            a.add_(g, alpha=lamb)
            z = x0 - a / (b.pow(1 / 3) + 1e-6)
            p.mul_(0.9).add_(z, alpha=0.1)


def time_it(fn, steps, warmup):
    for i in range(warmup):
        fn(i + 1)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
        fn(warmup + i + 1)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--torch-steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench needs a CUDA device (an H100)")
    layout = ParamLayout(_normalise_config(BERT_BASE))
    arenas = [Arena(layout, 1), Arena(layout, 2)]
    nparams = sum(A.p.numel() for A in arenas)
    sumsq = torch.zeros(1, device="cuda")
    tensors = [t for A in arenas for t in zip(*(A.views(x) for x in (A.p, A.g, A.a, A.b, A.x0)))]
    res = {}
    for kind in ("adamw", "lamb", "madgrad"):
        ms = time_it(lambda s: fused(kind, arenas, sumsq, s), args.steps, args.warmup)
        nbytes = STEP_BYTES[kind] * nparams
        res[f"fused_{kind}"] = {"ms_per_step": round(ms, 4), "bytes_per_step": nbytes,
                                "gbps": round(nbytes / (ms * 1e-3) / 1e9, 1),
                                "frac_hbm": round(nbytes / (ms * 1e-3) / HBM, 3),
                                "hbm_bound_ms": round(nbytes / HBM * 1e3, 3)}

        def loop(s):
            per_tensor(kind, tensors, s)
            for A in arenas:
                ops.cast_f32_bf16(A.p, A.shadow)
        res[f"torch_per_tensor_{kind}"] = {"ms_per_step": round(time_it(loop, args.torch_steps, 2), 3)}
    params = [torch.nn.Parameter(v) for A in arenas for v in A.views(A.p)]
    for prm, g in zip(params, [v for A in arenas for v in A.views(A.g)]):
        prm.grad = g
    opt = torch.optim.AdamW(params, lr=LR, weight_decay=WD, foreach=True)

    def foreach(s):
        torch.nn.utils.clip_grad_norm_(params, MAX_NORM, foreach=True)
        opt.step()
        for A in arenas:
            ops.cast_f32_bf16(A.p, A.shadow)
    res["torch_adamw_foreach"] = {"ms_per_step": round(time_it(foreach, args.torch_steps, 2), 3)}
    for kind in ("adamw", "lamb", "madgrad"):
        res[f"fused_{kind}"]["speedup_vs_per_tensor"] = round(
            res[f"torch_per_tensor_{kind}"]["ms_per_step"] / res[f"fused_{kind}"]["ms_per_step"], 1)
    res["fused_adamw"]["speedup_vs_adamw_foreach"] = round(
        res["torch_adamw_foreach"]["ms_per_step"] / res["fused_adamw"]["ms_per_step"], 1)
    print(json.dumps({"metric": "optimizer_step", "card": card(), "params": nparams, "tensors": len(tensors),
                      "steps": args.steps, "warmup": args.warmup, "results": res}))


if __name__ == "__main__":
    main()
