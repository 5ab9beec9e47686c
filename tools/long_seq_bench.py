#!/usr/bin/env python3
"""Long-sequence measurements (256 < S <= 512), one JSON line per result on stdout.

  python tools/long_seq_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--out DIR]

1. A full training step of BERT-base at S = 512 with 32 queries + 64 contexts (1 positive + 1 hard negative each) per
   GPU and dropout 0.1, on the dprb path and on stock HF + PyTorch (bench.time_stock: bf16 autocast, SDPA attention),
   alternated `rounds` times.  The dprb step is split into its GEMM time (CUDA events around every GEMM launch, as in
   bench.py's roofline leg) and an attention estimate (the attention forward + backward kernels timed alone at the
   step's shapes, times the layers that run them).
2. Attention forward / backward at S in {384, 512}, 12 heads, T = 131 072 tokens, all keys valid: the dprb kernels next
   to torch.nn.functional.scaled_dot_product_attention (bf16, same shapes) in the same process.
The card name, power limit and SM clock are recorded with the results.
"""
import argparse
import contextlib
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

B, NNEG, S, DROPOUT = 32, 1, 512, 0.1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def events_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


class DprbStep:
    def __init__(self, dev):
        from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
        from dpr_scale_b200.trainer import Trainer
        self.task = DenseRetrieverTask(
            transform={}, datamodule=None, shared_model=False, in_batch_negatives=True, warmup_steps=10,
            model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": bench.BERT_BASE,
                   "dropout": DROPOUT},
            optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 1e-5, "betas": [0.9, 0.999], "eps": 1e-8,
                   "weight_decay": 0.0})
        self.trainer = Trainer(max_steps=10 ** 6, gradient_clip_val=2.0, device=dev)
        with contextlib.redirect_stdout(sys.stderr):
            self.trainer.attach(self.task, None, "fit")
        self.task.train()
        self.batch = bench.to_device(bench.synth_batch(0, bench.BERT_BASE, B, NNEG, S), dev)
        self.i = 0

    def step(self):
        self.trainer.training_step(self.batch, self.i).detach()
        self.i += 1

    def gemm_ms(self, steps):
        """GEMM time per step (CUDA events around every GEMM launch, query encoder on the main stream)."""
        from dpr_scale_b200 import _lib
        lib = _lib.load()
        os.environ["DPRB_NO_STREAM_OVERLAP"] = "1"
        self.step()
        torch.cuda.synchronize()
        _lib.check(lib.dprb_gemm_profile_enable(1, 1500 * steps + 64), "profile_enable")
        step_ms = events_ms(self.step, steps, warmup=0)
        tms, tfl, nl = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        _lib.check(lib.dprb_gemm_profile_read(ctypes.byref(tms), ctypes.byref(tfl), ctypes.byref(nl)), "profile_read")
        _lib.check(lib.dprb_gemm_profile_enable(0, 0), "profile_disable")
        del os.environ["DPRB_NO_STREAM_OVERLAP"]
        return {"step_ms_serial": step_ms, "gemm_ms": tms.value / steps, "gemm_tflops": tfl.value / (tms.value / 1e3) / 1e12}


def attention_share_ms(dev):
    """Attention kernels of one step, timed alone: the 11 unpruned layers x (query + context sequences), forward with the
    lse and backward, dropout on, padding mask all ones (bench.synth_batch's variant A)."""
    from dpr_scale_b200 import ops
    heads, L = 12, bench.BERT_BASE["num_hidden_layers"]
    nseq = B + B * (1 + NNEG)
    qkv = torch.randn(nseq * S, 3 * heads * 64, device=dev, dtype=torch.bfloat16)
    am = torch.ones(nseq, S, dtype=torch.int32, device=dev)
    site = ops.dropout_site_seed(1, 0, 1)
    ctx, lse = ops.attn_fwd(qkv, am, nseq, S, heads, True, DROPOUT, site)
    dctx = torch.randn_like(ctx)
    dbias = torch.zeros(3 * heads * 64, device=dev)
    fwd = events_ms(lambda: ops.attn_fwd(qkv, am, nseq, S, heads, True, DROPOUT, site), 10)
    bwd = events_ms(lambda: ops.attn_bwd(qkv, am, ctx, lse, dctx, nseq, S, heads, dbias, DROPOUT, site), 10)
    return {"attn_fwd_ms": fwd, "attn_bwd_ms": bwd, "layers": L - 1, "attn_ms_per_step": (L - 1) * (fwd + bwd)}


def attention_bench(dev, S_, heads=12, T=131072, iters=10):
    from dpr_scale_b200 import ops
    import torch.nn.functional as F
    nseq, H = T // S_, heads * 64
    qkv = torch.randn(nseq * S_, 3 * H, device=dev, dtype=torch.bfloat16)
    ctx, lse = ops.attn_fwd(qkv, None, nseq, S_, heads)
    dctx = torch.randn_like(ctx)
    fl = 4.0 * S_ * H * T                      # QK^T + PV, forward
    r = {"what": "attention", "S": S_, "heads": heads, "T": T}
    r["dprb_fwd_us"] = 1e3 * events_ms(lambda: ops.attn_fwd(qkv, None, nseq, S_, heads), iters)
    r["dprb_bwd_us"] = 1e3 * events_ms(lambda: ops.attn_bwd(qkv, None, ctx, lse, dctx, nseq, S_, heads), iters)
    x = qkv.view(nseq, S_, 3, heads, 64)
    q, k, v = (x[:, :, i].transpose(1, 2).contiguous().requires_grad_(True) for i in range(3))
    do = dctx.view(nseq, S_, heads, 64).transpose(1, 2).contiguous()
    r["sdpa_fwd_us"] = 1e3 * events_ms(lambda: F.scaled_dot_product_attention(q, k, v), iters)
    out = F.scaled_dot_product_attention(q, k, v)
    r["sdpa_bwd_us"] = 1e3 * events_ms(lambda: torch.autograd.grad(out, (q, k, v), do, retain_graph=True), iters)
    for side in ("dprb", "sdpa"):
        r[f"{side}_fwd_tflops"] = fl / (r[f"{side}_fwd_us"] * 1e-6) / 1e12
        r[f"{side}_bwd_tflops"] = 2.5 * fl / (r[f"{side}_bwd_us"] * 1e-6) / 1e12
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/long_seq_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("long_seq_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lines = [dict(what="gpu", **gpu_info())]

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    print(json.dumps(lines[0]), flush=True)
    dprb, stock = [], []
    for rnd in range(args.rounds):
        run = DprbStep(dev)
        for _ in range(args.warmup):
            run.step()
        ms = events_ms(run.step, args.steps, warmup=0)
        dprb.append(ms)
        extra = {}
        if rnd == args.rounds - 1:
            extra = run.gemm_ms(min(args.steps, 5))
            extra["peak_mem_gb"] = torch.cuda.max_memory_allocated(dev) / 2 ** 30
        del run
        torch.cuda.empty_cache()
        emit(dict(what="train_step", impl="dprb", round=rnd, ms_per_step=ms, pairs_per_s=B / (ms / 1e3), **extra))
        s = bench.time_stock(bench.BERT_BASE, B, NNEG, S, DROPOUT, "bf16", args.steps, args.warmup, dev,
                             sample_clocks=False)
        stock.append(s["ms_per_step"])
        emit(dict(what="train_step", impl="stock", round=rnd, ms_per_step=s["ms_per_step"], pairs_per_s=s["value"],
                  peak_mem_gb=s["peak_mem_gb"], attn=s["attn"], dtype=s["dtype"]))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    emit(dict(what="train_step_summary", workload=f"bert-base S={S} {B} q + {B * (1 + NNEG)} ctx, dropout {DROPOUT}",
              dprb_ms=med(dprb), stock_ms=med(stock), dprb_ms_all=dprb, stock_ms_all=stock,
              ratio_pairs_per_s=med(stock) / med(dprb)))
    emit(dict(what="attention_share", **attention_share_ms(dev)))
    for S_ in (384, 512):
        emit(attention_bench(dev, S_))
    lines.append(dict(what="gpu_after", **gpu_info()))
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "long_seq_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
