#!/usr/bin/env python3
"""Per-kernel time of the headline training step, the step bench.py's kernel leg times.

  python tools/step_profile.py --out DIR [--workload W] [--steps K] [--warmup W] [--no-overlap]

The step runs under torch.profiler with CUDA activities; every kernel (and memcpy / memset) the GPU ran is summed by
name over the profiled steps.  The step time is taken with CUDA events in a separate, unprofiled window of the same
length, so tracing overhead does not enter it.  --no-overlap keeps the query encoder on the main stream
(DPRB_NO_STREAM_OVERLAP=1, as bench.py's roofline leg does), so that kernel times do not overlap and add up to the
step.  Writes DIR/step_profile.jsonl: one header line, then one line per kernel, largest first.
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def main():
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (step_profile.jsonl is written there)")
    ap.add_argument("--workload", default="bert-base_s128_b128_n7", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=3, help="profiled steps (and steps of the timed window)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.1)
    ap.add_argument("--no-overlap", action="store_true", help="query encoder on the main stream (DPRB_NO_STREAM_OVERLAP=1)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_profile.py needs a GPU"
    if args.no_overlap:
        os.environ["DPRB_NO_STREAM_OVERLAP"] = "1"

    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.trainer import Trainer

    cfg, B, n, S = bench.WORKLOADS[args.workload]
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    task = DenseRetrieverTask(
        transform={}, datamodule=None, shared_model=False, in_batch_negatives=True, warmup_steps=10,
        model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": cfg,
               "dropout": args.dropout},
        optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 1e-5, "betas": [0.9, 0.999], "eps": 1e-8,
               "weight_decay": 0.0})
    trainer = Trainer(max_steps=10 ** 6, gradient_clip_val=2.0, device=dev)
    with contextlib.redirect_stdout(sys.stderr):
        trainer.attach(task, None, "fit")
    task.train()
    task.query_encoder._drop_base, task.context_encoder._drop_base = 0x5EED0001, 0x5EED0002
    task.context_encoder.activation_chunk = bench.ACT_CHUNK.get(args.workload, 0)
    lean = args.workload in bench.LEAN and task.context_encoder.activation_chunk == 0
    task.context_encoder.lean_activations = task.query_encoder.lean_activations = lean
    batch = bench.to_device(bench.synth_batch(0, cfg, B, n, S), dev)

    def steps():
        for i in range(args.steps):
            trainer.training_step(batch, i).detach()

    for i in range(args.warmup):
        trainer.training_step(batch, i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    steps()
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        steps()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = tot.setdefault(e.name, [0, 0.0])
        t[0] += 1
        t[1] += e.time_range.elapsed_us() / 1e3
    rows = sorted(tot.items(), key=lambda kv: -kv[1][1])
    kernel_ms = sum(v[1] for _, v in rows) / args.steps

    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "step_profile.jsonl")
    with open(path, "w") as f:
        head = {"workload": args.workload, "dropout": args.dropout, "steps": args.steps, "warmup": args.warmup,
                "stream_overlap": not args.no_overlap, "step_ms": step_ms, "kernel_ms_per_step": kernel_ms,
                "gpu": gpu_info(),
                "how": "step_ms: CUDA events over an unprofiled window; kernel times: torch.profiler CUDA activities"}
        f.write(json.dumps(head) + "\n")
        for name, (calls, ms) in rows:
            f.write(json.dumps({"kernel": name, "calls_per_step": calls / args.steps, "ms_per_step": ms / args.steps,
                                "share_of_step": ms / args.steps / step_ms}) + "\n")
    print(json.dumps(head))
    for name, (calls, ms) in rows[:25]:
        print(f"{ms / args.steps:9.3f} ms {100 * ms / args.steps / step_ms:5.1f} % {calls / args.steps:7.1f} x  {name[:110]}")
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
