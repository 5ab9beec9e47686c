"""Process-group set-up shared by the entry points (main, generate_embeddings, run_retrieval, bench.py).

One process per GPU, NCCL over NVLink / NVSwitch.  The NCCL stream is created with HIGH priority: the gradient
all-reduce is issued bucket by bucket during backward, whose GEMMs fill every SM; a normal-priority
NCCL kernel only gets its ~24 CTAs at the next kernel boundary and in competition with the next GEMM's CTAs, so the
buckets queue up and part of the all-reduce is still outstanding when backward ends.  With priority its CTAs are placed as soon as any CTA retires.
"""
import os

import torch
import torch.distributed as dist


def init_process_group(device=None, backend=None):
    """Join the default group from torchrun's environment (no-op for WORLD_SIZE <= 1 or when already initialised)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 or dist.is_initialized():
        return world
    backend = backend or os.environ.get("DPRB_DIST_BACKEND", "nccl" if torch.cuda.is_available() else "gloo")
    if backend == "nccl":
        if device is None:
            device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
        torch.cuda.set_device(device)
        kw = {"device_id": device}
        if not os.environ.get("DPRB_NCCL_NORMAL_PRIORITY"):
            try:
                opts = dist.ProcessGroupNCCL.Options()
                opts.is_high_priority_stream = True
                kw["pg_options"] = opts
            except Exception:  # noqa: older torch without the option
                pass
        dist.init_process_group("nccl", **kw)
    else:
        dist.init_process_group(backend)
    return world
