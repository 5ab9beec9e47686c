#!/usr/bin/env python3
"""Golden vectors for MADGRAD, produced by the UNMODIFIED reference optimizer (dpr_scale/optim/madgrad.py).

  python tests/golden/make_golden_optim.py     # writes tests/golden/optim_madgrad.npz

The module is loaded from its file (it only imports torch).  Its ``initialize_state`` moves the state to the GPU with
``.cuda()``; this script runs on the CPU, so ``torch.Tensor.cuda`` is made a no-op while the optimizer is built.  No
reference source is edited.  For every case of CASES below, three seeded fp32 tensors of uneven shapes take STEPS
steps with seeded gradients; the group lr follows LRS, whose first entry 0 is a warmup step (the reference's
constructor refuses lr <= 0, so the rate is set on the param group, as LambdaLR does).  Recorded: the initial tensors,
each step's gradients (before the reference adds weight decay into them in place), the tensors after every step, and
the final grad_sum_sq and s.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(5, 7), (33,), (4, 4, 3)]
LRS = [0.0, 1e-2, 5e-3, 1e-2]
# name -> (momentum, weight_decay, eps)
CASES = {"m09_wd": (0.9, 0.01, 1e-6), "m0_wd": (0.0, 0.01, 1e-6), "m09": (0.9, 0.0, 1e-6), "m0_eps": (0.0, 0.0, 1e-3)}


def load_madgrad():
    path = os.path.join(REF, "dpr_scale", "optim", "madgrad.py")
    spec = importlib.util.spec_from_file_location("reference_madgrad", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.MADGRAD


def main():
    MADGRAD = load_madgrad()
    out = {"lrs": np.asarray(LRS, dtype=np.float64), "num_params": np.int64(len(SHAPES))}
    for ci, (name, (momentum, wd, eps)) in enumerate(CASES.items()):
        g = torch.Generator().manual_seed(100 + ci)
        params = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in SHAPES]
        for i, p in enumerate(params):
            out[f"{name}/p0/{i}"] = p.detach().numpy().copy()
        cuda = torch.Tensor.cuda
        torch.Tensor.cuda = lambda self, *a, **k: self
        try:
            opt = MADGRAD(params, lr=1e-2, momentum=momentum, weight_decay=wd, eps=eps)
        finally:
            torch.Tensor.cuda = cuda
        for step, lr in enumerate(LRS):
            opt.param_groups[0]["lr"] = lr
            for i, p in enumerate(params):
                grad = torch.randn(p.shape, generator=g) * 0.5
                out[f"{name}/g/{step}/{i}"] = grad.numpy().copy()
                p.grad = grad.clone()
            opt.step()
            for i, p in enumerate(params):
                out[f"{name}/p/{step}/{i}"] = p.detach().numpy().copy()
        for i, p in enumerate(params):
            out[f"{name}/grad_sum_sq/{i}"] = opt.state[p]["grad_sum_sq"].numpy().copy()
            out[f"{name}/s/{i}"] = opt.state[p]["s"].numpy().copy()
        out[f"{name}/hyper"] = np.asarray([momentum, wd, eps], dtype=np.float64)
    path = os.path.join(HERE, "optim_madgrad.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    sys.exit(main())
