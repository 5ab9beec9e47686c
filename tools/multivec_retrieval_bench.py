#!/usr/bin/env python3
"""Retrieval from a COIL / CITADEL expert index: ExpertIndex.search (dprb_expert_search) against a torch restatement
of the same search, on a synthetic CITADEL-shaped index built from a seed.

Index: N passages x E/N entries, experts Zipf-distributed over V = 30 522, P = 32, CLS width Pc = 128.  Queries: about
16 entries each, experts drawn from the same distribution.  The torch restatement, per query expert x: the [n_x, m_x]
matmul of the queries' payloads with the expert's postings, scatter_reduce(amax) onto [n_x, N] passages (from 0: the
clamp), index_add onto the queries' [Q, N] scores; then the CLS matmul and topk.  Both run in this process on the same
fp16 operands; the line records how many of our ids equal torch's and the largest score difference.

``index_build_s`` is the ExpertIndex constructor on fp16 tensors already on the device (tiling, checks, fp16
conversion): it does not include reading pickles or mapping corpus ids (ExpertIndex.load).
Times are CUDA-event / synchronised host-clock times on the card named in each line, with its power limit.
  python tools/multivec_retrieval_bench.py --out /tmp/multivec_retrieval.jsonl
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dpr_scale_b200 import ops  # noqa: E402
from dpr_scale_b200.task.citadel_retrieval_task import ExpertIndex  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def zipf_experts(rng, n, V):
    return (rng.zipf(1.2, n) - 1) % V


def build(args):
    rng = np.random.default_rng(args.seed)
    N, per = args.passages, args.entries
    row = np.repeat(np.arange(N, dtype=np.int64), per)
    ex = zipf_experts(rng, N * per, args.V)
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    pay = (torch.randn(N * per, args.P, generator=g, device="cuda") * 0.1).half()
    cls = (torch.randn(N, args.Pc, generator=g, device="cuda") * 0.1).half()
    order = np.lexsort((row, ex))                    # the generation writes each expert's entries in passage order
    ex, row = ex[order], row[order]
    pay = pay[torch.from_numpy(order).cuda()]
    ids = np.arange(N, dtype=np.int64)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx = ExpertIndex(ex, row, pay, ids, cls, args.V, "cuda")
    torch.cuda.synchronize()
    return idx, ex, time.perf_counter() - t0


def queries(args, Q):
    rng = np.random.default_rng(args.seed + 1)
    q_seq = np.repeat(np.arange(Q), args.q_entries)
    q_ex = zipf_experts(rng, q_seq.size, args.V)
    order = np.lexsort((q_seq, q_ex))
    g = torch.Generator(device="cuda").manual_seed(args.seed + 1)
    q_pay = (torch.randn(q_seq.size, args.P, generator=g, device="cuda") * 0.1).half()
    q_cls = (torch.randn(Q, args.Pc, generator=g, device="cuda") * 0.1).half()
    return q_ex[order], q_seq[order], q_pay, q_cls


def torch_search(idx, off, q_ex, q_seq, q_pay, q_cls, Q, k):
    """The CITADEL search restated in torch (per expert: matmul, scatter_reduce(amax) from 0, index_add; CLS; topk)."""
    N = idx.N
    S = torch.zeros(Q, N, dtype=torch.float32, device="cuda")
    seq_d = torch.from_numpy(q_seq).cuda()
    starts = np.flatnonzero(np.r_[True, q_ex[1:] != q_ex[:-1]])
    for lo, hi in zip(starts.tolist(), np.r_[starts[1:], q_ex.size].tolist()):
        x = int(q_ex[lo])
        a, b = int(off[x]), int(off[x + 1])
        if a == b:
            continue
        m = torch.zeros(hi - lo, N, dtype=torch.float32, device="cuda")
        step = max(1, (1 << 27) // (hi - lo))          # postings per matmul: [n_x, step] fp32 stays below 512 MB
        for c in range(a, b, step):
            d = min(b, c + step)
            s = q_pay[lo:hi].float() @ idx.payload[c:d, :idx.P].float().T                # [n_x, m]
            m.scatter_reduce_(1, idx.row[c:d].long().expand(hi - lo, -1), s, "amax", include_self=True)
        S.index_add_(0, seq_d[lo:hi], m)
    S += q_cls.float() @ idx.cls[:, :idx.Pc].float().T
    return torch.topk(S, k, dim=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--entries", type=int, default=64)
    ap.add_argument("--P", type=int, default=32)
    ap.add_argument("--Pc", type=int, default=128)
    ap.add_argument("--V", type=int, default=30522)
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--q-entries", type=int, default=16)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name = card()
    idx, ex_sorted, load_s = build(args)
    off = np.zeros(args.V + 1, np.int64)
    np.cumsum(np.bincount(ex_sorted, minlength=args.V), out=off[1:])
    Q = args.queries
    q_ex, q_seq, q_pay, q_cls = queries(args, Q)

    kernel_ms = []                                   # CUDA-event time of each dprb_expert_search call
    inner = ops.expert_search

    def timed(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = inner(*a, **kw)
        e1.record()
        kernel_ms.append((e0, e1))
        return out

    ops.expert_search = timed
    with torch.no_grad():
        ours = idx.search(q_ex, q_seq, q_pay, q_cls, Q, args.k)            # warm-up
        kernel_ms.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            ours = idx.search(q_ex, q_seq, q_pay, q_cls, Q, args.k)
        torch.cuda.synchronize()
        ours_s = (time.perf_counter() - t0) / args.steps
        k_ms = sum(a.elapsed_time(b) for a, b in kernel_ms) / args.steps
        ops.expert_search = inner
        ts, ti = torch_search(idx, off, q_ex, q_seq, q_pay, q_cls, Q, args.k)          # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(args.steps):
            ts, ti = torch_search(idx, off, q_ex, q_seq, q_pay, q_cls, Q, args.k)
        e1.record()
        torch.cuda.synchronize()
        torch_s = (time.perf_counter() - t0) / args.steps
        torch_ms = e0.elapsed_time(e1) / args.steps
    ts, ti = ts.cpu().numpy(), ti.cpu().numpy()
    same = float(np.mean([len(set(a) & set(b)) / args.k for a, b in zip(ours[1].tolist(), ti.tolist())]))
    line = {"bench": "multivec_retrieval", "passages": args.passages, "entries": int(idx.E), "P": args.P,
            "Pc": args.Pc, "V": args.V, "queries": Q, "query_entries": int(q_ex.size), "k": args.k,
            "tiles": int(idx.tile_bounds.numel() - 1), "block_queries": ops.expert_search_block_queries(idx.N),
            "ours_queries_per_s": Q / ours_s, "ours_kernel_ms": k_ms, "ours_search_ms": ours_s * 1e3,
            "torch_queries_per_s": Q / torch_s, "torch_ms": torch_ms, "speedup": torch_s / ours_s,
            "index_build_s": load_s, "topk_overlap_vs_torch": same,
            "max_score_diff_vs_torch": float(np.abs(np.sort(ours[0], 1)[:, ::-1] - ts).max()), "gpu": name}
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
