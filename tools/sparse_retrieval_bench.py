#!/usr/bin/env python3
"""SPLADE first-stage retrieval at MS MARCO size: dprb_sparse_search (SparseIndex.search) against two other ways to
run the same search on the H100.

Index: a synthetic passage CSR built on the device, ``--passages`` rows (8.8 M, the MS MARCO passage corpus) with
uniform(1, 2 * per_passage - 1) distinct Zipf(1.25)-distributed terms each (about 120 nonzeros, V = 30522; each term
at most once per row, as SPLADE emits them), fp16 weights; queries: ``--queries`` (6980, the MS MARCO dev set) with
about 25 distinct Zipf terms each.  Timed routes, CUDA events around
whole searches after a warm-up:

  * sparse   - SparseIndex.search: the inverted index, dprb_sparse_search, over all queries;
  * expert   - the same postings squeezed into dprb_expert_search: each term an expert, each weight an 8-wide padded
               fp16 payload (8x the posting bytes, one wgmma tile per 128 postings), on the first --baseline_queries
               queries;
  * torch    - torch.sparse CSR [N, V] fp32 @ a dense [V, Qb] query block + topk, on the first --baseline_queries
               queries, in blocks of --torch_block.

Reported per route: ms per query, and postings touched per second (the sum over query entries of their terms'
posting-list lengths).  The card's name and power limit are read in the same run.  Prints one JSON line.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "not read"]


def distinct_zipf_rows(counts, V, s, gen, device, chunk=16384):
    """Terms of CSR rows with counts[i] distinct Zipf(s)-distributed terms each, ascending inside a row, as a SPLADE
    encoder emits them: a weighted sample without replacement per row (the c largest of log(u) / p over the
    vocabulary, an exponential race), int32 [sum(counts)]."""
    p = (1.0 / torch.arange(1, V + 1, dtype=torch.float64, device=device) ** s).float()
    kmax = int(counts.max())
    out = []
    for a in range(0, counts.numel(), chunk):
        c = counts[a:a + chunk]
        keys = torch.rand(c.numel(), V, generator=gen, device=device).log_().div_(p)
        top = keys.topk(kmax, dim=1).indices
        del keys
        keep = torch.arange(kmax, device=device)[None, :] < c[:, None]
        top = torch.where(keep, top, V).sort(dim=1).values           # dropped slots sort to the end
        out.append(top[keep].to(torch.int32))
    return torch.cat(out)


def timed(fn, reps=1):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=8_841_823)
    ap.add_argument("--per_passage", type=int, default=120)
    ap.add_argument("--queries", type=int, default=6980)
    ap.add_argument("--per_query", type=int, default=25)
    ap.add_argument("--V", type=int, default=30522)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--baseline_queries", type=int, default=240)
    ap.add_argument("--torch_block", type=int, default=64)
    ap.add_argument("--skip_expert", action="store_true")
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs the H100"
    from dpr_scale_b200 import ops
    from dpr_scale_b200.splade_retrieval import SparseIndex
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    N, V, k = args.passages, args.V, args.k
    counts = torch.randint(1, 2 * args.per_passage, (N,), generator=g, device=dev)
    offsets = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=offsets[1:])
    nnz = int(offsets[-1])
    terms = distinct_zipf_rows(counts, V, 1.25, g, dev)
    assert terms.numel() == nnz
    weights = (torch.rand(nnz, generator=g, device=dev) * 3).half()
    t0 = time.perf_counter()
    index = SparseIndex(offsets, terms, weights, V, device=dev)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    rng = np.random.default_rng(1)
    qn = rng.integers(1, 2 * args.per_query, args.queries)
    q_off = np.r_[0, np.cumsum(qn)]
    q_t = distinct_zipf_rows(torch.from_numpy(qn).to(dev), V, 1.25, g, dev).cpu().numpy().astype(np.int64)
    q_w = (rng.random(q_t.size) * 2).astype(np.float32)
    lengths = np.diff(index.term_ptr_host)

    def touched(nq):
        return int(lengths[q_t[:q_off[nq]]].sum())

    res = {"bench": "sparse_retrieval", "card": card()[0], "power_limit": card()[1], "passages": N, "nnz": nnz,
           "V": V, "queries": args.queries, "query_nnz": int(q_off[-1]), "k": k,
           "index_bytes": int(index.row.numel() * 6 + index.term_ptr.numel() * 8 + index.ids.numel() * 8),
           "index_build_s": round(build_s, 2), "queries_per_block": ops.sparse_search_block_queries(N)}
    ms, (s_all, i_all) = timed(lambda: index.search(q_off, q_t, q_w, k))
    res["sparse_ms"] = round(ms, 1)
    res["sparse_ms_per_query"] = round(ms / args.queries, 4)
    res["sparse_postings_per_s"] = float(f"{touched(args.queries) / (ms * 1e-3):.4g}")
    res["postings_per_query"] = float(f"{touched(args.queries) / args.queries:.4g}")
    nb = min(args.baseline_queries, args.queries)
    sub = (q_off[:nb + 1], q_t[:q_off[nb]], q_w[:q_off[nb]])
    ms, _ = timed(lambda: index.search(*sub, k))
    res["baseline_queries"] = nb
    res["sparse_sub_ms_per_query"] = round(ms / nb, 4)

    # torch.sparse: passage CSR [N, V] @ dense query block [V, b], topk over the passages
    P = torch.sparse_csr_tensor(offsets, terms.long(), weights.float(), size=(N, V))
    del terms

    def torch_route():
        out_s, out_i = [], []
        for a in range(0, nb, args.torch_block):
            b = min(nb, a + args.torch_block)
            qd = torch.zeros(V, b - a, device=dev)
            rows = np.repeat(np.arange(b - a), qn[a:b])
            qd.index_put_((torch.from_numpy(q_t[q_off[a]:q_off[b]]).to(dev), torch.from_numpy(rows).to(dev)),
                          torch.from_numpy(q_w[q_off[a]:q_off[b]]).to(dev), accumulate=True)
            s, i = torch.topk(torch.sparse.mm(P, qd), k, dim=0)
            out_s.append(s.T)
            out_i.append(i.T)
        return torch.cat(out_s), torch.cat(out_i)
    try:
        ms, (ts, ti) = timed(torch_route)
        res["torch_ms_per_query"] = round(ms / nb, 4)
        res["torch_postings_per_s"] = float(f"{touched(nb) / (ms * 1e-3):.4g}")
        res["torch_vs_sparse_max_score_diff"] = float((ts - s_all[:nb]).abs().max())
        del ts, ti
    except RuntimeError as e:                       # e.g. out of memory: recorded, the other routes still run
        res["torch_error"] = str(e).splitlines()[0][:200]
    del P
    torch.cuda.empty_cache()

    if not args.skip_expert:
        # every posting a one-entry run of its term's expert; payload = [w, 0, ..., 0]
        E = index.nnz
        pay = torch.zeros(E, 8, dtype=torch.float16, device=dev)
        pay[:, 0] = index.weight[:E]
        tp = index.term_ptr
        ntiles = (tp[1:] - tp[:-1] + ops.EXPERT_SEARCH_TILE_WINDOW - 1) // ops.EXPERT_SEARCH_TILE_WINDOW
        tile_ptr = torch.zeros(V + 1, dtype=torch.int64, device=dev)
        torch.cumsum(ntiles, 0, out=tile_ptr[1:])
        T = int(tile_ptr[-1])
        tt = torch.repeat_interleave(torch.arange(V, device=dev), ntiles)
        starts = tp[:-1][tt] + (torch.arange(T, device=dev) - tile_ptr[:-1][tt]) * ops.EXPERT_SEARCH_TILE_WINDOW
        tile_bounds = torch.cat([starts, tp[-1:]]).to(torch.int32)
        tile_ptr_h = tile_ptr.cpu().numpy()
        row = index.row[:max(E, 1)]
        Qb = ops.expert_search_block_queries(N)

        def expert_route():
            out = []
            for a in range(0, nb, Qb):
                b = min(nb, a + Qb)
                qt, qw = q_t[q_off[a]:q_off[b]], q_w[q_off[a]:q_off[b]]
                seq = np.repeat(np.arange(b - a), qn[a:b])
                order = np.lexsort((seq, qt))
                groups, item_end, items = ops.expert_search_groups(qt[order], tile_ptr_h, 0, N)
                qp = torch.zeros(order.size, 8, dtype=torch.float16, device=dev)
                qp[:, 0] = torch.from_numpy(qw[order]).to(dev).half()
                out.append(ops.expert_search(pay, row, tile_bounds, 8, None, index.ids, qp,
                                             torch.from_numpy(seq[order].astype(np.int32)).to(dev), None, b - a,
                                             torch.from_numpy(groups).to(dev), torch.from_numpy(item_end).to(dev),
                                             items, k))
            return out
        try:
            ms, _ = timed(expert_route)
            res["expert_ms_per_query"] = round(ms / nb, 4)
            res["expert_postings_per_s"] = float(f"{touched(nb) / (ms * 1e-3):.4g}")
        except RuntimeError as e:
            res["expert_error"] = str(e).splitlines()[0][:200]
        res["expert_payload_bytes"] = int(pay.numel() * 2 + row.numel() * 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
