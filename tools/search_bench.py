#!/usr/bin/env python3
"""Retrieval microbenchmark: dprb_search_topk (fused wgmma scoring + running top-k) vs the reference's GPU path
(run_retrieval_pytorch.py:141-176: fp16 einsum into a [Q, N] matrix + torch.topk), same box, same operands.

  python tools/search_bench.py [N d Q k] ...      default: MS MARCO-sized and Wikipedia-sized indexes
Prints one JSON line per configuration (HBM roofline = corpus bytes streamed / time vs MEASURED_PEAKS.json hbm_gbs).
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpr_scale_b200 import ops


def peak_gbs():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(p))["hbm_gbs"]), "MEASURED_PEAKS.json"
    except Exception:
        return 3350.0, "H100 SXM data sheet (HBM3)"


def timeit(f, iters):
    f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def ref_search(q, corpus, batch, k):
    outs, outi = [], []
    for s in range(0, q.shape[0], batch):
        scores = torch.einsum("ik,jk->ij", q[s:s + batch], corpus)
        v, i = torch.topk(scores, dim=-1, k=k)
        outs.append(v)
        outi.append(i)
        del scores
    return torch.cat(outs), torch.cat(outi)


def run(N, d, Q, k, iters=10):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    corpus = torch.empty(N, d, dtype=torch.float16, device=dev)
    for s in range(0, N, 1 << 20):
        e = min(N, s + (1 << 20))
        corpus[s:e] = torch.randn(e - s, d, generator=g, device=dev, dtype=torch.float32).to(torch.float16)
    q = torch.randn(Q, d, generator=g, device=dev, dtype=torch.float32).to(torch.float16)
    ms = timeit(lambda: ops.search_topk(q, corpus, k), iters)
    if os.environ.get("SEARCH_BENCH_SKIP_REF"):
        ms_ref, same_scores, same_ids = float("nan"), float("nan"), float("nan")
        ref_rank_scores = ref_rank_ids_all = ref_rank_ids_distinct = ms_rr = float("nan")
    else:
        ms_ref = timeit(lambda: ref_search(q, corpus, 100, k), max(1, iters - 1))  # --batch 100 is the reference default
        s, i = ops.search_topk(q, corpus, k)
        rs, ri = ref_search(q, corpus, 100, k)
        # the reference ranks fp16-rounded scores; ours rounded the same way must be the same multiset per row
        same_scores = float((s.to(torch.float16) == rs).float().mean())
        same_ids = float((i == ri).float().mean())
        # --reference_ranking: rank by the fp16-rounded score like the reference's topk does; ids are then compared
        # where they are a property of the algorithm, i.e. where the reference's fp16 score is unique in its row
        s2, i2 = ops.search_topk(q, corpus, k, reference_ranking=True)
        uniq = torch.ones_like(rs, dtype=torch.bool)
        uniq[:, 1:] &= rs[:, 1:] != rs[:, :-1]
        uniq[:, :-1] &= rs[:, :-1] != rs[:, 1:]
        uniq[:, -1] = False                       # the k-th score may tie with rows left outside the list
        ref_rank_scores = float((s2.to(torch.float16) == rs).float().mean())
        ref_rank_ids_all = float((i2 == ri).float().mean())
        ref_rank_ids_distinct = float((i2 == ri)[uniq].float().mean()) if bool(uniq.any()) else float("nan")
        ms_rr = timeit(lambda: ops.search_topk(q, corpus, k, reference_ranking=True), iters)
    passes = (Q + 127) // 128
    peak, src = peak_gbs()
    gbs = passes * N * d * 2 / (ms * 1e-3) / 1e9
    print(json.dumps({"N": N, "d": d, "Q": Q, "k": k, "ms": round(ms, 3), "ms_torch_reference_path": round(ms_ref, 3),
                      "speedup": round(ms_ref / ms, 2), "queries_per_s": round(Q / ms * 1e3, 1),
                      "corpus_stream_GBs": round(gbs, 1) if passes == 1 else None, "hbm_peak_GBs": peak,
                      "hbm_frac": round(gbs / peak, 3) if passes == 1 else None,   # Q > 128: query tiles share the stream via L2 (tensor-bound there), no HBM fraction
                      "reference_ranking": {"ms": round(ms_rr, 3), "fp16_scores_equal": round(ref_rank_scores, 5),
                                            "ids_equal_all": round(ref_rank_ids_all, 5),
                                            "ids_equal_where_reference_fp16_score_is_unique": round(ref_rank_ids_distinct, 5),
                                            "unique_fraction": round(float(uniq.float().mean()), 4) if not os.environ.get("SEARCH_BENCH_SKIP_REF") else None},
                      "tflops": round(2.0 * Q * N * d / (ms * 1e-3) / 1e12, 1),
                      "peak_source": src, "fp16_scores_equal": round(same_scores, 5), "ids_equal": round(same_ids, 5)}),
          flush=True)
    del corpus


if __name__ == "__main__":
    a = [int(x) for x in sys.argv[1:]]
    cfgs = [tuple(a[i:i + 4]) for i in range(0, len(a), 4)] or [
        (8841823, 768, 100, 100), (8841823, 768, 1000, 100), (21015324, 768, 100, 100)]
    for c in cfgs:
        run(*c)
