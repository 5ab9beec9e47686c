#!/usr/bin/env python3
"""SPLADE and dense (DPR) reranking throughput, one JSON line per result on stdout.

  python tools/splade_rerank_bench.py [--rounds 3] [--iters 2] [--out DIR]

Workload: BERT-base dims with seeded weights (tests/splade_cases.py, tests/colbert_cases.py), encoders shared by queries
and passages; 1024 (query, passage) pairs, queries of at most 32 tokens, passages ~ U{S/3..S} with S = 256, in batches
of 128, each side padded to its longest, every query repeated over 8 consecutive pairs (tools/colbert_rerank_bench.py's
batches).  Implementations are alternated `rounds` times; each timing is `iters` passes between CUDA events after one
warm-up pass.
  (a) pool: on one batch's passages (the valid tokens 1.. compacted, the head's transform from the SPLADE encoder),
      dprb_splade_pool_fwd against the library's GEMM with DPRB_EPI_F32_STORE into [T, V padded to 8] fp32 logits
      followed by torch's relu / log1p / segmented max (torch.segment_reduce).  Achieved TFLOP/s = 2 T V H over the
      kernel time, against the data-sheet 989 TFLOP/s (dense fp16, H100 SXM at 700 W).
  (b) splade: RerankDenseRetrieverTask's step with SPLADEEncoder (each distinct query once, the fused pool) against HF
      BertForMaskedLM under torch.no_grad + torch.autocast(bf16) with SDPA attention and the reference's pooling
      (max over tokens 1.. of log(1 + relu(logits)) * mask), one query row per pair, then sum(q * d, 1).
  (c) dpr: the same task with HFEncoder (CLS, no projection, the CLS-pruned forward) against HF BertModel the same way.
The card name, power limit and SM clocks (nvidia-smi) are read in the same call, before and after.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from colbert_rerank_bench import BATCH, PAIRS, QLEN, batches  # noqa: E402
from long_seq_bench import events_ms, gpu_info  # noqa: E402

S = 256
PEAK_TFLOPS = 989.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/splade_rerank_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("splade_rerank_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from transformers import BertConfig, BertForMaskedLM, BertModel
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.colbert_model import encode_tokens
    from dpr_scale_b200.models.citadel_models.splade_model import SPLADEEncoder
    from dpr_scale_b200.models.hf_model import HFEncoder
    from dpr_scale_b200.task.dpr_rerank_task import RerankDenseRetrieverTask
    from tests import colbert_cases, splade_cases
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(what="gpu", **gpu_info()))
    data = batches(S, dev)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    workload = (f"bert-base, {PAIRS} pairs, queries <= {QLEN} tokens, passages U{{S/3..S}}, batches of {BATCH} padded "
                "to the longest, 8 pairs per query")

    def make_task(enc):
        task = RerankDenseRetrieverTask.__new__(RerankDenseRetrieverTask)     # the eval step only
        torch.nn.Module.__init__(task)
        task.query_encoder = task.context_encoder = enc
        task.dedupe_queries = True
        return task

    # ---------------------------------------------------------------- SPLADE: (a) and (b)
    sd, cfg = splade_cases.bert_base_state_dict()
    enc = SPLADEEncoder.from_config(cfg)
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(dev)
    hf = BertForMaskedLM(BertConfig(**cfg, attn_implementation="sdpa"))
    hf.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")},
                       strict=False)
    hf = hf.to(dev).eval()
    H, V = cfg["hidden_size"], cfg["vocab_size"]
    Vp = (V + 7) // 8 * 8

    # (a) the pool on one batch of passages
    d = data[0]["contexts_ids"]
    with torch.no_grad():
        hidden, am, N, Sd = encode_tokens(enc._body, d)
        keep = am != 0
        keep[:, 0] = False
        lens = keep.sum(1)
        off = torch.zeros(N + 1, dtype=torch.int32, device=dev)
        off[1:] = torch.cumsum(lens, 0)
        x = enc.router_tokens(hidden[keep.view(-1).nonzero().squeeze(1)])
        W = enc.router_operand()
        bias = enc.router_bias().detach().float().contiguous()
    T = x.shape[0]
    W_pad = torch.zeros(Vp, H + 8, dtype=torch.float16, device=dev)
    W_pad[:V] = W
    bias_pad = torch.zeros(Vp, device=dev)
    bias_pad[:V] = bias
    logits = torch.empty(T, Vp, device=dev)
    epi = ops.EPI_F32_STORE | ops.GEMM_A_F16 | ops.GEMM_B_F16

    def pool_dprb():
        return ops.splade_pool(x, W, off, H, bias)

    def pool_gemm_only():
        ops.gemm(x, W_pad, logits, T, Vp, H, H + 8, H + 8, Vp, False, False, epi, bias_pad)

    def pool_stock():
        pool_gemm_only()
        return torch.segment_reduce(torch.log1p(torch.relu(logits[:, :V])), "max", lengths=lens, axis=0, unsafe=True,
                                    initial=0.0)

    emit(dict(what="agreement", part="pool", max_abs_diff=float((pool_dprb() - pool_stock()).abs().max()),
              max_abs=float(pool_stock().abs().max())))
    flop = 2.0 * T * V * H
    res = {k: [] for k in ("pool", "pool_stock", "pool_stock_gemm")}
    for rnd in range(args.rounds):
        for impl, fn in (("pool", pool_dprb), ("pool_stock", pool_stock), ("pool_stock_gemm", pool_gemm_only)):
            ms = events_ms(fn, 20, warmup=3)
            res[impl].append(ms)
            emit(dict(what="pool", impl=impl, round=rnd, T=T, V=V, K=H, ms=ms, tflops=flop / (ms * 1e-3) / 1e12))
    emit(dict(what="pool_summary", T=T, V=V, K=H, tokens_per_passage_max=int(Sd), pool_ms=med(res["pool"]),
              stock_ms=med(res["pool_stock"]), stock_gemm_only_ms=med(res["pool_stock_gemm"]),
              speedup=med(res["pool_stock"]) / med(res["pool"]),
              pool_tflops=flop / (med(res["pool"]) * 1e-3) / 1e12,
              pool_share_of_989=flop / (med(res["pool"]) * 1e-3) / 1e12 / PEAK_TFLOPS,
              note="pool_tflops: 2 T V K over the measured time of the three launches (zero-fill, pool, log1p)"))
    del logits, W_pad

    # (b) SPLADE rerank end to end
    task = make_task(enc)

    def splade_stock_repr(t):
        lg = hf(**t).logits[:, 1:]
        return torch.max(torch.log(1 + torch.relu(lg)) * t["attention_mask"][:, 1:].unsqueeze(-1), dim=1).values

    def dense_run(task):
        def run():
            for b in data:
                task._scores(b)
        return run

    def stock_run(repr_fn):
        @torch.no_grad()
        def run():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                for b in data:
                    (repr_fn(b["query_ids"]).float() * repr_fn(b["contexts_ids"]).float()).sum(1)
        return run

    def bench_e2e(name, task, repr_fn):
        b = data[0]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = (repr_fn(b["query_ids"]).float() * repr_fn(b["contexts_ids"]).float()).sum(1)
        emit(dict(what="agreement", part=name, max_abs_dscore=float((task._scores(b) - ref).abs().max()),
                  max_abs_score=float(ref.abs().max())))
        r = {"dprb": [], "stock": []}
        for rnd in range(args.rounds):
            for impl, fn in (("dprb", dense_run(task)), ("stock", stock_run(repr_fn))):
                ms = events_ms(fn, args.iters, warmup=1)
                r[impl].append(PAIRS / (ms / 1e3))
                emit(dict(what=f"{name}_rerank", impl=impl, S=S, round=rnd, ms_per_1024_pairs=ms,
                          pairs_per_s=PAIRS / (ms / 1e3)))
        emit(dict(what=f"{name}_rerank_summary", S=S, workload=workload, dprb_pairs_per_s=med(r["dprb"]),
                  stock_pairs_per_s=med(r["stock"]), ratio=med(r["dprb"]) / med(r["stock"]), dprb_all=r["dprb"],
                  stock_all=r["stock"]))

    bench_e2e("splade", task, splade_stock_repr)
    del enc, hf, task
    torch.cuda.empty_cache()

    # ---------------------------------------------------------------- (c) DPR rerank end to end
    csd, ccfg = colbert_cases.bert_base_state_dict()
    body = {k: v for k, v in csd.items() if k.startswith("transformer.")}
    henc = HFEncoder.from_config(ccfg, dropout=0.0)
    henc.load_state_dict(body, strict=True)
    henc = henc.to(dev).eval()
    bm = BertModel(BertConfig(**ccfg, attn_implementation="sdpa"))
    bm.load_state_dict({k[len("transformer."):]: v for k, v in body.items()})
    bm = bm.to(dev).eval()
    bench_e2e("dpr", make_task(henc), lambda t: bm(**t)[0][:, 0])
    emit(dict(what="gpu_after", **gpu_info()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "splade_rerank_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
