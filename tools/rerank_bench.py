#!/usr/bin/env python3
"""Cross-encoder reranking throughput, one JSON line per result on stdout.

  python tools/rerank_bench.py [--rounds 3] [--iters 3] [--out DIR]

Workload: a BERT-base-dims BertForSequenceClassification(num_labels=1) (seeded weights), 1024 (query, passage) pairs
per S in {128, 256, 512}, lengths ~ U{S/3..S} with segment-B token types, in batches of 128 each padded to its longest
pair.  Two implementations on the same GPU with the same weights, alternated `rounds` times:
  dprb   CrossEncoder (forward-only encoder, CLS-pruned last layer, dprb head GEMM + dprb_seqcls_head_fwd);
  stock  the HF model under torch.no_grad + torch.autocast(bf16) with SDPA attention.
Each timing is `iters` passes over the 1024 pairs between CUDA events after one warm-up pass.  The largest logit
difference between the two on the first batch is reported next to the speeds.  The card name, power limit and SM
clocks (nvidia-smi) are read in the same call, before and after.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from long_seq_bench import events_ms, gpu_info  # noqa: E402

PAIRS, BATCH, SEQ_LENS = 1024, 128, (128, 256, 512)


def batches(S, dev):
    from tests.rerank_cases import pair_tokens
    gen = torch.Generator().manual_seed(S)
    out = []
    for lo in range(0, PAIRS, BATCH):
        t = pair_tokens(gen, BATCH, S, 30522, 0, lo=1000, cls_id=101, sep_id=102)
        t = {k: v[torch.randperm(BATCH, generator=gen)] for k, v in t.items()}   # the full-length row anywhere
        width = int(t["attention_mask"].sum(1).max())                             # pad to the batch's longest
        out.append({k: v[:, :width].contiguous().to(dev) for k, v in t.items()})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/rerank_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rerank_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    from tests.rerank_cases import bert_base_seqcls
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(what="gpu", **gpu_info()))
    stock, cfg = bert_base_seqcls()
    stock.config._attn_implementation = "sdpa"
    dprb = CrossEncoder.from_config(cfg)
    dprb.load_state_dict({"transformer." + k: v for k, v in stock.state_dict().items()
                          if not k.endswith(("position_ids", "token_type_ids"))}, strict=True)
    dprb, stock = dprb.to(dev), stock.to(dev).eval()
    data = {S: batches(S, dev) for S in SEQ_LENS}

    def run_dprb(S):
        for b in data[S]:
            dprb(b)

    @torch.no_grad()
    def run_stock(S):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            for b in data[S]:
                stock(**b).logits

    for S in SEQ_LENS:
        b = data[S][0]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = stock(**b).logits.float()
        emit(dict(what="agreement", S=S, max_abs_dlogit=float((dprb(b) - ref).abs().max()),
                  max_abs_logit=float(ref.abs().max()), width=int(b["input_ids"].shape[1])))
    res = {(impl, S): [] for impl in ("dprb", "stock") for S in SEQ_LENS}
    for rnd in range(args.rounds):
        for S in SEQ_LENS:
            for impl, fn in (("dprb", run_dprb), ("stock", run_stock)):
                ms = events_ms(lambda: fn(S), args.iters, warmup=1)
                res[(impl, S)].append(PAIRS / (ms / 1e3))
                emit(dict(what="rerank", impl=impl, S=S, round=rnd, ms_per_1024_pairs=ms, pairs_per_s=PAIRS / (ms / 1e3)))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    for S in SEQ_LENS:
        emit(dict(what="rerank_summary", S=S, workload=f"bert-base num_labels=1, {PAIRS} pairs, batches of {BATCH} "
                  f"padded to the longest, lengths U{{S/3..S}}", dprb_pairs_per_s=med(res[("dprb", S)]),
                  stock_pairs_per_s=med(res[("stock", S)]), ratio=med(res[("dprb", S)]) / med(res[("stock", S)]),
                  dprb_all=res[("dprb", S)], stock_all=res[("stock", S)]))
    emit(dict(what="gpu_after", **gpu_info()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rerank_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
