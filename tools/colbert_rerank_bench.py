#!/usr/bin/env python3
"""ColBERT (late-interaction) reranking throughput, one JSON line per result on stdout.

  python tools/colbert_rerank_bench.py [--rounds 3] [--iters 3] [--out DIR]

Workload: a BERT-base-dims ColBERT encoder with a 128-wide projection (seeded weights, tests/colbert_cases.py), shared by
queries and passages; 1024 (query, passage) pairs per S in {128, 256, 512}, queries of at most 32 tokens, passages
~ U{S/3..S}, in batches of 128, each side padded to its longest.  Every query is repeated over 8 consecutive pairs, as a
reranked run lists one query's passages together.  Two implementations with the same weights, alternated `rounds` times:
  dprb   RerankMultiVecRetrieverTask's step: each distinct query encoded once (dprb_encoder_fwd_tokens + the projection
         GEMM), the passages likewise, then dprb_maxsim_fwd on the unmasked tokens and the masks;
  stock  the HF BertModel + Linear under torch.no_grad + torch.autocast(bf16) with SDPA attention, expert_repr masked as
         the reference's ColBERTEncoder does, then the reference's bmm / max / sum (one query row per pair).
Each timing is `iters` passes over the 1024 pairs between CUDA events after one warm-up pass.  The MaxSim kernel alone
is also timed against the bmm / max / sum on the same bf16 tokens.  The largest score difference between the two
implementations on the first batch is reported.  The card name, power limit and SM clocks (nvidia-smi) are read in the
same call, before and after.
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

PAIRS, BATCH, SEQ_LENS, QLEN, PER_QUERY = 1024, 128, (128, 256, 512), 32, 8


def batches(S, dev):
    from tests.colbert_cases import seq_tokens
    gen = torch.Generator().manual_seed(S)
    out = []
    for _ in range(0, PAIRS, BATCH):
        q = seq_tokens(gen, BATCH // PER_QUERY, QLEN, 30522, 0, lo=1000, cls_id=101, sep_id=102, min_len=4)
        q = {k: v.repeat_interleave(PER_QUERY, 0) for k, v in q.items()}
        d = seq_tokens(gen, BATCH, S, 30522, 0, lo=1000, cls_id=101, sep_id=102)
        d = {k: v[torch.randperm(BATCH, generator=gen)] for k, v in d.items()}      # the full-length row anywhere
        qw, dw = int(q["attention_mask"].sum(1).max()), int(d["attention_mask"].sum(1).max())
        qid = [f"q{len(out)}_{i // PER_QUERY}" for i in range(BATCH)]
        out.append({"qid": qid, "query_ids": {k: v[:, :qw].contiguous().to(dev) for k, v in q.items()},
                    "contexts_ids": {k: v[:, :dw].contiguous().to(dev) for k, v in d.items()}})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/colbert_rerank_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("colbert_rerank_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from transformers import BertConfig, BertModel
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    from tests.colbert_cases import BASE_P, bert_base_state_dict
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(what="gpu", **gpu_info()))
    sd, cfg = bert_base_state_dict()
    enc = ColBERTEncoder.from_config(cfg, projection_dim=BASE_P)
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(dev)
    task = RerankMultiVecRetrieverTask.__new__(RerankMultiVecRetrieverTask)      # the eval step only: no checkpoint
    torch.nn.Module.__init__(task)
    task.query_encoder = task.context_encoder = enc
    task.query_pool, task.dedupe_queries = "sum", True
    body = BertModel(BertConfig(**cfg, attn_implementation="sdpa"))
    body.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")})
    proj = torch.nn.Linear(768, BASE_P)
    proj.load_state_dict({"weight": sd["project.0.weight"], "bias": sd["project.0.bias"]})
    body, proj = body.to(dev).eval(), proj.to(dev).eval()
    data = {S: batches(S, dev) for S in SEQ_LENS}

    def stock_repr(tok):
        h = proj(body(**tok).last_hidden_state[:, 1:, :])
        return tok["attention_mask"][:, 1:].unsqueeze(-1) * h

    def stock_scores(q, d):
        return torch.bmm(q, d.permute(0, 2, 1)).max(-1).values.sum(1)

    def run_dprb(S):
        for b in data[S]:
            task._scores(b)

    @torch.no_grad()
    def run_stock(S):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            for b in data[S]:
                stock_scores(stock_repr(b["query_ids"]), stock_repr(b["contexts_ids"]))

    for S in SEQ_LENS:
        b = data[S][0]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = stock_scores(stock_repr(b["query_ids"]), stock_repr(b["contexts_ids"])).float()
        emit(dict(what="agreement", S=S, max_abs_dscore=float((task._scores(b) - ref).abs().max()),
                  max_abs_score=float(ref.abs().max()), query_width=int(b["query_ids"]["input_ids"].shape[1]),
                  passage_width=int(b["contexts_ids"]["input_ids"].shape[1])))
    res = {(impl, S): [] for impl in ("dprb", "stock", "maxsim", "bmm") for S in SEQ_LENS}
    for rnd in range(args.rounds):
        for S in SEQ_LENS:
            for impl, fn in (("dprb", run_dprb), ("stock", run_stock)):
                ms = events_ms(lambda: fn(S), args.iters, warmup=1)
                res[(impl, S)].append(PAIRS / (ms / 1e3))
                emit(dict(what="colbert_rerank", impl=impl, S=S, round=rnd, ms_per_1024_pairs=ms,
                          pairs_per_s=PAIRS / (ms / 1e3)))
            # the scoring alone, on one batch's tokens: dprb_maxsim_fwd against the reference's bmm / max / sum
            b = data[S][0]
            with torch.no_grad():
                qr, qm = enc.token_reps(b["query_ids"])
                dr, dm = enc.token_reps(b["contexts_ids"])
                qz = (qr[:, 1:] * qm[:, 1:, None].to(qr.dtype)).contiguous()
                dz = (dr[:, 1:] * dm[:, 1:, None].to(dr.dtype)).contiguous()
            idx = torch.arange(BATCH, dtype=torch.int32)
            for impl, fn in (("maxsim", lambda: ops.maxsim(qr, dr, qm, dm, idx, "sum")),
                             ("bmm", lambda: stock_scores(qz, dz))):
                ms = events_ms(fn, 50, warmup=5)
                res[(impl, S)].append(ms * 1e3)
                emit(dict(what="scoring_kernel", impl=impl, S=S, round=rnd, us_per_batch_of_128=ms * 1e3))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    for S in SEQ_LENS:
        emit(dict(what="colbert_rerank_summary", S=S,
                  workload=f"bert-base ColBERT P={BASE_P}, {PAIRS} pairs, queries <= {QLEN} tokens, passages "
                  f"U{{S/3..S}}, batches of {BATCH} padded to the longest, {PER_QUERY} pairs per query",
                  dprb_pairs_per_s=med(res[("dprb", S)]), stock_pairs_per_s=med(res[("stock", S)]),
                  ratio=med(res[("dprb", S)]) / med(res[("stock", S)]),
                  maxsim_us_per_batch=med(res[("maxsim", S)]), bmm_max_sum_us_per_batch=med(res[("bmm", S)]),
                  dprb_all=res[("dprb", S)], stock_all=res[("stock", S)]))
    emit(dict(what="gpu_after", **gpu_info()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "colbert_rerank_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
