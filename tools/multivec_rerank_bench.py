#!/usr/bin/env python3
"""COIL and CITADEL reranking throughput, one JSON line per result on stdout.

  python tools/multivec_rerank_bench.py [--rounds 3] [--iters 2] [--out DIR]

Workload: BERT-base-dims COIL (token projection 128, CLS 128) and CITADEL (token projection 32, CLS 128, one expert per
token) encoders with seeded weights (tests/multivec_cases.py), shared by queries and passages, add_cls on; 1024
(query, passage) pairs, queries of at most 32 tokens, passages ~ U{S/3..S} with S = 256, in batches of 128, each side
padded to its longest, every query repeated over 8 consecutive pairs (tools/colbert_rerank_bench.py's batches).  Two
implementations with the same weights, alternated `rounds` times:
  dprb   RerankMultiVecRetrieverTask's step: each distinct query encoded once (dprb_encoder_fwd_tokens, the projection
         GEMMs and, for CITADEL, the router on dprb_search_topk), the passages likewise, then dprb_maxsim_expert_fwd;
  stock  HF BertModel / BertForMaskedLM + Linear under torch.no_grad + torch.autocast(bf16) with SDPA attention, the
         encoders' outputs as the reference computes them (CITADEL: log(1 + relu(logits)) * mask and its top-1, without
         the training statistics the reference's forward also computes), then the expert-matched bmm / max / sum and
         the CLS dot product (one query row per pair).
Each timing is `iters` passes over the 1024 pairs between CUDA events after one warm-up pass.  Also timed: the scoring
kernel alone against the stock scoring on one batch's tokens, and the CITADEL router alone (dprb: the head's GEMM,
LayerNorm and dprb_search_topk; stock: the HF masked-LM head and torch.topk over the logits) on one batch of passages.
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


def stock_expert_scores(q, d):
    """The expert-matched MaxSim + CLS term on the stock encoders' outputs (ids [B, L] or [B, L, 1])."""
    s = torch.bmm(q["expert_repr"], d["expert_repr"].permute(0, 2, 1))
    qi, di = q["expert_ids"].view(s.shape[0], -1), d["expert_ids"].view(s.shape[0], -1)
    qw, dw = q["expert_weights"].view(qi.shape), d["expert_weights"].view(di.shape)
    match = (qi.unsqueeze(2) == di.unsqueeze(1)).to(s.dtype) * (qw.unsqueeze(2) * dw.unsqueeze(1)).to(s.dtype)
    return (s * match).max(-1).values.sum(1) + (q["cls_repr"] * d["cls_repr"]).sum(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/multivec_rerank_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("multivec_rerank_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from transformers import BertConfig, BertForMaskedLM, BertModel
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.citadel_model import CITADELEncoder
    from dpr_scale_b200.models.citadel_models.coil_model import COILEncoder
    from dpr_scale_b200.models.citadel_models.colbert_model import encode_tokens
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    from tests import multivec_cases
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(what="gpu", **gpu_info()))
    data = batches(S, dev)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    for model in ("coil", "citadel"):
        sd, cfg = multivec_cases.bert_base_state_dict(model)
        proj_dim, cls_dim = multivec_cases.BASE[model]
        enc = (COILEncoder if model == "coil" else CITADELEncoder).from_config(cfg, proj_dim, cls_dim)
        enc.load_state_dict(sd, strict=True)
        enc = enc.to(dev)
        task = RerankMultiVecRetrieverTask.__new__(RerankMultiVecRetrieverTask)      # the eval step only
        torch.nn.Module.__init__(task)
        task.query_encoder = task.context_encoder = enc
        task.query_pool, task.dedupe_queries, task.add_cls, task.query_topk, task.context_topk = "sum", True, True, 1, 1
        hf_cfg = BertConfig(**cfg, attn_implementation="sdpa")
        if model == "coil":
            hf = BertModel(hf_cfg)
            hf.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")})
        else:
            hf = BertForMaskedLM(hf_cfg)
            hf.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")},
                               strict=False)
        tok = torch.nn.Linear(768, proj_dim)
        cls = torch.nn.Linear(768, cls_dim)
        tok_key = "project" if model == "coil" else "tok_project"
        tok.load_state_dict({"weight": sd[f"{tok_key}.0.weight"], "bias": sd[f"{tok_key}.0.bias"]})
        cls.load_state_dict({"weight": sd["cls_project.0.weight"], "bias": sd["cls_project.0.bias"]})
        hf, tok, cls = hf.to(dev).eval(), tok.to(dev).eval(), cls.to(dev).eval()

        def stock_repr(t):
            am = t["attention_mask"][:, 1:]
            if model == "coil":
                h = hf(**t, output_hidden_states=True).hidden_states[-1]
                ids, w = t["input_ids"][:, 1:], am
            else:
                out = hf(**t, output_hidden_states=True)
                h = out.hidden_states[-1]
                w, ids = torch.topk(torch.log(1 + torch.relu(out.logits[:, 1:])) * am.unsqueeze(-1), dim=2, k=1)
            return {"expert_repr": tok(h[:, 1:]) * am.unsqueeze(-1), "expert_ids": ids, "expert_weights": w,
                    "cls_repr": cls(h[:, 0])}

        def run_dprb():
            for b in data:
                task._scores(b)

        @torch.no_grad()
        def run_stock():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                for b in data:
                    stock_expert_scores(stock_repr(b["query_ids"]), stock_repr(b["contexts_ids"]))

        b = data[0]
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            ref = stock_expert_scores(stock_repr(b["query_ids"]), stock_repr(b["contexts_ids"])).float()
        emit(dict(what="agreement", model=model, max_abs_dscore=float((task._scores(b) - ref).abs().max()),
                  max_abs_score=float(ref.abs().max())))
        with torch.no_grad():
            qr, qi, qw, qc = enc.expert_reps(b["query_ids"], topk=1, add_cls=True)
            dr, di, dw, dc = enc.expert_reps(b["contexts_ids"], topk=1, add_cls=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                qs, ds = stock_repr(b["query_ids"]), stock_repr(b["contexts_ids"])
            hidden, _, _, _ = encode_tokens(enc._body, b["contexts_ids"])
        idx = torch.arange(BATCH, dtype=torch.int32)
        res = {k: [] for k in ("dprb", "stock", "kernel", "stock_scoring", "router", "stock_router")}
        for rnd in range(args.rounds):
            for impl, fn in (("dprb", run_dprb), ("stock", run_stock)):
                ms = events_ms(fn, args.iters, warmup=1)
                res[impl].append(PAIRS / (ms / 1e3))
                emit(dict(what="multivec_rerank", model=model, impl=impl, S=S, round=rnd, ms_per_1024_pairs=ms,
                          pairs_per_s=PAIRS / (ms / 1e3)))
            scoring = [("kernel", lambda: ops.maxsim_expert(qr, dr, qi, qw, di, dw, idx, "sum", qc, dc)),
                       ("stock_scoring", lambda: stock_expert_scores(qs, ds))]
            if model == "citadel":
                head = hf.cls

                def stock_router():
                    with torch.autocast("cuda", dtype=torch.bfloat16):
                        torch.topk(head(hidden.view(BATCH, -1, 768)), dim=2, k=1)
                scoring += [("router", lambda: enc.route(hidden, 1)), ("stock_router", stock_router)]
            with torch.no_grad():
                for impl, fn in scoring:
                    ms = events_ms(fn, 20, warmup=3)
                    res[impl].append(ms * 1e3)
                    emit(dict(what="component", model=model, impl=impl, S=S, round=rnd, us_per_batch_of_128=ms * 1e3))
        summary = dict(what="multivec_rerank_summary", model=model, S=S,
                       workload=f"bert-base {model} {multivec_cases.BASE[model]}, add_cls, 1 expert per token, {PAIRS} "
                       f"pairs, queries <= {QLEN} tokens, passages U{{S/3..S}}, batches of {BATCH} padded to the "
                       "longest, 8 pairs per query",
                       dprb_pairs_per_s=med(res["dprb"]), stock_pairs_per_s=med(res["stock"]),
                       ratio=med(res["dprb"]) / med(res["stock"]), kernel_us_per_batch=med(res["kernel"]),
                       stock_scoring_us_per_batch=med(res["stock_scoring"]), dprb_all=res["dprb"],
                       stock_all=res["stock"])
        if model == "citadel":
            summary.update(router_us_per_batch=med(res["router"]), stock_router_us_per_batch=med(res["stock_router"]))
        emit(summary)
        del enc, hf, task
        torch.cuda.empty_cache()
    emit(dict(what="gpu_after", **gpu_info()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "multivec_rerank_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
