#!/usr/bin/env python3
"""Cross-encoder training throughput, one JSON line per result on stdout.

  python tools/cross_encoder_train_bench.py [--rounds 3] [--iters 5] [--out DIR]

Workload: a BERT-base-dims BertForSequenceClassification(num_labels=1) (seeded weights, dropout 0.1), batches of 16
questions x 8 candidates = 128 (query, passage) pairs at S = 256 (lengths ~ U{S/3..S} with segment-B token types, the
batch padded to its longest pair, which is S), the grouped softmax cross-entropy with label 0.  One training step
(zero_grad, forward, loss, backward, optimizer step) of two implementations on the same GPU from the same weights,
alternated `rounds` times:
  dprb   CrossEncoder.group_ce (HFEncoder training forward / backward, dprb_seqcls_group_ce, the library's GEMMs) and
         FusedAdamW over the body arena;
  stock  the HF model in train mode under torch.autocast(bf16) with SDPA attention, torch cross_entropy and
         torch.optim.AdamW.
Each timing is `iters` steps between CUDA events after two warm-up steps.  The dprb_seqcls_group_ce kernel is also
timed alone on the step's [128, 768] head input.  The card name, power limit and SM clocks (nvidia-smi) are read in the
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

Q, G, S, LR = 16, 8, 256, 1e-5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/cross_encoder_train_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cross_encoder_train_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from transformers import BertConfig, BertForSequenceClassification

    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    from dpr_scale_b200.optim import FusedAdamW
    from tests.rerank_cases import BERT_BASE, pair_tokens
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(what="gpu", **gpu_info()))
    cfg = dict(BERT_BASE, model_type="bert", num_labels=1, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    torch.manual_seed(0)
    stock = BertForSequenceClassification(BertConfig(**cfg))
    stock.config._attn_implementation = "sdpa"
    dprb = CrossEncoder.from_config(cfg)
    dprb.load_state_dict({"transformer." + k: v for k, v in stock.state_dict().items()
                          if not k.endswith(("position_ids", "token_type_ids"))}, strict=True)
    dprb, stock = dprb.to(dev).train(), stock.to(dev).train()
    opt_d = FusedAdamW(dprb.parameters(), lr=LR)
    opt_d.attach_encoders([dprb._body])
    opt_s = torch.optim.AdamW(stock.parameters(), lr=LR)
    gen = torch.Generator().manual_seed(S)
    tok = {k: v.to(dev) for k, v in pair_tokens(gen, Q * G, S, 30522, 0, lo=1000, cls_id=101, sep_id=102).items()}
    labels = torch.zeros(Q, dtype=torch.int64, device=dev)

    def step_dprb():
        opt_d.zero_grad()
        loss, _ = dprb.group_ce(tok, labels, G)
        loss.backward()
        opt_d.step()

    def step_stock():
        opt_s.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = stock(**tok).logits.float().view(Q, G)
        torch.nn.functional.cross_entropy(logits, labels).backward()
        opt_s.step()

    H = cfg["hidden_size"]
    g = torch.Generator().manual_seed(1)
    pre, W, b = 2.0 * torch.randn(Q * G, H, generator=g), 0.05 * torch.randn(1, H, generator=g), torch.zeros(1)
    pre, W, b = pre.to(dev), W.to(dev), b.to(dev)
    kernel_ms = events_ms(lambda: ops.seqcls_group_ce(pre, W, b, labels, G, 0.1, 5), 200, warmup=5)
    emit(dict(what="seqcls_group_ce", N=Q * G, H=H, G=G, dropout_p=0.1, us_per_call=kernel_ms * 1e3,
              note="two launches (group pass + fixed-order final sum), ops wrapper allocations included"))
    res = {"dprb": [], "stock": []}
    for rnd in range(args.rounds):
        for impl, fn in (("dprb", step_dprb), ("stock", step_stock)):
            ms = events_ms(fn, args.iters, warmup=2)
            res[impl].append(Q * G / (ms / 1e3))
            emit(dict(what="train_step", impl=impl, round=rnd, ms_per_step=ms, pairs_per_s=Q * G / (ms / 1e3)))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    emit(dict(what="train_summary", workload=f"bert-base num_labels=1 dropout 0.1, {Q} questions x {G} candidates, "
              f"S={S}, grouped cross-entropy, AdamW", dprb_pairs_per_s=med(res["dprb"]),
              stock_pairs_per_s=med(res["stock"]), ratio=med(res["dprb"]) / med(res["stock"]),
              dprb_all=res["dprb"], stock_all=res["stock"]))
    emit(dict(what="gpu_after", **gpu_info()))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cross_encoder_train_bench.jsonl"), "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
