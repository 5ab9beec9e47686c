#!/usr/bin/env python3
"""SPAR measurements on one GPU; prints one JSON line per measurement, each with the card's name and power limit:
  spar_encode  SalientPhraseAwareDenseRetrieverTask.encode_contexts with two BERT-base encoders loaded from checkpoints
               (S = 128, 512 passages per batch) vs two stock HF BertModels under fp16 autocast: passages/s;
  spar_search  ops.search_topk over an MS MARCO-sized store (8 841 823 passages) of the 1536-wide concatenation,
               against the 768-wide single-model store, 6 980 queries, k = 100: ms and queries/s;
  spar_tune    tune_spar_weights over 300 questions (200 000 passages, 768-wide models), default 19 weights, by stage
               (load, answer matching, pool scoring + per-weight accuracy, writing the 19 runs), and the same
               accuracies computed the reference's way: eval_dpr over each written run (19 matching passes).
  python tools/spar_bench.py [--out profiles/h100_spar_bench.jsonl]
"""
import argparse
import json
import os
import pickle
import random
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512)
MSMARCO_PASSAGES, MSMARCO_DEV_QUERIES = 8_841_823, 6_980


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa
        pl = f"unknown ({e})"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_encode(emit, steps, warmup):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.task.spar_task import SalientPhraseAwareDenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    N, S = 512, 128
    gen = torch.Generator().manual_seed(2)
    ids = torch.randint(1000, 30000, (N, S), generator=gen)
    ids[:, 0] = 101
    toks = {"input_ids": ids.cuda(), "token_type_ids": torch.zeros_like(ids).cuda(),
            "attention_mask": torch.ones_like(ids).cuda()}
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for seed in (0, 1):
            torch.manual_seed(seed)
            t = DenseRetrieverTask(transform={}, datamodule=None, optim={}, shared_model=False,
                                   model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                          "config": BERT_BASE, "dropout": 0.0})
            t.setup("fit")
            paths.append(os.path.join(tmp, f"m{seed}.ckpt"))
            torch.save(ModelCheckpoint._payload(t, 0, 0), paths[-1])
            del t
        spar = SalientPhraseAwareDenseRetrieverTask(pretrained_checkpoint_path=paths[0],
                                                    lexical_model_checkpoint_path=paths[1], lexical_weight=0.5,
                                                    transform={}, model={}, datamodule=None, optim={})
        spar.setup("test")
    spar = spar.cuda().eval()

    @torch.no_grad()
    def ours():
        return spar.encode_contexts(toks)
    ms = timed(ours, steps, warmup)
    del spar
    torch.cuda.empty_cache()
    from transformers import BertConfig, BertModel
    stock = [BertModel(BertConfig(**BERT_BASE), add_pooling_layer=False).cuda().eval() for _ in range(2)]

    @torch.no_grad()
    def hf():
        with torch.autocast("cuda", dtype=torch.float16):
            return torch.cat([m(**toks).last_hidden_state[:, 0, :].float() for m in stock], 1)
    ms_s = timed(hf, steps, warmup)
    del stock
    torch.cuda.empty_cache()
    emit({"metric": "spar_encode", "encoders": 2, "passages": N, "S": S, "ms_per_batch": ms,
          "passages_per_s": N / (ms * 1e-3), "stock_ms_per_batch": ms_s, "stock_passages_per_s": N / (ms_s * 1e-3),
          "speedup": ms_s / ms})


def bench_search(emit, steps, warmup):
    from dpr_scale_b200 import ops
    N, Q, k = MSMARCO_PASSAGES, MSMARCO_DEV_QUERIES, 100
    g = torch.Generator(device="cuda").manual_seed(5)
    store = torch.empty(N, 1536, dtype=torch.float16, device="cuda")
    for r in range(0, N, 1 << 20):
        store[r:r + (1 << 20)] = torch.randn(min(1 << 20, N - r), 1536, device="cuda", generator=g).half()
    q = torch.randn(Q, 1536, device="cuda", generator=g).half()
    res = {}
    ms = timed(lambda: ops.search_topk(q, store, k), steps, warmup)
    res[1536] = ms
    del store
    torch.cuda.empty_cache()
    single = torch.empty(N, 768, dtype=torch.float16, device="cuda")
    for r in range(0, N, 1 << 20):
        single[r:r + (1 << 20)] = torch.randn(min(1 << 20, N - r), 768, device="cuda", generator=g).half()
    q1 = q[:, :768].contiguous()
    res[768] = timed(lambda: ops.search_topk(q1, single, k), steps, warmup)
    del single
    torch.cuda.empty_cache()
    for d, ms in res.items():
        emit({"metric": "spar_search", "width": d, "passages": N, "queries": Q, "k": k, "store_GB": N * d * 2 / 1e9,
              "ms": ms, "queries_per_s": Q / (ms * 1e-3), "ms_over_768_wide": ms / res[768]})


def bench_tune(emit, device="cuda"):
    from dpr_scale_b200 import eval_dpr
    from dpr_scale_b200.tune_spar_weights import DEFAULT_WEIGHTS, grid_search_weights
    Q, N, D, K = 300, 200_000, 768, 100
    rnd = random.Random(3)
    words = [f"w{i}" for i in range(5000)]
    g = torch.Generator().manual_seed(4)
    with tempfile.TemporaryDirectory() as tmp:
        questions = [{"question": f"question {i}", "answers": [f"{rnd.choice(words)} {rnd.choice(words)}"]}
                     for i in range(Q)]
        texts = {}

        def text(row):
            if row not in texts:
                texts[row] = " ".join(rnd.choice(words) for _ in range(100))
            return texts[row]
        shared = [rnd.sample(range(N), K) for _ in range(Q)]
        for m in (1, 2):
            d = os.path.join(tmp, f"m{m}")
            os.makedirs(d)
            for i, n in enumerate((N // 2, N - N // 2)):
                with open(os.path.join(d, f"reps_{i:04}.pkl"), "wb") as f:
                    pickle.dump(torch.randn(n, D, generator=g), f, protocol=4)
            with open(os.path.join(d, "query_reps.pkl"), "wb") as f:
                pickle.dump(torch.randn(Q, D, generator=g), f, protocol=4)
            run = []
            for i, q in enumerate(questions):
                rows = shared[i][:K // 2] + rnd.sample(range(N), K // 2) if m == 2 else shared[i]
                rows = list(dict.fromkeys(rows))[:K]
                run.append(dict(q, ctxs=[{"id": str(r + 1), "title": "t", "text": text(r), "score": 0.0}
                                         for r in rows], id=str(i)))
            for i in range(0, Q, 4):                  # plant answers in a quarter of the questions' pools
                c = run[i]["ctxs"][rnd.randrange(K)]
                c["text"] = c["text"] + " " + questions[i]["answers"][0]
            with open(os.path.join(d, "dev.json"), "w") as f:
                json.dump(run, f)
        timings = {}
        t0 = time.perf_counter()
        grid_search_weights(os.path.join(tmp, "m1"), os.path.join(tmp, "m2"), "dev.json", "query_reps.pkl",
                            output_dir=os.path.join(tmp, "out"), device=device, timings=timings)
        total = time.perf_counter() - t0
        t0 = time.perf_counter()
        for w in DEFAULT_WEIGHTS:
            eval_dpr.evaluate_retrieval(os.path.join(tmp, "out", f"weight{w}_dev.json"), [1, 5, 10, 20, 50, 100])
        per_weight = time.perf_counter() - t0
    emit({"metric": "spar_tune", "questions": Q, "passages": N, "width": D, "weights": len(DEFAULT_WEIGHTS),
          "cpu_cores": os.cpu_count(), "stage_s": timings, "total_s": total,
          "per_weight_matching_s": per_weight,
          "matching_once_over_per_weight": timings["answer_matching"] / per_weight})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "spar_bench measures on the GPU; there is no CPU path"
    info = card()
    lines = []

    def emit(d):
        d = dict(d, **info)
        lines.append(d)
        print(json.dumps(d), flush=True)
    bench_encode(emit, args.steps, args.warmup)
    bench_search(emit, args.steps, args.warmup)
    bench_tune(emit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
