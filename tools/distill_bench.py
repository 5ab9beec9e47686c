#!/usr/bin/env python3
"""Distillation / DrBoost measurements on one GPU; prints one JSON line per measurement, each with the card's name and
power limit:

  sqerr        dprb_sqerr_fwd (loss + dx) vs torch ((x - t) ** 2).sum() and 2 * (x - t): time, GB/s over the bytes it
               must move (read x and t, write dx) and that rate's fraction of the H100 SXM data-sheet 3.35 TB/s;
  distill_step one DPRDistillTask step at BERT-base, S = 32, 128 questions (256 rows), target width 768, dropout 0.1,
               fused AdamW with clip 2.0, vs stock HF BertModel under fp16 autocast + GradScaler with
               nn.MSELoss(reduction="sum"), torch.optim.AdamW and the same clip: questions/s;
  host_batch   DPRDistillJsonlDataModule host assembly (JSON, sampling, vector parsing, tokenisation) per batch of
               128 questions with 768-wide vectors, next to the GPU step time above;
  drboost      passage encoding with K = 4 weak BERT-base encoders with a 32-dim projection (S = 128, 512 passages per
               batch) vs K stock HF encoders under fp16 autocast: passages/s.

  python tools/distill_bench.py [--out distill_bench.jsonl]
"""
import argparse
import json
import os
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
HBM_TBS = 3.35


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


def tokens(n, S, gen):
    ids = torch.randint(1000, 30000, (n, S), generator=gen)
    ids[:, 0] = 101
    am = torch.ones(n, S, dtype=torch.long)
    return {"input_ids": ids.cuda(), "token_type_ids": torch.zeros_like(ids).cuda(), "attention_mask": am.cuda()}


def bench_sqerr(emit):
    from dpr_scale_b200 import ops
    for rows, d in ((256, 768), (65536, 1024)):
        x = torch.randn(rows, d, device="cuda")
        t = torch.randn(rows, d, device="cuda")
        ms = timed(lambda: ops.sqerr(x, t), 200, 20)

        def stock():
            ((x - t) ** 2).sum()
            2 * (x - t)
        ms_t = timed(stock, 200, 20)
        nbytes = 3 * rows * d * 4
        gbs = nbytes / (ms * 1e-3) / 1e9
        emit({"metric": "sqerr", "rows": rows, "d": d, "bytes": nbytes, "ms": ms, "GB/s": gbs,
              "frac_of_3.35TB/s": gbs / (HBM_TBS * 1e3), "torch_ms": ms_t, "speedup": ms_t / ms})


def bench_step(emit, steps, warmup):
    from dpr_scale_b200.optim import FusedAdamW
    from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask
    gen = torch.Generator().manual_seed(0)
    B, S = 128, 32
    toks = tokens(B, S, gen)
    toks = {k: v.repeat_interleave(2, 0) for k, v in toks.items()}
    targets = torch.randn(2 * B, 768, generator=gen).cuda()
    task = DPRDistillTask(transform={}, datamodule=None, optim={},
                          model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                 "config": BERT_BASE, "dropout": 0.1})
    task.setup("fit")
    task = task.cuda().train()
    opt = FusedAdamW(task.parameters(), lr=1e-5, max_grad_norm=2.0)
    opt.attach_encoders([task.query_encoder])
    batch = {"query_ids": toks, "target_vectors": targets}

    def step():
        opt.zero_grad()
        task.training_step(batch, 0).backward()
        opt.step()
    ms = timed(step, steps, warmup)
    del task, opt
    torch.cuda.empty_cache()

    from transformers import BertConfig, BertModel
    model = BertModel(BertConfig(**BERT_BASE, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1),
                      add_pooling_layer=False).cuda().train()
    sopt = torch.optim.AdamW(model.parameters(), lr=1e-5)
    scaler = torch.amp.GradScaler("cuda")
    mse = torch.nn.MSELoss(reduction="sum")

    def stock():
        sopt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            rep = model(**toks).last_hidden_state[:, 0, :]
        loss = mse(rep.float(), targets)
        scaler.scale(loss).backward()
        scaler.unscale_(sopt)
        torch.nn.utils.clip_grad_norm_(model.parameters(), 2.0)
        scaler.step(sopt)
        scaler.update()
    ms_s = timed(stock, steps, warmup)
    del model, sopt
    torch.cuda.empty_cache()
    emit({"metric": "distill_step", "questions": B, "rows": 2 * B, "S": S, "target_width": 768, "dropout": 0.1,
          "ms_per_step": ms, "questions_per_s": B / (ms * 1e-3), "stock_ms_per_step": ms_s,
          "stock_questions_per_s": B / (ms_s * 1e-3), "speedup": ms_s / ms})
    return ms


def bench_host(emit, step_ms):
    from transformers import BertConfig
    from dpr_scale_b200.datamodule.dpr import DPRDistillJsonlDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    rnd = random.Random(1)
    vocab = open(os.path.join(ROOT, "tests", "golden", "data", "vocab.txt")).read()
    words = vocab.split()[5:]
    with tempfile.TemporaryDirectory() as tmp:
        BertConfig(vocab_size=len(vocab.split())).save_pretrained(tmp)
        with open(os.path.join(tmp, "vocab.txt"), "w") as f:
            f.write(vocab)
        path = os.path.join(tmp, "distill.jsonl")
        nb, B = 8, 128
        with open(path, "w") as f:
            for _ in range(nb * B):
                vec = lambda: [rnd.gauss(0, 1) for _ in range(768)]  # noqa: E731
                f.write(json.dumps({"question": " ".join(rnd.choice(words) for _ in range(12)),
                                    "qry_target_vector": vec(), "ctx_target_vectors": [vec(), vec()]}) + "\n")
        dm = DPRDistillJsonlDataModule(HFTransform(tmp, max_seq_len=32), path, path, path, batch_size=B,
                                       prefetch_batches=0, device_prefetch=False)
        rows = [dm.datasets["train"][i] for i in range(nb * B)]
        dm.collate(rows[:B], "train")
        t0 = time.perf_counter()
        for i in range(nb):
            dm.collate(rows[i * B:(i + 1) * B], "train")
        ms = (time.perf_counter() - t0) * 1e3 / nb
    emit({"metric": "host_batch", "questions": B, "target_width": 768, "positives_per_row": 2,
          "host_ms_per_batch": ms, "gpu_step_ms": step_ms, "host_over_gpu": ms / step_ms if step_ms else None,
          "cpu_cores": os.cpu_count()})


def bench_drboost(emit, steps, warmup):
    from dpr_scale_b200.models.hf_model import HFEncoder
    K, N, S, P = 4, 512, 128, 32
    gen = torch.Generator().manual_seed(2)
    toks = tokens(N, S, gen)
    encs = [HFEncoder.from_config(BERT_BASE, dropout=0.0, projection_dim=P, seed=k).cuda().eval() for k in range(K)]

    @torch.no_grad()
    def ours():
        return torch.cat([e(toks) for e in encs], 1)
    ms = timed(ours, steps, warmup)
    del encs
    torch.cuda.empty_cache()
    from transformers import BertConfig, BertModel
    stock = [(BertModel(BertConfig(**BERT_BASE), add_pooling_layer=False).cuda().eval(),
              torch.nn.Sequential(torch.nn.Linear(768, P), torch.nn.LayerNorm(P)).cuda().eval()) for _ in range(K)]

    @torch.no_grad()
    def hf():
        with torch.autocast("cuda", dtype=torch.float16):
            return torch.cat([pj(m(**toks).last_hidden_state[:, 0, :]).float() for m, pj in stock], 1)
    ms_s = timed(hf, steps, warmup)
    emit({"metric": "drboost_encode", "K": K, "projection_dim": P, "passages": N, "S": S, "ms_per_batch": ms,
          "passages_per_s": N / (ms * 1e-3), "stock_ms_per_batch": ms_s, "stock_passages_per_s": N / (ms_s * 1e-3),
          "speedup": ms_s / ms})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "distill_bench measures on the GPU; there is no CPU path"
    info = card()
    lines = []

    def emit(d):
        d = dict(d, **info)
        lines.append(d)
        print(json.dumps(d), flush=True)
    bench_sqerr(emit)
    step_ms = bench_step(emit, args.steps, args.warmup)
    bench_host(emit, step_ms)
    bench_drboost(emit, args.steps, args.warmup)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
