#!/usr/bin/env python3
"""Input-pipeline microbenchmark (CPU side of the training step): seconds per training batch of cfg 2
(128 queries, 1 + 7 contexts each, truncated to 128 tokens) from a synthetic DPR-format JSONL.

  python tools/pipeline_bench.py [rows] [batches]

Prints one JSON line: ms per batch for (a) the synchronous loader tokenising through the HF wrapper call = what the
reference does on the training thread with num_workers 0, (b) the synchronous loader with the direct Rust-tokeniser
path, (c) the BatchStream consumer-side wait while a simulated 88 ms GPU step runs per batch.
"""
import json
import os
import random
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from dpr_scale_b200.datamodule.dpr import DenseRetrieverJsonlDataModule
from dpr_scale_b200.transforms.hf_transform import HFTransform


def synth(tmp, rows, rnd):
    from transformers import BertConfig
    words = ["w%05d" % i for i in range(30000)]
    with open(os.path.join(tmp, "vocab.txt"), "w") as f:
        f.write("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words) + "\n")
    BertConfig(vocab_size=30005).save_pretrained(tmp)
    path = os.path.join(tmp, "train.jsonl")

    def text(n):
        return " ".join(rnd.choice(words) for _ in range(n))
    with open(path, "w") as f:
        for r in range(rows):
            f.write(json.dumps({"question": text(rnd.randint(6, 14)),
                                "positive_ctxs": [{"title": text(3), "text": text(100), "passage_id": str(r)}],
                                "negative_ctxs": [],
                                "hard_negative_ctxs": [{"title": text(3), "text": text(100), "passage_id": str(r * 50 + j)}
                                                       for j in range(30)]}) + "\n")
    return path


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
    nb = int(sys.argv[2]) if len(sys.argv) > 2 else 12
    step_ms = 88.0
    with tempfile.TemporaryDirectory() as tmp:
        path = synth(tmp, rows, random.Random(0))
        tf = HFTransform(model_path=tmp, max_seq_len=128)
        out = {"rows": rows, "batch": "128 q + 1024 ctx, S<=128", "cores": os.cpu_count(),
               "file_MB": round(os.path.getsize(path) / 1e6, 1)}
        for name, prefetch, fast in (("reference_style_sync_ms_per_batch", 0, False), ("sync_ms_per_batch", 0, True),
                                     ("stream_wait_ms_per_batch", 4, True)):
            t0 = time.perf_counter()
            dm = DenseRetrieverJsonlDataModule(transform=tf, train_path=path, val_path=path, test_path=path,
                                               batch_size=128, num_negative=7, prefetch_batches=prefetch,
                                               fast_tokenize=fast, device_prefetch=torch.cuda.is_available())
            out["index_build_ms_per_file"] = round((time.perf_counter() - t0) * 1e3 / 3, 2)
            waited, n = 0.0, 0
            it = iter(dm.train_dataloader())
            for _ in range(5):
                next(it)                                # warm-up (tokeniser thread pool ramp-up, first pinned allocation)
            while n < nb:
                t0 = time.perf_counter()
                try:
                    next(it)
                except StopIteration:
                    break
                waited += time.perf_counter() - t0
                n += 1
                if prefetch:
                    time.sleep(step_ms / 1e3)           # the GPU step the pipeline has to hide behind
            it.close()
            out[name] = round(waited / max(n, 1) * 1e3, 2)
        out["hidden_behind_step_ms"] = step_ms
        print(json.dumps(out))


if __name__ == "__main__":
    main()
