#!/usr/bin/env python3
"""Golden cross-encoder training groups: runs the UNMODIFIED reference ``DPRCrossAttentionTransform``
(/root/reference/dpr_scale/transforms/dpr_transform.py:190-326) on the fixture JSONL files with seeded ``np.random`` and
a recording text transform that returns the dict it is given, and stores the strings it would tokenise
(``" ".join([question, sep_token, passage])``) and its labels.  Only this data is committed.

  python tests/golden/make_golden_cross_train.py     # writes tests/golden/cross_train_groups.npz

The cases (CASES) are shared with tests/test_cross_encoder_train_cpu.py, which replays them through this repository's
transform.  Rows 4 (positives given as token lists), 13 and 14 (the DPR retriever-output format) are left out: the reference
fails on them (its batch fill keeps the token lists, and it reads ``positive_ctxs`` of every row before normalising).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "data")

# name -> (file, rows, batch size, stage, seed, transform keywords)
ROWS = [0, 1, 2, 3, 5, 6, 7, 8, 9, 10, 11, 12]
CASES = {
    "train": ("synth.jsonl", ROWS, 4, "train", 11, dict(num_negative=3, neg_ctx_sample=True)),
    "train_truncate": ("synth.jsonl", ROWS, 3, "train", 15, dict(num_negative=2, neg_ctx_sample=False)),
    "eval": ("synth.jsonl", ROWS, 4, "eval", 12, dict(num_val_negative=4)),
    "test": ("synth.jsonl", ROWS, 5, "test", 13, dict(num_val_negative=4, num_test_negative=2)),
    "train_pos_sample": ("synth.jsonl", [0, 3, 6, 9, 12], 5, "train", 14,
                         dict(num_negative=5, pos_ctx_sample=True, rel_sample=True, num_random_negs=1)),
}


def batches(case):
    path, rows, bs, stage, seed, kw = CASES[case]
    lines = open(os.path.join(DATA, path), "rb").read().splitlines(keepends=True)
    picked = [lines[i] for i in rows]
    return [picked[lo:lo + bs] for lo in range(0, len(picked), bs)], stage, seed, kw


def main():
    sys.path.insert(0, HERE)
    from make_golden_data import install_stubs
    install_stubs()
    import torch.nn as nn
    from dpr_scale.transforms.dpr_transform import DPRCrossAttentionTransform

    class Recorder(nn.Module):
        def forward(self, d):
            return d

    out = {}
    for case in CASES:
        chunks, stage, seed, kw = batches(case)
        tf = DPRCrossAttentionTransform(Recorder(), **kw)
        np.random.seed(seed)
        texts, labels, sizes = [], [], []
        for chunk in chunks:
            d = tf([line.decode() for line in chunk], stage)
            texts += d["text"]
            labels += d["label"]
            sizes.append(len(d["text"]) // len(d["label"]))
        out[f"{case}/text"] = np.array(texts)
        out[f"{case}/label"] = np.array([int(x) for x in labels], dtype=np.int64)
        out[f"{case}/group_size"] = np.array(sizes, dtype=np.int64)
    np.savez(os.path.join(HERE, "cross_train_groups.npz"), **out)
    print(json.dumps({k: list(v.shape) for k, v in out.items()}))


if __name__ == "__main__":
    main()
