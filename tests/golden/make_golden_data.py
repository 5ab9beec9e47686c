#!/usr/bin/env python3
"""Golden batches for the input pipeline: runs the UNMODIFIED reference data code
(/root/reference/dpr_scale/datamodule/dpr.py DenseRetrieverJsonlDataModule, transforms/dpr_transform.py DPRTransform,
transforms/hf_transform.py HFTransform, utils/utils.py ContiguousDistributedSampler) on a synthetic DPR-format JSONL
written by this script, and stores every batch it produces.

  python tests/golden/make_golden_data.py     # writes tests/golden/data/{synth.jsonl,vocab.txt} and data_batches.npz

hydra / pytorch_lightning / ujson are not installed: the reference modules are imported through stub modules
(hydra.utils.instantiate, pytorch_lightning.LightningDataModule, ujson := json).
"""
import json
import os
import random
import sys
import types

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "data")
WORDS = ["alpha", "bravo", "charlie", "delta", "echo", "foxtrot", "golf", "hotel", "india", "juliet", "kilo", "lima",
         "mike", "november", "oscar", "papa", "quebec", "romeo", "sierra", "tango", "uniform", "victor", "whiskey",
         "xray", "yankee", "zulu", "?", ".", ","]


def write_inputs():
    os.makedirs(DATA, exist_ok=True)
    with open(os.path.join(DATA, "vocab.txt"), "w") as f:
        f.write("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS) + "\n")
    rnd = random.Random(7)

    def text(lo, hi):
        return " ".join(rnd.choice(WORDS) for _ in range(rnd.randint(lo, hi)))

    def ctx(i, **extra):
        d = {"title": text(1, 3), "text": text(3, 30), "passage_id": str(i)}
        d.update(extra)
        return d

    rows = []
    for r in range(13):
        n_neg = [9, 0, 1, 12, 3, 7, 2, 20, 5, 8, 1, 4, 6][r]
        row = {"question": text(2, 12),
               "positive_ctxs": [ctx(1000 + r * 3 + j, score=str(50 + j), relevance=1 + j) for j in range(1 + r % 3)],
               "negative_ctxs": [],
               "hard_negative_ctxs": [ctx(r * 100 + j, score=round(rnd.random() * 10, 3), relevance=rnd.randint(1, 5))
                                      for j in range(n_neg)]}
        if r == 4:     # token-list text (dpr_transform.py:94-99)
            row["positive_ctxs"][0]["text"] = row["positive_ctxs"][0]["text"].split(" ")
        if r == 6:     # no score fields
            for c in row["positive_ctxs"] + row["hard_negative_ctxs"]:
                c.pop("score", None)
        rows.append(row)
    # DPR retriever-output format (dpr_transform.py:78-88), with and without an answer-bearing context
    rows.append({"question": text(3, 6), "ctxs": [dict(ctx(9000 + j), has_answer=(j == 2)) for j in range(6)]})
    rows.append({"question": text(3, 6), "ctxs": [dict(ctx(9100 + j), has_answer=False) for j in range(4)]})
    with open(os.path.join(DATA, "synth.jsonl"), "w") as f:
        for row in rows[:-1]:
            f.write(json.dumps(row) + "\n")
        f.write(json.dumps(rows[-1]))            # last line without newline
    # passage table (generate_embeddings input) with csv quoting and one malformed row, question files (both formats)
    with open(os.path.join(DATA, "passages.tsv"), "w") as f:
        f.write("id\ttext\ttitle\n")
        for i in range(11):
            t = text(3, 30)
            if i == 3:
                t = '"' + t + ' ""quoted"" tail"'
            f.write(f"{i + 1}\t{t}\t{text(1, 3)}\n")
    # DRAGON-style inputs: corpus table + two light training files that reference it by docidx
    with open(os.path.join(DATA, "corpus.tsv"), "w") as f:
        f.write("id\ttext\ttitle\n")
        for i in range(40):
            f.write(f"d{i}\t{text(3, 20)}\t{text(1, 3)}\n")
    for name, nrows in (("light_a.jsonl", 9), ("light_b.jsonl", 7)):
        with open(os.path.join(DATA, name), "w") as f:
            for r in range(nrows):
                f.write(json.dumps({"query_id": str(r), "question": text(2, 10),
                                    "positive_ctxs": [{"docidx": rnd.randrange(40), "score": str(rnd.random())}
                                                      for _ in range(1 + r % 2)],
                                    "hard_negative_ctxs": [{"docidx": rnd.randrange(40)} for _ in range(r % 4)]}) + "\n")
    with open(os.path.join(DATA, "malformed.tsv"), "w") as f:
        f.write("id\ttext\ttitle\n1\tfine text\tfine title\nbroken row without tabs\n")
    with open(os.path.join(DATA, "questions.csv"), "w") as f:
        for i in range(7):
            f.write(f"{text(2, 9)}\t{[text(1, 2), text(1, 1)]!r}\n")
    with open(os.path.join(DATA, "questions.tsv"), "w") as f:
        for i in range(7):
            f.write(f"q{i}\t{text(2, 9)}\n")
    return len(rows)


def install_stubs():
    sys.modules["ujson"] = json
    hydra = types.ModuleType("hydra")
    hu = types.ModuleType("hydra.utils")
    hu.instantiate = lambda conf, *a, **k: (_ for _ in ()).throw(RuntimeError("not used"))
    hydra.utils = hu
    sys.modules["hydra"], sys.modules["hydra.utils"] = hydra, hu
    pl = types.ModuleType("pytorch_lightning")

    class LightningDataModule:
        def __init__(self):
            self.trainer = None
    pl.LightningDataModule = LightningDataModule
    sys.modules["pytorch_lightning"] = pl
    sys.path.insert(0, REF)


def model_dir(tmp):
    from transformers import BertConfig
    os.makedirs(tmp, exist_ok=True)
    BertConfig(vocab_size=5 + len(WORDS), hidden_size=16, num_hidden_layers=1, num_attention_heads=1,
               intermediate_size=16).save_pretrained(tmp)
    with open(os.path.join(DATA, "vocab.txt")) as s, open(os.path.join(tmp, "vocab.txt"), "w") as d:
        d.write(s.read())
    return tmp


def dump(out, prefix, batch):
    for key in ("query_ids", "contexts_ids"):
        for kk in batch[key].keys():
            out[f"{prefix}/{key}/{kk}"] = batch[key][kk].numpy()
    for key in ("pos_ctx_indices", "scores", "ctx_mask"):
        out[f"{prefix}/{key}"] = batch[key].numpy()


def main():
    n_rows = write_inputs()
    install_stubs()
    import tempfile
    from dpr_scale.datamodule.dpr import DenseRetrieverJsonlDataModule, MemoryMappedDataset
    from dpr_scale.transforms.hf_transform import HFTransform
    from dpr_scale.utils.utils import ContiguousDistributedSampler
    path = os.path.join(DATA, "synth.jsonl")
    out = {"n_rows": n_rows}
    with tempfile.TemporaryDirectory() as tmp:
        tf = HFTransform(model_path=model_dir(tmp), max_seq_len=24)
        cases = {
            "a": dict(batch_size=4, num_negative=3, neg_ctx_sample=True, pos_ctx_sample=False, num_val_negative=2,
                      num_test_negative=5, use_title=True),
            "b": dict(batch_size=5, num_negative=7, neg_ctx_sample=True, pos_ctx_sample=True, num_val_negative=7,
                      num_test_negative=0, use_title=False, rel_sample=True),
            "c": dict(batch_size=15, num_negative=0, neg_ctx_sample=False, num_val_negative=1, use_title=False),
        }
        for name, kw in cases.items():
            dm = DenseRetrieverJsonlDataModule(transform=tf, train_path=path, val_path=path, test_path=path, **kw)
            np.random.seed(1234)
            for stage, loader in (("train", dm.train_dataloader()), ("valid", dm.val_dataloader()),
                                  ("test", dm.test_dataloader())):
                nb = 0
                for i, batch in enumerate(loader):
                    dump(out, f"{name}/{stage}/{i}", batch)
                    nb += 1
                out[f"{name}/{stage}/num_batches"] = nb
        from dpr_scale.datamodule.dpr import (CSVDataset, DenseRetrieverPassagesDataModule,
                                              DenseRetrieverQueriesDataModule)
        from dpr_scale.utils.utils import ContiguousDistributedSamplerForTest
        pdm = {"t": DenseRetrieverPassagesDataModule(tf, os.path.join(DATA, "passages.tsv"), test_batch_size=5, use_title=True),
               "n": DenseRetrieverPassagesDataModule(tf, os.path.join(DATA, "passages.tsv"), test_batch_size=12)}
        for name, dm in pdm.items():
            for i, batch in enumerate(dm.test_dataloader()):
                for kk in batch["contexts_ids"].keys():
                    out[f"passages/{name}/{i}/{kk}"] = batch["contexts_ids"][kk].numpy()
                out[f"passages/{name}/{i}/corpus_ids"] = np.array(batch["corpus_ids"])
            out[f"passages/{name}/num_batches"] = i + 1
        for name, fn, trec in (("csv", "questions.csv", False), ("tsv", "questions.tsv", True)):
            dm = DenseRetrieverQueriesDataModule(tf, os.path.join(DATA, fn), test_batch_size=3, trec_format=trec)
            for i, batch in enumerate(dm.test_dataloader()):
                for kk in batch["query_ids"].keys():
                    out[f"queries/{name}/{i}/{kk}"] = batch["query_ids"][kk].numpy()
            out[f"queries/{name}/num_batches"] = i + 1
        csv = CSVDataset(os.path.join(DATA, "passages.tsv"))
        out["csv_len"] = len(csv)
        out["csv_row3_text"] = np.array(csv[3]["text"])
        bad = CSVDataset(os.path.join(DATA, "malformed.tsv"))
        out["csv_malformed_is_none"] = np.array(bad[1] is None)      # dpr.py:102-107 evaluates row 0 and returns None
        for world in (2, 3, 8):
            for rank in range(world):
                smp = ContiguousDistributedSamplerForTest(csv, num_replicas=world, rank=rank)
                out[f"test_sampler/{world}/{rank}"] = np.array(list(iter(smp)), dtype=np.int64)
        from dpr_scale.datamodule.dpr import DenseRetrieverMultiJsonlDataModule
        la, lb = os.path.join(DATA, "light_a.jsonl"), os.path.join(DATA, "light_b.jsonl")
        mdm = DenseRetrieverMultiJsonlDataModule(transform=tf, train_path=[la, lb], val_path=la, test_path=lb,
                                                 corpus_path=os.path.join(DATA, "corpus.tsv"), batch_size=3, num_negative=2,
                                                 pos_ctx_sample=True, num_val_negative=1, num_test_negative=3, use_title=True)
        random.seed(5)
        np.random.seed(99)
        for stage, loader in (("train", mdm.train_dataloader()), ("valid", mdm.val_dataloader()),
                              ("test", mdm.test_dataloader())):
            nb = 0
            for i, batch in enumerate(loader):
                dump(out, f"multi/{stage}/{i}", batch)
                nb += 1
            out[f"multi/{stage}/num_batches"] = nb
        ds = MemoryMappedDataset(path)
        out["lines"] = np.array([len(ds[i]) for i in range(len(ds))])
        # sampler orders: (world, rank, replicas_per_node, epoch)
        for world, per_node in ((2, 2), (4, 2), (8, 8), (3, 1)):
            for epoch in (0, 3):
                for rank in range(world):
                    s = ContiguousDistributedSampler(ds, num_replicas=world, rank=rank, num_replicas_per_node=per_node)
                    s.set_epoch(epoch)
                    out[f"sampler/{world}/{per_node}/{epoch}/{rank}"] = np.array(list(iter(s)))
    np.savez_compressed(os.path.join(HERE, "data_batches.npz"), **out)
    print("wrote data_batches.npz with", len(out), "arrays;", n_rows, "rows")


if __name__ == "__main__":
    main()
