#!/usr/bin/env python3
"""Cross-encoder reranking of a TREC run: the configured task's test loop (every rank scores its contiguous slice of the
run file and writes ``scores_/qids_/ctx_ids_{rank:04}.pkl`` under ``task.output_dir``), then rank 0 merges the shards
into ``<output_dir>/rerank.trec``, in the line format of run_retrieval.write_run, each query's passages in descending
score order (ties keep their run-file order).

  python -m dpr_scale_b200.rerank task=cross_encoder_rerank task/model=cross_encoder datamodule=cross_encoder_rerank \\
      task.model.model_path=<cross-encoder dir> datamodule.test_path=run.trec \\
      datamodule.test_question_path=queries.tsv datamodule.test_passage_path=psgs.tsv +task.output_dir=<out>

``+run_name=<name>`` sets the run column of rerank.trec (default ``rerank``).
"""
import glob
import os
import pickle
import sys

import torch

from .trainer import Trainer
from .utils.config import compose, instantiate


def load_shards(output_dir, world=None):
    """(qids, ctx_ids, scores as a flat float list) of ranks 0 .. world-1 (default: every scores_*.pkl there),
    concatenated in rank order."""
    qids, ctx_ids, scores = [], [], []
    if world is None:
        world = len(glob.glob(os.path.join(output_dir, "scores_*.pkl")))
    for rank in (f"{r:04}" for r in range(world)):
        with open(os.path.join(output_dir, f"scores_{rank}.pkl"), "rb") as f:
            s = pickle.load(f)
        with open(os.path.join(output_dir, f"qids_{rank}.pkl"), "rb") as f:
            q = pickle.load(f)
        with open(os.path.join(output_dir, f"ctx_ids_{rank}.pkl"), "rb") as f:
            c = pickle.load(f)
        s = torch.as_tensor(s).reshape(-1).tolist()
        assert len(s) == len(q) == len(c), f"shard {rank}: {len(s)} scores, {len(q)} qids, {len(c)} ctx ids"
        qids += q
        ctx_ids += c
        scores += s
    return qids, ctx_ids, scores


def write_rerank_run(path, qids, ctx_ids, scores, run_name="rerank"):
    """Queries in order of first appearance; within a query descending score, ties in input order (stable sort)."""
    rows = {}
    for i, q in enumerate(qids):
        rows.setdefault(q, []).append(i)
    with open(path, "w") as g:
        for q, idx in rows.items():
            for rank, i in enumerate(sorted(idx, key=lambda j: -scores[j]), start=1):
                g.write("{} Q0 {} {} {} {}\n".format(q, ctx_ids[i], rank, float(scores[i]), run_name))
    return path


def merge(output_dir, run_name="rerank", world=None):
    qids, ctx_ids, scores = load_shards(output_dir, world)
    out = write_rerank_run(os.path.join(output_dir, "rerank.trec"), qids, ctx_ids, scores, run_name)
    print(f"Wrote {len(qids)} reranked rows to {out}")
    return out


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    name = "config"
    if "--config-name" in argv:
        i = argv.index("--config-name")
        name = argv[i + 1].replace(".yaml", "")
        del argv[i:i + 2]
    argv = [a for a in argv if a != "-m"]
    from .utils.dist_init import init_process_group
    init_process_group()
    cfg = compose(name, argv)
    if not cfg.task.get("output_dir"):
        raise SystemExit("rerank: give the output directory with +task.output_dir=<dir>")
    run_name = str(cfg.get("run_name", "rerank"))
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    transform = instantiate(cfg.task.transform)
    datamodule = instantiate(cfg.datamodule, transform=transform)
    trainer = Trainer(max_steps=0)
    trainer.test(task, datamodule)                  # test_epoch_end: every rank's pickles are on disk after it
    if trainer.global_rank != 0:
        return None
    return merge(cfg.task.output_dir, run_name, trainer.world_size)


if __name__ == "__main__":
    main()
