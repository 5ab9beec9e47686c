#!/usr/bin/env python3
"""Passage-embedding generation in the shape of /root/reference/dpr_scale/generate_embeddings.py:9-29: the configured
task's ``_target_`` is swapped for GenerateEmbeddingsTask, the passages datamodule is instantiated, and the test loop
writes ``reps_{rank:04}.pkl`` (under torchrun every rank encodes its contiguous slice of the passage file).

  python -m dpr_scale_b200.generate_embeddings datamodule=generate datamodule.test_path=psgs.tsv \\
      task.model.model_path=/path/to/bert +task.ctx_embeddings_dir=/out +task.checkpoint_path=/path/to.ckpt
"""
import os
import sys

import torch
import torch.distributed as dist

from .trainer import Trainer
from .utils.config import compose, instantiate

TASK = "dpr_scale_b200.task.dpr_eval_task.GenerateEmbeddingsTask"
QUERY_TASK = "dpr_scale_b200.task.dpr_eval_task.GenerateQueryEmbeddingsTask"
# ensemble tasks (task=drboost, task=spar): the same dumps over the ensemble's concatenated embeddings
ENSEMBLE_DUMPS = {
    "dpr_scale_b200.task.drboost_task.DrBoostTask": {
        TASK: "dpr_scale_b200.task.drboost_task.DrBoostGenerateEmbeddingsTask",
        QUERY_TASK: "dpr_scale_b200.task.drboost_task.DrBoostGenerateQueryEmbeddingsTask",
    },
    "dpr_scale_b200.task.spar_task.SalientPhraseAwareDenseRetrieverTask": {
        TASK: "dpr_scale_b200.task.spar_task.SparGenerateEmbeddingsTask",
        QUERY_TASK: "dpr_scale_b200.task.spar_task.SparGenerateQueryEmbeddingsTask",
    },
}


def run(argv, target):
    argv = list(argv)
    name = "config"
    if "--config-name" in argv:
        i = argv.index("--config-name")
        name = argv[i + 1].replace(".yaml", "")
        del argv[i:i + 2]
    argv = [a for a in argv if a != "-m"]
    from .utils.dist_init import init_process_group
    init_process_group()
    cfg = compose(name, argv)
    cfg.task.datamodule = None
    cfg.task._target_ = ENSEMBLE_DUMPS.get(cfg.task._target_, {}).get(target, target)
    cfg.task.setdefault("checkpoint_path", None)
    task = instantiate(cfg.task, _recursive_=False)
    transform = instantiate(cfg.task.transform)
    datamodule = instantiate(cfg.datamodule, transform=transform)
    trainer = Trainer(max_steps=0)
    return trainer.test(task, datamodule)      # setup("test") loads the checkpoint; no optimizer is built


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
