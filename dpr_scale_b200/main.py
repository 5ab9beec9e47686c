#!/usr/bin/env python3
"""Entry point in the shape of /root/reference/dpr_scale/main.py:20-50: compose the config, instantiate task /
transform / datamodule by `_target_`, fit, test.  Uses real Hydra/Lightning when importable, else the in-repo
composer (utils/config.py) and mini trainer (trainer.py).

  python -m dpr_scale_b200.main --config-name msmarco_baseline task.model.model_path=/path/to/bert datamodule.train_path=...
"""
import os
import sys

import torch
import torch.distributed as dist

from .trainer import Trainer
from .utils.config import compose, instantiate


def init_distributed():
    """One process per GPU under torchrun: bind the device and join the NCCL group BEFORE the Trainer reads the world
    size (what Lightning's DDP strategy does inside `Trainer.fit`, main.py:32-44 of the reference).  Without it every
    rank would train alone on cuda:0."""
    from .utils.dist_init import init_process_group
    return init_process_group()


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    init_distributed()
    name = "config"
    if "--config-name" in argv:
        i = argv.index("--config-name")
        name = argv[i + 1]
        del argv[i:i + 2]
    cfg = compose(name, argv)
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert cfg.task.model.model_path == cfg.task.transform.model_path
    transform = instantiate(cfg.task.transform)
    datamodule = instantiate(cfg.datamodule, transform=transform)
    tr_kw = {k: v for k, v in cfg.trainer.items() if k in ("max_steps", "max_epochs", "gradient_clip_val", "precision",
                                                             "strategy", "log_every_n_steps", "limit_train_batches",
                                                             "limit_val_batches", "check_val_every_n_epoch")}
    checkpoint_callback = instantiate(cfg.checkpoint_callback) if cfg.get("checkpoint_callback") else None
    trainer = Trainer(callbacks=[checkpoint_callback] if checkpoint_callback is not None else [], **tr_kw)
    if cfg.test_only:
        trainer.test(task, datamodule, ckpt_path=cfg.task.get("pretrained_checkpoint_path"))
    else:
        trainer.fit(task, datamodule)
        if checkpoint_callback is not None:
            print(f"*** Best model path is {checkpoint_callback.best_model_path}")
        trainer.test(task, datamodule, ckpt_path="best")


if __name__ == "__main__":
    main()
