#!/usr/bin/env python3
"""COIL / CITADEL expert-index generation in the shape of generate_embeddings: the configured task's ``_target_`` is
swapped for GenerateMultiVecEmbeddingsTask and every rank writes ``expert_{rank:04}/{expert}.pkl`` (and, with
``add_cls``, ``cls_{rank:04}.pkl``) for its contiguous slice of the passage table.

  python -m dpr_scale_b200.generate_multivec_embeddings task=generate_multivec_embeddings task/model=citadel_model \\
      datamodule=generate datamodule.test_path=psgs.tsv task.model.model_path=/path/to/bert \\
      +task.ctx_embeddings_dir=/out +task.checkpoint_path=/path/to.ckpt +task.add_cls=true +task.context_topk=1
"""
import sys

from .generate_embeddings import run

TASK = "dpr_scale_b200.task.citadel_eval_task.GenerateMultiVecEmbeddingsTask"


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
