#!/usr/bin/env python3
"""Sparse SPLADE passage embeddings in the shape of generate_embeddings: every rank writes ``sparse_{rank:04}.pkl``
(CSR: offsets, terms, fp16 weights, V) for its contiguous slice of the passage table.

  python -m dpr_scale_b200.generate_sparse_embeddings task=generate_sparse_embeddings task/model=splade_model \\
      datamodule=generate datamodule.test_path=psgs.tsv task.model.model_path=/path/to/bert \\
      +task.ctx_embeddings_dir=/out +task.checkpoint_path=/path/to.ckpt
"""
import sys

from .generate_embeddings import run

TASK = "dpr_scale_b200.task.splade_index_task.GenerateSparseEmbeddingsTask"


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
