#!/usr/bin/env python3
"""Sparse SPLADE query embeddings in the shape of generate_query_embeddings: writes ``sparse_query.pkl`` (CSR with fp32
weights, and the topic ids with ``datamodule.trec_format=true``) to ``task.query_emb_output_path``, by default
``<task.ctx_embeddings_dir>/sparse_query.pkl``.

  python -m dpr_scale_b200.generate_sparse_query_embeddings task=generate_sparse_query_embeddings \\
      task/model=splade_model datamodule=generate_multivec_query_emb datamodule.test_path=queries.tsv \\
      datamodule.trec_format=true task.model.model_path=/path/to/bert +task.ctx_embeddings_dir=/out \\
      +task.checkpoint_path=/path/to.ckpt
"""
import sys

from .generate_embeddings import run

TASK = "dpr_scale_b200.task.splade_index_task.GenerateSparseQueryEmbeddingsTask"


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
