#!/usr/bin/env python3
"""Query-embedding generation in the shape of /root/reference/dpr_scale/generate_query_embeddings.py:9-31; writes
``<ctx_embeddings_dir>/query_reps.pkl`` (or ``task.query_emb_output_path``), the file run_retrieval reads.

  python -m dpr_scale_b200.generate_query_embeddings datamodule=generate_query_emb datamodule.test_path=queries.tsv \\
      +datamodule.trec_format=true task.model.model_path=/path/to/bert +task.ctx_embeddings_dir=/out \\
      +task.checkpoint_path=/path/to.ckpt
"""
import sys

from .generate_embeddings import QUERY_TASK as TASK, run


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
