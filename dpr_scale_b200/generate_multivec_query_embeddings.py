#!/usr/bin/env python3
"""COIL / CITADEL query expert dictionaries in the shape of generate_query_embeddings: writes ``query_id.pkl``,
``query_repr.pkl``, ``query_weight.pkl`` (and, with ``add_cls``, ``query_cls.pkl``) to ``task.query_emb_output_dir``,
by default ``task.ctx_embeddings_dir``.

  python -m dpr_scale_b200.generate_multivec_query_embeddings task=generate_multivec_query_embeddings \\
      task/model=citadel_model datamodule=generate_multivec_query_emb datamodule.test_path=queries.tsv \\
      datamodule.trec_format=true task.model.model_path=/path/to/bert +task.ctx_embeddings_dir=/out \\
      +task.checkpoint_path=/path/to.ckpt +task.add_cls=true +task.query_topk=1
"""
import sys

from .generate_embeddings import run

TASK = "dpr_scale_b200.task.citadel_eval_task.GenerateMultiVecQueryEmbeddingsTask"


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
