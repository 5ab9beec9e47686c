#!/usr/bin/env python3
"""COIL / CITADEL retrieval from an expert index in the shape of generate_embeddings: the configured task's
``_target_`` is swapped for CITADELRetrievalTask; every rank loads the whole index, searches its contiguous slice of
the queries and writes ``output_path/retrieval_{rank:04}.trec`` (or ``.json`` for question / answers files).

  python -m dpr_scale_b200.multivec_retrieval task=multivec_retrieval task/model=citadel_model \\
      datamodule=generate_multivec_query_emb datamodule.test_path=queries.tsv datamodule.trec_format=true \\
      task.model.model_path=/path/to/bert +task.ctx_embeddings_dir=/index +task.checkpoint_path=/path/to.ckpt \\
      +task.passages=psgs.tsv +task.output_path=/out +task.topk=100 +task.add_cls=true +task.query_topk=1
"""
import sys

from .generate_embeddings import run

TASK = "dpr_scale_b200.task.citadel_retrieval_task.CITADELRetrievalTask"


def main(argv=None):
    return run(sys.argv[1:] if argv is None else argv, TASK)


if __name__ == "__main__":
    main()
