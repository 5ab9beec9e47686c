"""DrBoostTask - drop-in for ``dpr_scale.task.drboost_task.DrBoostTask`` (DrBoost, arXiv:2112.07771): K weak DPR
checkpoints served as one ensemble whose query and context embeddings are the concatenation of the weak encoders'
outputs, ``[n, sum d_k]`` in checkpoint order.  Evaluation is DenseRetrieverTask's own loop (``main.py
task=drboost test_only=true``); ``generate_embeddings`` / ``generate_query_embeddings task=drboost`` write the
ensemble's embeddings (``DrBoostGenerateEmbeddingsTask`` / ``DrBoostGenerateQueryEmbeddingsTask``).

Each weak encoder is rebuilt from a checkpoint this repository's ``ModelCheckpoint`` wrote (its ``hyper_parameters``
and ``state_dict``), keeps its own ``shared_model`` and runs on the sm_90a encoder kernels.  Inference only: there is
no optimizer and no TorchScript export.
"""
import os
from typing import List

import torch

from .dpr_eval_task import GenerateEmbeddingsTask, GenerateQueryEmbeddingsTask
from .dpr_task import DenseRetrieverTask


def load_weak_encoders(checkpoint_paths):
    """One DenseRetrieverTask per checkpoint, in order; a missing or unreadable file raises naming its path."""
    if not checkpoint_paths:
        raise ValueError("DrBoostTask needs checkpoint_paths: the weak encoders' checkpoints "
                         "(+task.checkpoint_paths=[a.ckpt,b.ckpt])")
    if isinstance(checkpoint_paths, str):
        checkpoint_paths = [checkpoint_paths]
    weak = torch.nn.ModuleList()
    for idx, path in enumerate(checkpoint_paths):
        if not os.path.isfile(path):
            raise FileNotFoundError(f"weak encoder #{idx}: no checkpoint at {path}")
        try:
            task = DenseRetrieverTask.load_from_checkpoint(path)
        except Exception as e:
            raise RuntimeError(f"weak encoder #{idx}: cannot load the checkpoint {path}: {e}") from e
        weak.append(task)
        print(f"Loaded weak encoder #{idx} state dict from {path} ...")
    return weak


class DrBoostTask(DenseRetrieverTask):
    def __init__(self, checkpoint_paths: List[str] = None, **kwargs):
        super().__init__(**kwargs)
        self.checkpoint_paths = checkpoint_paths

    def setup(self, stage: str):
        if stage == "test" and self.setup_done:
            return
        self.weak_encoders = load_weak_encoders(self.checkpoint_paths)
        self.setup_done = True

    @property
    def query_encoder(self):
        """The first weak encoder's query encoder: where the inherited evaluation step finds the device."""
        return self.weak_encoders[0].query_encoder

    def forward(self, query_ids, contexts_ids):
        return self.encode_queries(query_ids), self.encode_contexts(contexts_ids)

    def configure_optimizers(self):
        pass

    def encode_queries(self, query_ids):
        return torch.cat([self._encode_sequence(query_ids, w.query_encoder) for w in self.weak_encoders], dim=1)

    def encode_contexts(self, contexts_ids):
        return torch.cat([self._encode_sequence(contexts_ids, w.context_encoder) for w in self.weak_encoders], dim=1)


class DrBoostGenerateEmbeddingsTask(GenerateEmbeddingsTask, DrBoostTask):
    """Passage embeddings of the ensemble: ``reps_XXXX.pkl`` of width sum d_k."""


class DrBoostGenerateQueryEmbeddingsTask(GenerateQueryEmbeddingsTask, DrBoostTask):
    """Query embeddings of the ensemble: ``query_reps.pkl`` of width sum d_k."""
