"""SalientPhraseAwareDenseRetrieverTask - drop-in for ``dpr_scale.task.spar_task`` (SPAR, arXiv:2110.06918): a dense
DPR model and Λ, a DPR model trained to imitate a lexical retriever, served as one.  Query vectors are
``[q_dense, lexical_weight * q_lex]`` and passage vectors ``[p_dense, p_lex]``, so the inner product is
``q_dense . p_dense + lexical_weight * q_lex . p_lex``; the weight applies to queries only.

SPAR is a two-checkpoint DrBoost ensemble with a weight on the query side: the checkpoints load through
``load_weak_encoders`` and the passage side is DrBoost's concatenation.  The models are kept as ``dense_model`` and
``lexical_model``, so the ``state_dict`` keys are ``dense_model.*`` / ``lexical_model.*`` as in the reference.
Inference only: evaluate with ``main.py task=spar test_only=true``, or write the embeddings with
``generate_embeddings`` / ``generate_query_embeddings task=spar`` (width ``d_dense + d_lex``).
"""
import torch

from .dpr_eval_task import GenerateEmbeddingsTask, GenerateQueryEmbeddingsTask
from .drboost_task import DrBoostTask, load_weak_encoders


class SalientPhraseAwareDenseRetrieverTask(DrBoostTask):
    def __init__(self, pretrained_checkpoint_path: str = "", lexical_model_checkpoint_path: str = "",
                 lexical_weight: float = 0, **kwargs):
        super().__init__(**kwargs)
        self.pretrained_checkpoint_path = pretrained_checkpoint_path
        self.lexical_model_checkpoint_path = lexical_model_checkpoint_path
        self.lexical_weight = lexical_weight

    def setup(self, stage: str):
        if stage == "test" and self.setup_done:
            return
        for key in ("pretrained_checkpoint_path", "lexical_model_checkpoint_path"):
            if not getattr(self, key):
                raise ValueError(f"SPAR needs task.{key}: the {key.split('_')[0]} model's DPR checkpoint")
        self.dense_model, self.lexical_model = load_weak_encoders(
            [self.pretrained_checkpoint_path, self.lexical_model_checkpoint_path])
        self.setup_done = True

    @property
    def weak_encoders(self):
        """DrBoost's view of the pair: the dense model first, so the passage vector is ``[p_dense, p_lex]``."""
        return [self.dense_model, self.lexical_model]

    def encode_queries(self, query_ids):
        dense = self._encode_sequence(query_ids, self.dense_model.query_encoder).float()
        lex = self._encode_sequence(query_ids, self.lexical_model.query_encoder).float()
        return torch.cat([dense, self.lexical_weight * lex], dim=1)


class SparGenerateEmbeddingsTask(GenerateEmbeddingsTask, SalientPhraseAwareDenseRetrieverTask):
    """Passage embeddings ``[p_dense, p_lex]``: ``reps_XXXX.pkl`` of width d_dense + d_lex."""


class SparGenerateQueryEmbeddingsTask(GenerateQueryEmbeddingsTask, SalientPhraseAwareDenseRetrieverTask):
    """Query embeddings ``[q_dense, lexical_weight * q_lex]``: ``query_reps.pkl`` of width d_dense + d_lex."""
