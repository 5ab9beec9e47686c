"""RerankDenseRetrieverTask — drop-in for ``dpr_scale.task.dpr_rerank_task.RerankDenseRetrieverTask``: scores every
(query, passage) row of a TREC run with a bi-encoder, score = sum(q_repr * ctx_repr, 1), and writes
``scores_{rank:04}.pkl`` (fp32 CPU tensor ``[n]``), ``qids_{rank:04}.pkl`` and ``ctx_ids_{rank:04}.pkl`` (lists),
pickle protocol 4, in the row order of the rank's shard.  ``python -m dpr_scale_b200.rerank`` merges them into a run
file.

Takes the reference's keywords (``checkpoint_path``, ``output_dir`` and DenseRetrieverTask's).  ``setup`` builds the two
encoders and strictly loads ``checkpoint_path`` (a Lightning checkpoint with a ``state_dict``).  The encoders are any
whose forward returns one fp32 vector per sequence: HFEncoder (the CLS vector, with its optional projection, on the
CLS-pruned forward) or SPLADEEncoder (a vocabulary-sized vector from the fused decoder max-pool).  Each eval step
encodes each distinct query of the batch once; encoding every row instead gives the same scores bit for bit.
"""
import os

import torch

from .dpr_task import DenseRetrieverTask
from .rerank_common import distinct_queries, write_rerank_pickles


class RerankDenseRetrieverTask(DenseRetrieverTask):
    def __init__(self, checkpoint_path, output_dir, **kwargs):
        super().__init__(**kwargs)
        self.checkpoint_path = checkpoint_path
        self.output_dir = output_dir
        self.dedupe_queries = True      # False: encode every row's query (the same scores, bit for bit)
        os.makedirs(output_dir, exist_ok=True)

    def setup(self, stage: str):
        if self.setup_done:
            return
        super().setup("train")
        print(f"Loading checkpoint from {self.checkpoint_path}")
        ckpt = torch.load(self.checkpoint_path, map_location="cpu", weights_only=False)
        self.load_state_dict(ckpt["state_dict"])

    def _scores(self, batch):
        """fp32 [n]: the row-wise dot product of each row's query and passage vectors."""
        q_tok, index = distinct_queries(batch["qid"], batch["query_ids"], self.dedupe_queries)
        with torch.no_grad():
            q = self.query_encoder(q_tok).float()
            c = self.context_encoder(batch["contexts_ids"]).float()
            return (q[index.to(q.device).long()] * c).sum(1)

    def _eval_step(self, batch, batch_idx):
        return [batch["qid"], batch["ctx_id"], self._scores(batch).cpu()]

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, test_outputs):
        return write_rerank_pickles(self.output_dir, self.global_rank, test_outputs)
