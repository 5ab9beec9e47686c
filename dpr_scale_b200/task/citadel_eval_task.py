"""RerankMultiVecRetrieverTask — drop-in for ``dpr_scale.task.citadel_eval_task.RerankMultiVecRetrieverTask``
(/root/reference/dpr_scale/task/citadel_eval_task.py:215-313) with ColBERT, COIL or CITADEL encoders: scores every
(query, passage) row
of a TREC run by late interaction and writes ``scores_{rank:04}.pkl`` (fp32 CPU tensor ``[n]``), ``qids_{rank:04}.pkl``
and ``ctx_ids_{rank:04}.pkl`` (lists), pickle protocol 4, in the row order of the rank's shard.
``python -m dpr_scale_b200.rerank`` merges them into a run file.

Accepts the keywords of the reference's ``MultiVecRetrieverTask`` (dpr_scale/task/citadel_task.py:8-24) on top of
DenseRetrieverTask's; ``query_pool`` ("sum" or "max"), ``add_cls`` and ``query_topk`` / ``context_topk`` (the experts
per CITADEL token) change what an eval step computes - the others belong to training.  ColBERT ignores the last
three, as in the reference.  ``setup`` builds the two encoders and strictly loads
``checkpoint_path`` (a Lightning checkpoint with a ``state_dict``).

An eval step never materialises ``expert_repr``: each distinct query of the batch is encoded once (rows are encoded
independently at the batch's padded width, so this equals encoding every row), the passages are encoded, both are
projected by the library's GEMM, and ``dprb_maxsim_fwd`` scores the pairs from the unmasked tokens and the masks.
With COIL / CITADEL encoders (those with ``expert_reps``) the encoders also give each token's expert ids and weights
(the mask for COIL, the router's top-k for CITADEL) and, with ``add_cls``, a CLS vector, and
``dprb_maxsim_expert_fwd`` scores the pairs with the expert-matching rule and the CLS term.
"""
import os

import torch

from .. import ops
from .dpr_task import DenseRetrieverTask
from .rerank_common import distinct_queries, write_rerank_pickles


class RerankMultiVecRetrieverTask(DenseRetrieverTask):
    def __init__(self, checkpoint_path, output_dir, add_cls: bool = False, query_topk: int = 1, context_topk: int = 1,
                 query_expert_load_loss_coef: float = 0, context_expert_load_loss_coef: float = 0,
                 query_router_marg_load_loss_coef: float = 0, context_router_marg_load_loss_coef: float = 0,
                 cross_batch: bool = True, in_batch: bool = True, query_pool: str = "sum", anneal_factor: float = 0.0,
                 teacher_coef: float = 0.0, tau: float = 1.0, **kwargs):
        super().__init__(**kwargs)
        self.query_pool = query_pool
        self.add_cls = add_cls
        self.query_topk, self.context_topk = query_topk, context_topk
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
        if self.query_pool not in ops.MAXSIM_POOLS:
            raise NotImplementedError("Invalid query pooling! Available: [max, sum]")
        c_tok = batch["contexts_ids"]
        q_tok, index = distinct_queries(batch["qid"], batch["query_ids"], self.dedupe_queries)
        with torch.no_grad():
            if hasattr(self.query_encoder, "expert_reps"):                       # COIL / CITADEL
                q, q_ids, q_w, q_cls = self.query_encoder.expert_reps(q_tok, topk=self.query_topk, add_cls=self.add_cls)
                d, d_ids, d_w, d_cls = self.context_encoder.expert_reps(c_tok, topk=self.context_topk,
                                                                        add_cls=self.add_cls)
                return ops.maxsim_expert(q, d, q_ids, q_w, d_ids, d_w, index, self.query_pool, q_cls, d_cls)
            q, q_mask = self.query_encoder.token_reps(q_tok)
            d, d_mask = self.context_encoder.token_reps(c_tok)
            return ops.maxsim(q, d, q_mask, d_mask, index, self.query_pool)

    def _eval_step(self, batch, batch_idx):
        return [batch["qid"], batch["ctx_id"], self._scores(batch).cpu()]

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_epoch_end(self, test_outputs):
        return write_rerank_pickles(self.output_dir, self.global_rank, test_outputs)
