"""RerankCrossEncoderTask — drop-in for ``dpr_scale.task.cross_encoder_eval_task.RerankCrossEncoderTask``
(/root/reference/dpr_scale/task/cross_encoder_eval_task.py): scores every (query, passage) row of a TREC run with the
cross-encoder and writes ``scores_{rank:04}.pkl`` (fp32 CPU tensor: ``[n]``, the max over labels, when the model has
several labels; ``[n, 1]`` with one label), ``qids_{rank:04}.pkl`` and ``ctx_ids_{rank:04}.pkl`` (lists), pickle
protocol 4, in the row order of the rank's shard.  ``python -m dpr_scale_b200.rerank`` merges them into a run file.
"""
import os
import pickle

import torch
import torch.distributed as dist

from .cross_encoder_task import CrossEncoderTask


class RerankCrossEncoderTask(CrossEncoderTask):
    def __init__(self, output_dir, **kwargs):
        super().__init__(**kwargs)
        self.output_dir = output_dir
        os.makedirs(output_dir, exist_ok=True)

    def _eval_step(self, batch, batch_idx):
        token_ids = batch["text_ids"]
        enc = self.cross_encoder
        if hasattr(enc, "logits_and_scores"):
            logits, best = enc.logits_and_scores(token_ids)     # the label max comes from the head kernel
            scores = best if logits.shape[-1] > 1 else logits
        else:
            scores = self(token_ids)
            if len(scores.shape) > 1 and scores.shape[-1] > 1:
                scores = scores.max(1).values
        return [batch["qid"], batch["ctx_id"], scores.cpu()]

    def training_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def _out(self, what):
        return os.path.join(self.output_dir, f"{what}_{self.global_rank:04}.pkl")

    def test_epoch_end(self, test_outputs):
        qids, ctx_ids, scores = [], [], []
        for b_qids, b_ctx_ids, b_scores in test_outputs:
            qids.extend(b_qids)
            ctx_ids.extend(b_ctx_ids)
            scores.append(b_scores)
        if scores:
            scores = torch.cat(scores, dim=0)
        else:                                         # an empty shard: an empty tensor of the model's score shape
            L = getattr(getattr(self, "cross_encoder", None), "num_labels", 1)
            scores = torch.zeros((0, 1) if L == 1 else (0,), dtype=torch.float32)
        out_file = self._out("scores")
        print(f"\nWriting scores to {out_file}")
        for what, obj in (("scores", scores), ("qids", qids), ("ctx_ids", ctx_ids)):
            with open(self._out(what), "wb") as f:
                pickle.dump(obj, f, protocol=4)
        if dist.is_available() and dist.is_initialized():
            dist.barrier()                            # rank 0 merges only once every shard is on disk
        return out_file
