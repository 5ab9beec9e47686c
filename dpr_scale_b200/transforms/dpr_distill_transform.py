"""Batch assembly for query-encoder distillation - the behaviour of the reference's ``DPRDistillTransform``
(dpr_scale/transforms/dpr_distill_transform.py): JSONL rows ``{"question", "qry_target_vector": [d],
"ctx_target_vectors": [[d], ...]}`` -> every question twice, with one positive-context target vector and then the
question's own target vector.

The positive is drawn with ``random.sample(positives, 1)`` in the train stage (the reference's call, so a seeded run
draws the same rows) and is the first positive otherwise.  Output keys are the reference's: ``query_ids`` (tokeniser
output, 2B rows) and ``target_vectors`` fp32 [2B, d].  Target values are parsed to double by ``json`` and rounded once
to fp32, which is what ``torch.Tensor(list_of_floats)`` does.
"""
import json
import random

import numpy as np
import torch
import torch.nn as nn

from ..utils.config import instantiate
from .hf_transform import HFTransform


class DPRDistillTransform(nn.Module):
    def __init__(self, text_transform, pos_ctx_sample: bool = True, text_column: str = "text"):
        super().__init__()
        self.text_transform = text_transform if isinstance(text_transform, nn.Module) else instantiate(text_transform)
        self.pos_ctx_sample = pos_ctx_sample
        self.text_column = text_column

    def _transform(self, texts):
        if isinstance(self.text_transform, HFTransform):
            return self.text_transform(texts)
        return self.text_transform({"text": texts})["token_ids"]

    def select(self, rows, stage="train"):
        """The parsing and sampling half of forward(): (questions [2B], target vectors fp32 [2B, d] as numpy)."""
        questions, targets = [], []
        for raw in rows:
            row = json.loads(raw)
            pos = row["ctx_target_vectors"]
            assert len(pos) > 0, f"No Positive Contexts in Row '{row['question']}'."
            assert isinstance(pos[0], list), \
                f"Positive Contexts needs to be a list of embeddings in Row '{row['question']}'."
            picked = random.sample(pos, 1)[0] if stage == "train" and self.pos_ctx_sample else pos[0]
            questions.extend([row["question"]] * 2)
            targets.append(picked)
            targets.append(row["qry_target_vector"])
        # one double -> fp32 rounding per value, as torch.Tensor(list_of_floats)
        vectors = np.asarray(targets, dtype=np.float64).astype(np.float32)
        if vectors.ndim != 2:
            raise ValueError(f"target vectors of a batch must all have one width (got an array of shape {vectors.shape})")
        return questions, vectors

    def finish(self, selection, fast=True):
        """The tokenisation half of forward(); ``fast`` goes straight to the Rust tokeniser (HFTransform.encode_fast)."""
        questions, vectors = selection
        enc = self.text_transform.encode_fast if fast and hasattr(self.text_transform, "encode_fast") else self._transform
        return {"query_ids": enc(questions), "target_vectors": torch.from_numpy(vectors)}

    def forward(self, batch, stage="train"):
        rows = batch if type(batch) is list else batch[self.text_column]
        return self.finish(self.select(rows, stage), fast=False)
