"""Batch assembly for bi-encoder training - the behaviour of the reference's ``DPRTransform``
(/root/reference/dpr_scale/transforms/dpr_transform.py:20-187): JSONL rows -> questions, 1 positive + n hard
negatives per question (sampled in the train stage, truncated otherwise), dummy contexts + ``ctx_mask`` when a row has
too few negatives, optional ``title sep text`` concatenation, tokenisation of questions and contexts.

The random draws go through ``np.random.choice`` with the same arguments in the same order as the reference, so a
seeded run selects the same contexts.  Output dict keys and dtypes are the reference's:
``query_ids``, ``contexts_ids`` (tokeniser outputs), ``pos_ctx_indices`` int64 [B], ``scores`` fp32 [B, 1+n],
``ctx_mask`` bool [B*(1+n)] (True = dummy context).
"""
import json

import numpy as np
import torch
import torch.nn as nn

from ..utils.config import instantiate
from .hf_transform import HFTransform


def maybe_add_title(text, title, use_title, sep_token):
    """utils/utils.py:24-28."""
    return " ".join([title, sep_token, text]) if use_title else text


def _normalise_row(row):
    """DPR retriever-output rows ({"ctxs": [{has_answer}]}) -> positive_ctxs / hard_negative_ctxs (:78-88)."""
    if "positive_ctxs" not in row and "ctxs" in row:
        row["positive_ctxs"] = [c for c in row["ctxs"] if c["has_answer"]]
        row["hard_negative_ctxs"] = [c for c in row["ctxs"] if not c["has_answer"]]
        if not row["positive_ctxs"]:
            row["positive_ctxs"].append(row["ctxs"][0])
    return row


def _draw(ctxs, count, rel_sample):
    """``count`` contexts without replacement, probability proportional to ``relevance`` when rel_sample (:100-109)."""
    rel = [c.get("relevance", 1.0) if rel_sample else 1.0 for c in ctxs]
    total = sum(rel)
    proba = [float(r) / total for r in rel]
    picked = np.random.choice(len(ctxs), count, replace=False, p=proba)
    return [ctxs[int(j)] for j in picked]


class DPRTransform(nn.Module):
    def __init__(self, text_transform, num_positive: int = 1, num_negative: int = 7, neg_ctx_sample: bool = True,
                 pos_ctx_sample: bool = False, num_val_negative: int = 7, num_test_negative=None,
                 use_title: bool = False, sep_token: str = " ", rel_sample: bool = False, corpus=None,
                 text_column: str = "text"):
        super().__init__()
        if num_positive > 1:
            raise ValueError("Only 1 positive example is supported. Update the loss to support more!")
        self.text_transform = text_transform if isinstance(text_transform, nn.Module) else instantiate(text_transform)
        self.num_positive = num_positive
        self.num_negative = num_negative
        self.neg_ctx_sample = neg_ctx_sample
        self.pos_ctx_sample = pos_ctx_sample
        self.num_val_negative = num_val_negative
        self.num_test_negative = num_test_negative if num_test_negative else self.num_val_negative
        self.use_title = use_title
        self.sep_token = sep_token
        if isinstance(self.text_transform, HFTransform):
            self.sep_token = self.text_transform.sep_token
        self.text_column = text_column
        self.rel_sample = rel_sample
        self.corpus = corpus

    def _transform(self, texts):
        if isinstance(self.text_transform, HFTransform):
            return self.text_transform(texts)
        return self.text_transform({"text": texts})["token_ids"]

    def _negatives_wanted(self, stage):
        return {"train": self.num_negative, "eval": self.num_val_negative, "test": self.num_test_negative}[stage]

    def select(self, rows, stage="train"):
        """The sampling half of forward(): (questions, context texts, positive indices, ctx_mask, scores)."""
        questions, ctx_text, positive_idx, ctx_mask, scores = [], [], [], [], []
        want = self._negatives_wanted(stage)
        for raw in rows:
            row = _normalise_row(json.loads(raw))
            pos = row["positive_ctxs"]
            if pos and self.corpus is None and not isinstance(pos[0]["text"], str):
                for c in pos:                       # text given as a token list
                    c["text"] = " ".join(c["text"])
            if stage == "train" and self.pos_ctx_sample:
                pos = _draw(pos, self.num_positive, self.rel_sample)
            else:
                pos = pos[: self.num_positive]
            neg = row["hard_negative_ctxs"]
            if want > 0:
                if stage == "train" and self.neg_ctx_sample and len(neg) > want:
                    neg = _draw(neg, want, self.rel_sample)
                else:
                    neg = neg[:want]
            else:
                neg = []
            ctxs = pos + neg
            mask = [0] * len(ctxs)
            missing = want - len(neg)
            if missing > 0:                          # pad with dummy contexts, masked out of the loss
                dummy = {"text": "0", "title": "0", "score": 0} if self.corpus is None else {"docidx": "0", "score": 0}
                ctxs = ctxs + [dummy] * missing
                mask += [1] * missing
            assert len(ctxs) == self.num_positive + want, f"Row has improper ctx count. Check positive ctxs in: {row}"
            scores.append([float(c["score"]) if "score" in c else 0 for c in ctxs])
            positive_idx.append(len(ctx_text))
            for c in ctxs:
                if self.corpus is None:
                    ctx_text.append(maybe_add_title(c["text"], c["title"], self.use_title, self.sep_token))
                else:
                    _, text, title = self.corpus[int(c["docidx"])].decode("UTF-8").strip().split("\t")
                    ctx_text.append(maybe_add_title(text, title, self.use_title, self.sep_token))
            questions.append(row["question"])
            ctx_mask.extend(mask)
        return questions, ctx_text, positive_idx, ctx_mask, scores

    def finish(self, selection, fast=True):
        """The tokenisation half of forward(); ``fast`` goes straight to the Rust tokeniser (HFTransform.encode_fast)."""
        questions, ctx_text, positive_idx, ctx_mask, scores = selection
        enc = self.text_transform.encode_fast if fast and hasattr(self.text_transform, "encode_fast") else self._transform
        return {
            "query_ids": enc(questions),
            "contexts_ids": enc(ctx_text),
            "pos_ctx_indices": torch.tensor(positive_idx, dtype=torch.long),
            "scores": torch.tensor(scores, dtype=torch.float32),
            "ctx_mask": torch.tensor(ctx_mask, dtype=torch.bool),
        }

    def forward(self, batch, stage="train"):
        rows = batch if type(batch) is list else batch[self.text_column]
        questions, ctx_text, positive_idx, ctx_mask, scores = self.select(rows, stage)
        return {
            "query_ids": self._transform(questions),
            "contexts_ids": self._transform(ctx_text),
            "pos_ctx_indices": torch.tensor(positive_idx, dtype=torch.long),
            "scores": torch.tensor(scores, dtype=torch.float32),
            "ctx_mask": torch.tensor(ctx_mask, dtype=torch.bool),
        }


class DPRCrossAttentionTransform(DPRTransform):
    """Cross-encoder training groups - the sampling of the reference's ``DPRCrossAttentionTransform``
    (/root/reference/dpr_scale/transforms/dpr_transform.py:190-326): per question, its positive and then its hard
    negatives (sampled in the train stage, truncated otherwise), and, when a row has fewer negatives than wanted, a fill
    drawn without replacement from every positive and hard negative of the batch (``num_random_negs`` more in the train
    stage).  The pair at position 0 of each group is the relevant one.  ``np.random`` is drawn with the reference's
    arguments in the reference's order.

    Where this departs from the reference:
      * each (question, passage) goes through ``text_transform(questions, passages)``, the pair encoding the rerank
        datamodule uses, so the model trains on exactly what it reranks.  The reference hands its tokenizer a
        ``{"text", "label"}`` dict of ``" ".join([question, sep_token, passage])`` strings, which neither of its
        transforms accepts;
      * with ``pos_ctx_sample`` the sampled positives form the group; the reference draws them and then keeps every
        positive, which gives groups of unequal size;
      * rows in the DPR retriever-output format (``ctxs`` + ``has_answer``) are normalised before the batch fill is
        collected, and a passage given as a token list is joined wherever it is used; the reference reads
        ``positive_ctxs`` of every row first and joins the token lists of a row's own positives only, so it fails on
        both.

    The batch is ``{"text_ids": tokens [B*G, S], "labels": int64 [B] (zeros), "group_size": G}``."""

    def __init__(self, text_transform, num_positive: int = 1, num_negative: int = 7, neg_ctx_sample: bool = True,
                 pos_ctx_sample: bool = False, num_val_negative: int = 7, num_test_negative=None,
                 use_title: bool = False, sep_token: str = " ", rel_sample: bool = False, corpus=None,
                 text_column: str = "text", num_random_negs: int = 0):
        super().__init__(text_transform, num_positive, num_negative, neg_ctx_sample, pos_ctx_sample, num_val_negative,
                         num_test_negative, use_title, sep_token, rel_sample, corpus, text_column)
        self.num_random_negs = num_random_negs

    def _text(self, ctx):
        if self.corpus is not None:
            return self.corpus[int(ctx["docidx"])].decode("UTF-8").strip().split("\t")[1]
        text = ctx["text"]
        return text if isinstance(text, str) else " ".join(text)     # text given as a token list

    def select(self, rows, stage="train"):
        """The sampling half of forward(): (questions, passages), one entry per pair, group by group."""
        rows = [_normalise_row(json.loads(raw)) for raw in rows]
        candidates = [c for row in rows for c in row["positive_ctxs"] + row["hard_negative_ctxs"]]
        want = self._negatives_wanted(stage)
        extra = self.num_random_negs if stage == "train" else 0
        questions, passages = [], []
        for row in rows:
            pos = row["positive_ctxs"]
            if stage == "train" and self.pos_ctx_sample:
                pos = _draw(pos, self.num_positive, self.rel_sample)
            else:
                pos = pos[: self.num_positive]
            neg = row["hard_negative_ctxs"]
            if want > 0:
                if stage == "train" and self.neg_ctx_sample and len(neg) > want:
                    neg = _draw(neg, want, self.rel_sample)
                else:
                    neg = neg[:want]
            else:
                neg = []
            ctxs = pos + neg
            if len(neg) < want + extra:
                picked = np.random.choice(len(candidates), want + extra - len(neg), replace=False)
                ctxs += [candidates[int(j)] for j in picked]
            questions += [row["question"]] * len(ctxs)
            passages += [self._text(c) for c in ctxs]
        return questions, passages, len(rows)

    def finish(self, selection, fast=True):
        """The tokenisation half of forward(): one pair encoding of every (question, passage)."""
        questions, passages, B = selection
        if B == 0 or len(passages) % B:
            raise ValueError(f"{len(passages)} pairs do not form {B} equal groups")
        return {"text_ids": self.text_transform(questions, passages),
                "labels": torch.zeros(B, dtype=torch.long),
                "group_size": len(passages) // B}

    def forward(self, batch, stage="train"):
        rows = batch if type(batch) is list else batch[self.text_column]
        return self.finish(self.select(rows, stage))
