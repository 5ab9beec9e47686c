"""Sparse SPLADE embeddings for first-stage retrieval: ``GenerateSparseEmbeddingsTask`` (passages ->
``sparse_{rank:04}.pkl``) and ``GenerateSparseQueryEmbeddingsTask`` (questions -> ``sparse_query.pkl``), the inputs of
``python -m dpr_scale_b200.splade_retrieval``.

A SPLADE vector is vocabulary-wide ([N, V] fp32, 122 KB per passage at V = 30522) but mostly zero, so only each row's
nonzeros are kept, as one CSR matrix per file (utils/csr_writer.py): offsets int64 [N + 1], terms int32 [nnz], weights
fp16 (passages) or fp32 (queries) [nnz], V, and the queries' topic ids when the batches carry them (trec_format).

Each step runs SPLADEEncoder under no_grad, extracts the nonzeros of the pooled [B, V] block with ``torch.nonzero``
and copies them into a pinned ring slot without waiting; the slot that is due is appended to the file's spools, as
GenerateEmbeddingsTask does with dense rows.  A weight that does not fit fp16 raises ValueError, as does an
encoder that is not a SPLADEEncoder.
"""
import collections
import os
import pathlib

import numpy as np
import torch
import torch.distributed as dist

from .. import ops
from ..models.citadel_models.splade_model import SPLADEEncoder
from ..utils.csr_writer import StreamingCSRPickle
from .dpr_eval_task import _EmbeddingDumpTask


class GenerateSparseEmbeddingsTask(_EmbeddingDumpTask):
    """Passage side: the context encoder over ``batch["contexts_ids"]``; every rank writes ``sparse_{rank:04}.pkl`` for
    its contiguous slice of the passage table (rows in table order)."""

    batch_key = "contexts_ids"
    weight_dtype = torch.float16

    def _encoder(self):
        return self.context_encoder

    def _out_path(self):
        if not self.ctx_embeddings_dir:
            self.ctx_embeddings_dir = getattr(self.trainer, "weights_save_path", ".")
        return os.path.join(self.ctx_embeddings_dir, f"sparse_{self.global_rank:04}.pkl")

    def _encode(self, tokens):
        enc = self._encoder()
        if not isinstance(enc, SPLADEEncoder):
            raise ValueError(f"sparse embedding generation needs a SPLADEEncoder (got {type(enc).__name__}): use "
                             "task/model=splade_model")
        return enc(tokens)

    def _ring_slot(self, nnz, rows):
        """(counts int64 [rows], terms int32 [nnz], weights [nnz]) views of a pinned ring slot."""
        if len(self._ring) < self.RING:
            self._ring.append(None)
        i = self._next % self.RING
        self._next += 1
        slot = self._ring[i]
        pin = torch.cuda.is_available()
        if slot is None or slot[0].numel() < rows or slot[1].numel() < nnz:
            slot = (torch.empty(max(rows, 1), dtype=torch.int64, pin_memory=pin),
                    torch.empty(max(nnz, 1), dtype=torch.int32, pin_memory=pin),
                    torch.empty(max(nnz, 1), dtype=self.weight_dtype, pin_memory=pin))
            self._ring[i] = slot
        return slot[0][:rows], slot[1][:nnz], slot[2][:nnz]

    def _write_due(self, keep):
        while len(self._inflight) > keep:
            (counts, terms, weights), ev = self._inflight.popleft()
            if ev is not None:
                ev.synchronize()
            self._writer.append(counts.numpy(), terms.numpy(), weights.numpy())

    @torch.no_grad()
    def _eval_step(self, batch, batch_idx):
        rep = self(batch[self.batch_key])
        B, V = rep.shape
        nz = torch.nonzero(rep)                                  # row-major: terms ascend inside a row
        rows, terms = nz[:, 0], nz[:, 1]
        w = rep[rows, terms]
        if w.numel() and not (float(w.abs().max()) <= ops.FP16_MAX):          # NaN fails too
            raise ValueError(f"a SPLADE weight does not fit fp16 (|w| > {ops.FP16_MAX:g} or not finite): the sparse "
                             "index stores fp16 passage weights")
        counts = torch.bincount(rows, minlength=B)
        self._ring_init()
        self._write_due(self.RING - 1)
        if self._writer is None:
            out = self._out_path()
            pathlib.Path(out).parent.mkdir(parents=True, exist_ok=True)
            self._writer = StreamingCSRPickle(out, V, np.float16 if self.weight_dtype == torch.float16 else np.float32)
        slot = self._ring_slot(terms.numel(), B)
        for dst, src in zip(slot, (counts, terms.to(torch.int32), w.to(self.weight_dtype))):
            dst.copy_(src, non_blocking=True)
        ev = None
        if rep.is_cuda:
            ev = torch.cuda.Event()
            ev.record()
        self._inflight.append((slot, ev))
        self._after_step(batch)
        return B

    def _after_step(self, batch):
        pass

    def _finish(self, topic_ids=None):
        """Drain the ring and close the file; returns (path, rows written)."""
        if not hasattr(self, "_ring") or self._writer is None:          # no batch at all: an empty matrix
            out = self._out_path()
            pathlib.Path(out).parent.mkdir(parents=True, exist_ok=True)
            self._writer = StreamingCSRPickle(out, self._encoder().dim,
                                              np.float16 if self.weight_dtype == torch.float16 else np.float32)
            self._ring, self._inflight, self._next = [], collections.deque(), 0
        self._write_due(0)
        n, nnz = self._writer.rows, self._writer.nnz
        out = self._writer.close(topic_ids)
        print(f"\nWrote {n} sparse rows ({nnz} nonzeros) to {out}")
        del self._ring, self._inflight, self._writer, self._next
        return out, n

    def test_epoch_end(self, rows_per_batch):
        out_file, _ = self._finish()
        if dist.is_available() and dist.is_initialized():
            dist.barrier()                           # nobody leaves before every shard is on disk
        return out_file


class GenerateSparseQueryEmbeddingsTask(GenerateSparseEmbeddingsTask):
    """Question side: the query encoder over ``batch["query_ids"]``; writes ``sparse_query.pkl`` (fp32 weights) to
    ``query_emb_output_path``, by default next to the passage shards, with the topic ids when the batches have them."""

    batch_key = "query_ids"
    weight_dtype = torch.float32

    def __init__(self, hnsw_index=False, output_path="/tmp/results.jsonl", query_emb_output_path=None, passages="",
                 **kwargs):
        super().__init__(**kwargs)
        self.hnsw_index = hnsw_index
        self.output_path = output_path
        self.query_emb_output_path = query_emb_output_path or os.path.join(self.ctx_embeddings_dir, "sparse_query.pkl")
        self._topic_ids = []

    def _encoder(self):
        return self.query_encoder

    def _out_path(self):
        return self.query_emb_output_path

    def _after_step(self, batch):
        if "topic_ids" in batch:
            self._topic_ids.extend(batch["topic_ids"])

    def test_epoch_end(self, rows_per_batch):
        topic_ids, self._topic_ids = self._topic_ids, []
        return self._finish(topic_ids or None)[0]
