"""Forward-only embedding dumps: ``GenerateEmbeddingsTask`` (passages -> ``reps_{rank:04}.pkl``) and
``GenerateQueryEmbeddingsTask`` (questions -> ``query_reps.pkl``), drop-ins for the classes of the same names in
/root/reference/dpr_scale/task/dpr_eval_task.py (:13-49 and :52-84): same constructor keywords, same Lightning test
hooks, same output files (pickle protocol 4 of ONE fp32 CPU tensor, which is what run_retrieval reads).

How this path changes the loop: the encoder runs in its forward-only mode (two activation slots instead of one per layer),
every batch result goes to one of a few pinned host buffers with an asynchronous copy instead of the reference's blocking
``.cpu()`` per batch, and the rows are appended to the pickle's payload as their copies land
(utils/reps_writer.StreamingTensorPickle) - the shard is never held in RAM, where the reference holds it twice
(list of batches + ``torch.cat``, dpr_eval_task.py:40-45: 2 x 8 GB per rank for the 21 M-passage corpus).
"""
import os
import pathlib
import pickle

import collections

import torch
import torch.distributed as dist

from ..utils.reps_writer import StreamingTensorPickle
from .dpr_task import DenseRetrieverTask


class _EmbeddingDumpTask(DenseRetrieverTask):
    """Shared machinery: which batch entry to encode, with which encoder, and where the shard goes."""

    batch_key = None

    def __init__(self, ctx_embeddings_dir, checkpoint_path, **task_kwargs):
        super().__init__(**task_kwargs)
        self.ctx_embeddings_dir = ctx_embeddings_dir
        self.checkpoint_path = checkpoint_path
        pathlib.Path(ctx_embeddings_dir).mkdir(parents=True, exist_ok=True)

    def setup(self, stage: str):
        super().setup("train")                       # always build the encoders, whatever stage the trainer names
        if not self.checkpoint_path:
            return
        print(f"Loading checkpoint from {self.checkpoint_path}")
        state = torch.load(self.checkpoint_path, map_location="cpu", weights_only=False)["state_dict"]
        self._load_state(state)

    def _load_state(self, state):
        self.load_state_dict(state)

    # -- per-batch: encode, then park the result in pinned memory without waiting for it
    def _encode(self, tokens):
        raise NotImplementedError

    def forward(self, tokens):
        return self._encode(tokens)

    # -- per-batch: encode, park the result in a pinned ring slot without waiting for it, write the slot that is due
    RING = 8            # batches in flight between the GPU and the file

    def _out_path(self):
        raise NotImplementedError

    def _ring_init(self):
        if not hasattr(self, "_ring"):
            self._ring, self._inflight, self._writer, self._next = [], collections.deque(), None, 0

    def _ring_slot(self, rows, dim):
        if len(self._ring) < self.RING:
            self._ring.append(None)
        i = self._next % self.RING
        self._next += 1
        buf = self._ring[i]
        if buf is None or buf.shape[0] < rows or buf.shape[1] != dim:
            buf = torch.empty(max(rows, 1), dim, dtype=torch.float32, pin_memory=torch.cuda.is_available())
            self._ring[i] = buf
        return buf

    def _write_due(self, keep):
        """Append to the file every parked batch beyond the `keep` most recent ones (their copies have had time to land)."""
        while len(self._inflight) > keep:
            buf, rows, ev = self._inflight.popleft()
            if ev is not None:
                ev.synchronize()
            self._writer.append(buf[:rows])

    @torch.no_grad()
    def _eval_step(self, batch, batch_idx):
        rep = self(batch[self.batch_key])
        rows, dim = rep.shape
        self._ring_init()
        self._write_due(self.RING - 1)               # the slot about to be reused must have been written out
        buf = self._ring_slot(rows, dim)
        if self._writer is None:
            out = self._out_path()
            pathlib.Path(out).parent.mkdir(parents=True, exist_ok=True)
            self._writer = StreamingTensorPickle(out, dim)
        buf[:rows].copy_(rep.float(), non_blocking=True)
        ev = None
        if rep.is_cuda:
            ev = torch.cuda.Event()
            ev.record()
        self._inflight.append((buf, rows, ev))
        return rows

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, batch_idx)

    def _finish(self):
        """Drain the ring, close the file; returns (path, rows written)."""
        if not hasattr(self, "_ring") or self._writer is None:           # no batch at all: an empty [0, d] tensor
            dim = self.query_encoder.config["hidden_size"] if hasattr(self.query_encoder, "config") else 0
            out = self._out_path()
            pathlib.Path(out).parent.mkdir(parents=True, exist_ok=True)
            w = StreamingTensorPickle(out, dim)
            w.close()
            return out, 0
        self._write_due(0)
        n = self._writer.rows
        out = self._writer.close()
        print(f"\nWrote tensor of size [{n}, {self._writer.dim}] to {out}")
        del self._ring, self._inflight, self._writer, self._next
        return out, n


class GenerateEmbeddingsTask(_EmbeddingDumpTask):
    """Passage side: context encoder over ``batch["contexts_ids"]``; every rank writes its own shard file."""

    batch_key = "contexts_ids"

    def _encode(self, contexts_ids):
        return self.encode_contexts(contexts_ids)

    def _out_path(self):
        if not self.ctx_embeddings_dir:
            self.ctx_embeddings_dir = getattr(self.trainer, "weights_save_path", ".")
        return os.path.join(self.ctx_embeddings_dir, f"reps_{self.global_rank:04}.pkl")

    def test_epoch_end(self, rows_per_batch):
        out_file, _ = self._finish()
        if dist.is_available() and dist.is_initialized():
            dist.barrier()                           # nobody leaves before every shard is on disk (:49)
        return out_file


class GenerateQueryEmbeddingsTask(GenerateEmbeddingsTask):
    """Question side: query encoder over ``batch["query_ids"]``; one file, by default next to the passage shards."""

    batch_key = "query_ids"

    def __init__(self, hnsw_index=False, output_path="/tmp/results.jsonl", query_emb_output_path=None, passages="",
                 **kwargs):
        super().__init__(**kwargs)
        self.hnsw_index = hnsw_index
        self.output_path = output_path
        self.query_emb_output_path = query_emb_output_path or os.path.join(self.ctx_embeddings_dir, "query_reps.pkl")

    def _load_state(self, state):
        """A distillation checkpoint (task/dpr_distill_task.py) holds a query encoder only: its context encoder keys
        may be absent.  Every other missing or unexpected key raises, as a strict load does."""
        if any(k.startswith("context_encoder.") for k in state):
            return self.load_state_dict(state)
        missing, unexpected = self.load_state_dict(state, strict=False)
        missing = [k for k in missing if not k.startswith("context_encoder.")]
        if missing or unexpected:
            raise RuntimeError(f"Error(s) in loading state_dict for {type(self).__name__}: missing keys {missing}, "
                               f"unexpected keys {unexpected}")

    def _encode(self, query_ids):
        return self.encode_queries(query_ids)

    def _out_path(self):
        return self.query_emb_output_path

    def test_epoch_end(self, rows_per_batch):
        return self._finish()[0]
