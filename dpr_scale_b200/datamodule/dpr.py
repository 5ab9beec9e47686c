"""Input pipeline for the training step with the interface of the reference's
``dpr_scale.datamodule.dpr.DenseRetrieverJsonlDataModule`` (/root/reference/dpr_scale/datamodule/dpr.py:263-331,
loaders :178-216) and ``MemoryMappedDataset`` (:23-53).

What the reference does per step, on the training thread with ``num_workers: 0``: seek + readline for every row, ujson
parse, negative sampling, tokenise ~(2+n)·B sequences, then a blocking H2D copy inside the step.  At the GPU step times of
this path (tens of ms for 128 queries + 1024 contexts) that serial CPU work is longer than the GPU work.  Here:

  * ``LineFile``: the JSONL file is mmap'ed once and its line offsets are found with a vectorised newline scan
    (numpy over the mapping, 64 MB at a time) instead of a Python readline loop; rows are zero-copy slices.
  * ``BatchStream``: a background thread assembles batch i+1.. while the GPU runs batch i: row fetch, JSON and the
    sampling draws (cheap; the draw order is part of the reference's behaviour), then ONE ``encode_batch`` on the Rust
    tokeniser (parallel over the ~1000 contexts, GIL released) with the int64 tensors built directly - the HuggingFace
    Python wrapper the reference calls costs 4x the tokenisation itself (270 ms vs 46 ms per batch on 8 cores).  The
    batch is staged in pinned memory and copied H2D on a side CUDA stream; the training thread only waits on a CUDA
    event.  Depth-bounded queue (``prefetch_batches``).
  * Batch order, sampling draws and tensor contents are the reference's: sequential rows on one GPU
    (DataLoader(shuffle=False), :187-193), ``ContiguousDistributedSampler`` (utils/utils.py:31-80) across ranks.

``prefetch_batches=0`` gives the plain synchronous loader (used by the parity tests to compare batch for batch).
"""
import ast
import math
import mmap
import os
import queue
import random
import sys
import threading

import numpy as np
import torch

from ..transforms.dpr_distill_transform import DPRDistillTransform
from ..transforms.dpr_transform import DPRCrossAttentionTransform, DPRTransform, maybe_add_title
from ..transforms.hf_transform import HFTransform
from ..utils.lightning_shim import LightningDataModule

_SCAN_BYTES = 64 << 20


class LineFile:
    """Random access to the lines of a text file through an mmap (MemoryMappedDataset, datamodule/dpr.py:23-53):
    ``len()`` = number of lines (a last line without newline counts), ``[i]`` = the line as bytes incl. its newline."""

    def __init__(self, path, header=False):
        self.path = path
        self._file = open(path, mode="rb")
        size = os.fstat(self._file.fileno()).st_size
        self.mm = mmap.mmap(self._file.fileno(), 0, access=mmap.ACCESS_READ) if size else b""
        starts = [np.zeros(1, dtype=np.int64)]
        for lo in range(0, size, _SCAN_BYTES):
            chunk = np.frombuffer(self.mm, dtype=np.uint8, count=min(_SCAN_BYTES, size - lo), offset=lo)
            starts.append(np.flatnonzero(chunk == 10).astype(np.int64) + (lo + 1))
        bounds = np.concatenate(starts)
        if size == 0 or bounds[-1] != size:
            bounds = np.append(bounds, size)        # unterminated last line (or empty file: bounds = [0, 0])
        if header:
            bounds = bounds[1:]
        self._bounds = bounds
        self.count = max(len(bounds) - 1, 0) if size else 0

    def __len__(self):
        return self.count

    def process_line(self, line):
        return line

    def __getitem__(self, index):
        if not 0 <= index < self.count:
            raise KeyError(index)
        index = int(index)                  # retrieval hands over float row ids (np.zeros result arrays)
        return self.process_line(bytes(self.mm[self._bounds[index]:self._bounds[index + 1]]))

    def __iter__(self):
        return (self[i] for i in range(self.count))


MemoryMappedDataset = LineFile   # the reference's name


class MultiSourceDataset:
    """Several JSONL files of (at least) ``min`` rows: row i is read from a file drawn with ``random.choice`` at every
    access (datamodule/dpr.py:56-77); the draw order is part of the behaviour, so accesses stay sequential."""

    def __init__(self, paths, header=False):
        self.datasets = [LineFile(path, header) for path in paths]
        self.data_size = min(len(d) for d in self.datasets)
        assert self.data_size > 0, "One of the path in datamodule.train_path is empty"

    def __len__(self):
        return self.data_size

    def __getitem__(self, index):
        return random.choice(self.datasets)[index]


def _split_quoted(line, sep):
    """One delimited row with the reference's minimal csv unquoting (datamodule/dpr.py:94-100)."""
    row = line.decode().rstrip("\r\n").split(sep)
    return [v.strip('"').replace('""', '"') if v and v[0] == '"' and v[-1] == '"' else v for v in row]


class CSVDataset(LineFile):
    """Delimited file with a header row -> dict per row (datamodule/dpr.py:80-107).  A row whose field count differs
    from the header yields None, as in the reference (its fallback evaluates row 0 but does not return it)."""

    def __init__(self, path, sep="\t"):
        super().__init__(path, header=False)
        self.sep = sep
        self.columns = _split_quoted(bytes(self.mm[self._bounds[0]:self._bounds[1]]), sep) if self.count else []
        self._bounds = self._bounds[1:]
        self.count = max(self.count - 1, 0)

    def process_line(self, line):
        vals = _split_quoted(line, self.sep)
        if len(self.columns) == len(vals):
            return dict(zip(self.columns, vals))
        return None


class QueryCSVDataset(LineFile):
    """question <sep> python-literal list of answers, no header (datamodule/dpr.py:110-134)."""

    def __init__(self, path, sep="\t"):
        super().__init__(path, header=False)
        self.sep = sep

    def process_line(self, line):
        vals = _split_quoted(line, self.sep)
        return {"question": vals[0], "answers": ast.literal_eval(vals[1])}


class QueryTSVDataset(LineFile):
    """qid <sep> question, no header (datamodule/dpr.py:137-159)."""

    def __init__(self, path, sep="\t"):
        super().__init__(path, header=False)
        self.sep = sep

    def process_line(self, line):
        vals = _split_quoted(line, self.sep)
        return {"id": vals[0], "question": vals[1]}


def contiguous_test_shard(n, num_replicas, rank):
    """Row range of ``ContiguousDistributedSamplerForTest`` (utils/utils.py:83-91): contiguous, unpadded."""
    shard = n // num_replicas + 1
    return list(range(rank * shard, min((rank + 1) * shard, n)))


def contiguous_shard_indices(n, num_replicas, rank, replicas_per_node=1, shuffle=True, seed=0, epoch=0,
                             drop_last=False):
    """Row order of ``ContiguousDistributedSampler`` (utils/utils.py:31-80): every NODE owns one contiguous chunk of
    the (padded) row range, shuffled with a generator seeded by seed + epoch + node_rank; the node's GPUs take
    interleaved slices of it."""
    if drop_last and n % num_replicas != 0:
        num_samples = math.ceil((n - num_replicas) / num_replicas)
    else:
        num_samples = math.ceil(n / num_replicas)
    total = num_samples * num_replicas
    indices = list(range(n))
    if not drop_last:
        pad = total - n
        indices += indices[:pad] if pad <= n else (indices * math.ceil(pad / n))[:pad]
    else:
        indices = indices[:total]
    chunk = num_samples * replicas_per_node
    node_rank, local_rank = rank // replicas_per_node, rank % replicas_per_node
    indices = indices[node_rank * chunk:(node_rank + 1) * chunk]
    if shuffle:
        g = torch.Generator()
        g.manual_seed(seed + epoch + node_rank)
        indices = [indices[j] for j in torch.randperm(len(indices), generator=g).tolist()]
    indices = indices[local_rank::replicas_per_node]
    assert len(indices) == num_samples
    return indices


def _plain(obj):
    """BatchEncoding -> dict so that the staged batch is made of tensors and dicts only."""
    if hasattr(obj, "keys") and not isinstance(obj, dict):
        return {k: obj[k] for k in obj.keys()}
    return obj


def _map_tensors(obj, fn):
    obj = _plain(obj)
    if isinstance(obj, dict):
        return {k: _map_tensors(v, fn) for k, v in obj.items()}
    return fn(obj) if torch.is_tensor(obj) else obj


class BatchStream:
    """Iterable over collated batches with background assembly and device staging (see module docstring)."""

    def __init__(self, dataset, order, batch_size, collate, drop_last=False, prefetch_batches=4, device=None):
        self.dataset, self.order, self.batch_size, self.collate = dataset, order, int(batch_size), collate
        self.drop_last, self.prefetch_batches = drop_last, int(prefetch_batches)
        self.device = torch.device(device) if device is not None else None

    def __len__(self):
        n = len(self.order())
        return n // self.batch_size if self.drop_last else math.ceil(n / self.batch_size)

    def _batches(self):
        idx = self.order()
        for lo in range(0, len(idx), self.batch_size):
            rows = idx[lo:lo + self.batch_size]
            if self.drop_last and len(rows) < self.batch_size:
                return
            yield self.collate([self.dataset[i] for i in rows])

    def _stage(self, batch, copy_stream):
        """Pinned staging + async H2D on the side stream; returns (device batch, event) or (batch, None) on CPU."""
        if self.device is None or self.device.type != "cuda":
            return _map_tensors(batch, lambda t: t), None
        with torch.cuda.stream(copy_stream):
            out = _map_tensors(batch, lambda t: t.pin_memory().to(self.device, non_blocking=True))
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return out, ev

    def _deliver(self, item):
        batch, ev = item
        if ev is not None:
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ev)
            _map_tensors(batch, lambda t: (t.record_stream(cur), t)[1])
        return batch

    def __iter__(self):
        copy_stream = torch.cuda.Stream(self.device) if self.device is not None and self.device.type == "cuda" else None
        if self.prefetch_batches <= 0:
            for b in self._batches():
                yield self._deliver(self._stage(b, copy_stream))
            return
        q = queue.Queue(maxsize=self.prefetch_batches)
        stop = threading.Event()

        def offer(msg):
            """Blocking put that gives up as soon as the consumer has gone away."""
            while not stop.is_set():
                try:
                    q.put(msg, timeout=0.1)
                    return True
                except queue.Full:
                    continue
            return False

        def produce():
            try:
                if copy_stream is not None:
                    torch.cuda.set_device(self.device)
                for b in self._batches():
                    if not offer(("batch", self._stage(b, copy_stream))):
                        return
                offer(("end", None))
            except BaseException as e:  # noqa: surfaced on the training thread
                offer(("error", e))

        worker = threading.Thread(target=produce, name="dprb-batch-stream", daemon=True)
        # the assembly thread holds the GIL for tens of ms per batch (JSON, Python loops, list -> array); a short
        # switch interval lets the training thread take it back within 0.5 ms whenever it needs to launch kernels
        old_interval = sys.getswitchinterval()
        sys.setswitchinterval(min(old_interval, 5e-4))
        worker.start()
        try:
            while True:
                kind, item = q.get()
                if kind == "end":
                    return
                if kind == "error":
                    raise item
                yield self._deliver(item)
        finally:
            stop.set()
            worker.join(timeout=5.0)
            sys.setswitchinterval(old_interval)


class DenseRetrieverDataModuleBase(LightningDataModule):
    """Loaders of datamodule/dpr.py:162-216 on top of BatchStream."""

    def __init__(self, transform, *args, **kwargs):
        super().__init__()
        self.text_transform = transform
        self.prefetch_batches = 4
        self.device_prefetch = True
        self.fast_tokenize = True
        self.epoch = 0

    def _transform(self, texts):
        if isinstance(self.text_transform, HFTransform):
            return self.text_transform(texts)
        return self.text_transform({"text": texts})["token_ids"]

    def _device(self):
        if not (self.device_prefetch and torch.cuda.is_available()):
            return None
        tr = getattr(self, "trainer", None)
        return getattr(tr, "device", None) or torch.device("cuda", torch.cuda.current_device())

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def _train_order(self):
        n = len(self.datasets["train"])
        tr = getattr(self, "trainer", None)
        world = getattr(tr, "world_size", 1) if tr is not None else 1
        if world and world > 1:
            per_node = getattr(tr, "gpus", None) or world
            return contiguous_shard_indices(n, world, tr.global_rank, per_node, True, 0, self.epoch, False)
        return list(range(n))

    def _eval_order(self, split):
        """Lightning (replace_sampler_ddp, the reference's default) wraps the un-sampled val / test loaders of
        datamodule/dpr.py:197-216 in DistributedSampler(shuffle=False): rank r reads rows r, r+W, r+2W, ... of the row
        range padded (by wrapping around) to a multiple of W.  Single process: the plain row order."""
        n = len(self.datasets[split])
        tr = getattr(self, "trainer", None)
        world = getattr(tr, "world_size", 1) if tr is not None else 1
        if world and world > 1 and n > 0:
            total = math.ceil(n / world) * world
            idx = list(range(n))
            idx += (idx * math.ceil((total - n) / n))[:total - n]
            return idx[tr.global_rank:total:world]
        return list(range(n))

    def _stream(self, split, order, batch_size, collate):
        return BatchStream(self.datasets[split], order, batch_size, collate, drop_last=False,
                           prefetch_batches=self.prefetch_batches, device=self._device())

    def train_dataloader(self):
        return self._stream("train", self._train_order, self.batch_size, self.collate_train)

    def val_dataloader(self):
        return self._stream("valid", lambda: self._eval_order("valid"), self.val_batch_size, self.collate_eval)

    def test_dataloader(self):
        return self._stream("test", lambda: self._eval_order("test"), self.test_batch_size, self.collate_test)

    def collate_eval(self, batch):
        return self.collate(batch, "eval")

    def collate_test(self, batch):
        return self.collate(batch, "test")

    def collate_train(self, batch):
        return self.collate(batch, "train")


class DenseRetrieverJsonlDataModule(DenseRetrieverDataModuleBase):
    """DPR-format JSONL (datamodule/dpr.py:263-331); same keyword arguments, plus ``prefetch_batches`` (0 = synchronous)
    ``device_prefetch`` (stage batches on the GPU from the background thread) and ``fast_tokenize``.  With
    ``use_cross_attention`` the batches are cross-encoder training groups (transforms.dpr_transform
    DPRCrossAttentionTransform), assembled on the same background thread."""

    def __init__(self, transform, train_path: str, val_path: str, test_path: str, batch_size: int = 2,
                 val_batch_size: int = 0, test_batch_size: int = 0, num_positive: int = 1, num_negative: int = 7,
                 neg_ctx_sample: bool = True, pos_ctx_sample: bool = False, num_val_negative: int = 7,
                 num_test_negative: int = 0, drop_last: bool = False, num_workers: int = 0, use_title: bool = False,
                 sep_token: str = " ", use_cross_attention: bool = False, rel_sample: bool = False,
                 prefetch_batches: int = 4, device_prefetch: bool = True, fast_tokenize: bool = True, *args,
                 **kwargs):
        super().__init__(transform)
        self.batch_size = batch_size
        self.val_batch_size = val_batch_size if val_batch_size else batch_size
        self.test_batch_size = test_batch_size if test_batch_size else self.val_batch_size
        transform_class = DPRCrossAttentionTransform if use_cross_attention else DPRTransform
        self.dpr_transform = transform_class(transform, num_positive, num_negative, neg_ctx_sample, pos_ctx_sample,
                                          num_val_negative, num_test_negative, use_title, sep_token, rel_sample,
                                          **kwargs)
        self.num_workers = num_workers     # accepted; assembly runs on the BatchStream thread
        self.prefetch_batches = prefetch_batches
        self.device_prefetch = device_prefetch
        self.fast_tokenize = fast_tokenize      # False: tokenise through the HF wrapper call, as the reference does
        self.datasets = {"train": LineFile(train_path), "valid": LineFile(val_path), "test": LineFile(test_path)}

    def collate(self, batch, stage):
        if not self.fast_tokenize:
            return self.dpr_transform(batch, stage)
        rows = batch if type(batch) is list else batch[self.dpr_transform.text_column]
        return self.dpr_transform.finish(self.dpr_transform.select(rows, stage))


class DPRDistillJsonlDataModule(DenseRetrieverDataModuleBase):
    """Distillation JSONL (datamodule/dpr.py:225-266 of the reference): question + target vectors per row, assembled by
    DPRDistillTransform on the BatchStream thread (JSON, sampling, vector parsing, one tokeniser call), staged in pinned
    memory and copied to the GPU on the side stream.  Same keyword arguments, plus ``prefetch_batches`` (0 =
    synchronous), ``device_prefetch`` and ``fast_tokenize``."""

    def __init__(self, transform, train_path: str, val_path: str, test_path: str, batch_size: int = 2,
                 val_batch_size: int = 0, test_batch_size: int = 0, pos_ctx_sample: bool = True, drop_last: bool = False,
                 num_workers: int = 0, prefetch_batches: int = 4, device_prefetch: bool = True, fast_tokenize: bool = True,
                 *args, **kwargs):
        super().__init__(transform)
        self.batch_size = batch_size
        self.val_batch_size = val_batch_size if val_batch_size else batch_size
        self.test_batch_size = test_batch_size if test_batch_size else self.val_batch_size
        self.drboost_distill_transform = DPRDistillTransform(transform, pos_ctx_sample, **kwargs)
        self.num_workers = num_workers     # accepted; assembly runs on the BatchStream thread
        self.prefetch_batches = prefetch_batches
        self.device_prefetch = device_prefetch
        self.fast_tokenize = fast_tokenize
        self.datasets = {"train": LineFile(train_path), "valid": LineFile(val_path), "test": LineFile(test_path)}

    def collate(self, batch, stage):
        tf = self.drboost_distill_transform
        if not self.fast_tokenize:
            return tf(batch, stage)
        rows = batch if type(batch) is list else batch[tf.text_column]
        return tf.finish(tf.select(rows, stage))


class DenseRetrieverMultiJsonlDataModule(DenseRetrieverJsonlDataModule):
    """Several training files sampled per row + contexts given as ``docidx`` into a corpus table
    (datamodule/dpr.py:333-412, the DRAGON configs): the JSONL rows stay light and DPRTransform reads text / title of
    the selected contexts from the mmap'ed corpus."""

    def __init__(self, transform, train_path, val_path: str, test_path: str, corpus_path: str = None, *args, **kwargs):
        first = train_path[0] if not isinstance(train_path, str) else train_path
        super().__init__(transform, first, val_path, test_path, *args, **kwargs)
        paths = [train_path] if isinstance(train_path, str) else list(train_path)
        self.datasets["train"] = MultiSourceDataset(paths)
        if corpus_path is not None:
            self.dpr_transform.corpus = LineFile(corpus_path, header=True)


class _EncodeOnlyDataModule(DenseRetrieverDataModuleBase):
    """Shared loader logic of the two embedding-generation datamodules (datamodule/dpr.py:457-479, :507-529): one
    'test' split, every loader is the test loader, contiguous unpadded shards across ranks."""

    def _encode(self, texts):
        tf = self.text_transform
        if self.fast_tokenize and hasattr(tf, "encode_fast"):
            return tf.encode_fast(texts)
        return self._transform(texts)

    def _test_order(self):
        n = len(self.datasets["test"])
        tr = getattr(self, "trainer", None)
        world = getattr(tr, "world_size", 1) if tr is not None else 1
        if world and world > 1:
            return contiguous_test_shard(n, world, tr.global_rank)
        return list(range(n))

    def test_dataloader(self):
        return self._stream("test", self._test_order, self.test_batch_size, self.collate_test)

    def val_dataloader(self):
        return self.test_dataloader()

    def train_dataloader(self):
        return self.test_dataloader()


class DenseRetrieverPassagesDataModule(_EncodeOnlyDataModule):
    """Passage TSV (id, text, title) for generate_embeddings (datamodule/dpr.py:415-479)."""

    def __init__(self, transform, test_path: str, test_batch_size: int = 128, num_workers: int = 0,
                 use_title: bool = False, sep_token: str = " [SEP] ", prefetch_batches: int = 4,
                 device_prefetch: bool = True, fast_tokenize: bool = True, *args, **kwargs):
        super().__init__(transform)
        self.test_batch_size = test_batch_size
        self.use_title = use_title
        self.sep_token = sep_token
        self.num_workers = num_workers
        self.prefetch_batches, self.device_prefetch, self.fast_tokenize = prefetch_batches, device_prefetch, fast_tokenize
        self.datasets = {"test": CSVDataset(test_path)}

    def collate(self, batch, stage):
        ctx = self._encode([maybe_add_title(row["text"], row["title"], self.use_title, self.sep_token) for row in batch])
        if "id" in batch[0]:
            return {"contexts_ids": ctx, "corpus_ids": [row["id"] for row in batch]}
        return {"contexts_ids": ctx}


class DenseRetrieverQueriesDataModule(_EncodeOnlyDataModule):
    """Question file for generate_query_embeddings (datamodule/dpr.py:482-529)."""

    def __init__(self, transform, test_path: str, test_batch_size: int = 128, num_workers: int = 0,
                 trec_format: bool = False, prefetch_batches: int = 4, device_prefetch: bool = True,
                 fast_tokenize: bool = True, *args, **kwargs):
        super().__init__(transform)
        self.test_batch_size = test_batch_size
        self.num_workers = num_workers
        self.prefetch_batches, self.device_prefetch, self.fast_tokenize = prefetch_batches, device_prefetch, fast_tokenize
        self.datasets = {"test": QueryTSVDataset(test_path) if trec_format else QueryCSVDataset(test_path)}

    def collate(self, batch, stage):
        return {"query_ids": self._encode([row["question"] for row in batch])}
