"""Streaming writer and reader for the sparse embedding files ``sparse_{rank:04}.pkl`` / ``sparse_query.pkl``.

A file is a pickle (protocol 4) of one dict of numpy arrays, one CSR row per passage or query:

    offsets  int64 [N + 1]     row i's entries are [offsets[i], offsets[i + 1])
    terms    int32 [nnz]       vocabulary ids, ascending inside a row
    weights  fp16 [nnz] (passages) or fp32 [nnz] (queries)
    V        int               the vocabulary size
    topic_ids list [N]         (queries read with topic ids only)

Batches are appended to raw spool files next to the output as they arrive, so a shard is never held in RAM; ``close``
writes the pickle around the spooled bytes by hand (each array is ``numpy.frombuffer(BINBYTES8 <raw>, dtype)``, no
memo) and removes the spools.
"""
import os
import pickle
import shutil
import struct

import numpy as np

from .reps_writer import _body

_COPY = 1 << 24


def _str(s):
    b = s.encode()
    return b"\x8c" + bytes([len(b)]) + b                     # SHORT_BINUNICODE


def _array_head(nbytes):
    # numpy.frombuffer(<bytes>, dtype): STACK_GLOBAL, then BINBYTES8 <len>; the raw bytes follow
    return _str("numpy") + _str("frombuffer") + b"\x93" + b"\x8e" + struct.pack("<Q", int(nbytes))


def _array_tail(dtype):
    return _str(np.dtype(dtype).str) + b"\x86R"               # TUPLE2, REDUCE


class StreamingCSRPickle:
    """``w = StreamingCSRPickle(path, V, np.float16); w.append(counts, terms, weights) ...; w.close()``."""

    def __init__(self, path, V, weight_dtype):
        self.path, self.V, self.wdtype = path, int(V), np.dtype(weight_dtype)
        self.rows, self.nnz = 0, 0
        self._spools = {k: open(f"{path}.{k}.part", "wb") for k in ("counts", "terms", "weights")}

    def append(self, counts, terms, weights):
        """counts int64 [b] (entries per row), terms int32 [m], weights [m] of the file's weight dtype (numpy or CPU
        tensors, m = counts.sum())."""
        counts, terms, weights = (np.asarray(x) for x in (counts, terms, weights))
        assert counts.dtype == np.int64 and terms.dtype == np.int32 and weights.dtype == self.wdtype
        assert terms.size == weights.size
        for k, a in (("counts", counts), ("terms", terms), ("weights", weights)):
            self._spools[k].write(memoryview(np.ascontiguousarray(a)).cast("B"))
        self.rows += counts.size
        self.nnz += terms.size

    def close(self, topic_ids=None):
        if self._spools is None:
            return self.path
        for f in self._spools.values():
            f.close()
        parts = {k: f"{self.path}.{k}.part" for k in self._spools}
        self._spools = None
        with open(self.path, "wb") as g:
            g.write(b"\x80\x04}(")                                     # PROTO 4, EMPTY_DICT, MARK
            g.write(_str("offsets") + _array_head(8 * (self.rows + 1)))
            g.write(np.zeros(1, np.int64).tobytes())
            run = 0
            with open(parts["counts"], "rb") as f:
                while True:
                    c = np.frombuffer(f.read(_COPY), dtype=np.int64)
                    if not c.size:
                        break
                    off = run + np.cumsum(c)
                    run = int(off[-1])
                    g.write(off.tobytes())
            assert run == self.nnz
            g.write(_array_tail(np.int64))
            for key, dt in (("terms", np.int32), ("weights", self.wdtype)):
                g.write(_str(key) + _array_head(self.nnz * np.dtype(dt).itemsize))
                with open(parts[key], "rb") as f:
                    shutil.copyfileobj(f, g, _COPY)
                g.write(_array_tail(dt))
            g.write(_str("V") + _body(self.V))
            if topic_ids is not None:
                g.write(_str("topic_ids") + _body(list(topic_ids)))
            g.write(b"u.")                                           # SETITEMS, STOP
        for p in parts.values():
            os.remove(p)
        return self.path


def load_csr(path):
    """The dict of a sparse embedding file; ValueError when it is not one (missing keys, inconsistent offsets)."""
    with open(path, "rb") as f:
        d = pickle.load(f)
    if not isinstance(d, dict) or not {"offsets", "terms", "weights", "V"} <= set(d):
        raise ValueError(f"{path} is not a sparse embedding file (a dict with offsets, terms, weights and V)")
    off, terms, w = d["offsets"], d["terms"], d["weights"]
    if off.ndim != 1 or off.size < 1 or off[0] != 0 or int(off[-1]) != terms.size or terms.size != w.size or \
            bool(np.any(np.diff(off) < 0)):
        raise ValueError(f"{path}: offsets, terms and weights do not form a CSR matrix")
    return d
