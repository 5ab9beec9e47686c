"""world_size-2 gloo test (CPU) of the refusals of ``splade_retrieval.search_distributed`` under torchrun: input that
one rank refuses (its shard's vocabulary, a repeated term in a passage row, a topk above the passages of all ranks)
fails every rank with ValueError before the search's collectives, instead of leaving the other ranks waiting in
them.  The GPU kernels are not involved: every case is refused before a search."""
import os
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _write(path, offsets, terms, V):
    from dpr_scale_b200.utils.csr_writer import StreamingCSRPickle
    w = StreamingCSRPickle(path, V, np.float16)
    w.append(np.diff(np.asarray(offsets)).astype(np.int64), np.asarray(terms, np.int32),
             np.ones(len(terms), np.float16))
    w.close()


def _worker(rank, world, port, tmp, ret):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dpr_scale_b200 import splade_retrieval as SR
    q = {"offsets": np.array([0, 1]), "terms": np.array([1], np.int32), "weights": np.ones(1, np.float32), "V": 10}
    out = {}
    for case in ("vocab", "repeat", "topk"):
        d = os.path.join(tmp, case)
        try:
            out[case] = ("ok", SR.search_distributed(SR.shard_paths(d), q, 5 if case == "topk" else 1, "cpu"))
        except ValueError as e:
            out[case] = ("ValueError", str(e))
        dist.barrier()
    ret[rank] = out
    dist.destroy_process_group()


def test_refusal_on_one_rank_fails_every_rank(tmp_path):
    for case in ("vocab", "repeat", "topk"):
        d = tmp_path / case
        d.mkdir()
        _write(str(d / "sparse_0000.pkl"), [0, 2, 3], [1, 4, 2], 10)
        if case == "vocab":
            _write(str(d / "sparse_0001.pkl"), [0, 1], [3], 12)
        elif case == "repeat":
            _write(str(d / "sparse_0001.pkl"), [0, 2], [3, 3], 10)
        else:
            _write(str(d / "sparse_0001.pkl"), [0, 1], [3], 10)           # 3 passages in all, topk 5
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, 29641, str(tmp_path), ret), nprocs=2, join=True)
    assert ret[1]["vocab"][0] == "ValueError" and "differs" in ret[1]["vocab"][1]
    assert ret[1]["repeat"][0] == "ValueError" and "repeats a term" in ret[1]["repeat"][1]
    for case in ("vocab", "repeat"):
        assert ret[0][case] == ("ValueError", "rank 1 refused its sparse shards or the queries")
    for r in (0, 1):
        assert ret[r]["topk"][0] == "ValueError" and "exceeds the 3 passages" in ret[r]["topk"][1]
