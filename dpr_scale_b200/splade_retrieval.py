#!/usr/bin/env python3
"""First-stage retrieval with SPLADE encoders from the sparse files GenerateSparseEmbeddingsTask writes
(``sparse_{rank:04}.pkl`` per passage shard, ``sparse_query.pkl``), with run_retrieval's flags and output files:

  python -m dpr_scale_b200.splade_retrieval --ctx_embeddings_dir /idx --questions_tsv_path queries.tsv \\
      --passages_tsv_path psgs.tsv --output_runfile_path /out/run.trec --topk 100 --trec_format

score(q, d) = sum over the terms t both hold of w_q[t] * w_d[t], searched on the device by ``dprb_sparse_search``
over an inverted index (``SparseIndex``): passage weights are stored as fp16, every product is formed in fp32 and the
sums are int64 fixed point at 2^-32, so two runs give identical results and a query's results do not depend on the
other queries.  Ranking: descending score, ties towards the lower passage row.  Scores are written rounded to fp16
like run_retrieval's unless ``--fp32_scores`` is given.

Under torchrun every rank loads the contiguous block of ``sparse_*`` shards it owns (run_retrieval.rank_files) and
searches it; the per-rank [Q, k] lists are merged with one all-gather and ops.topk_merge, and rank 0 writes the run.
"""
import argparse
import glob
import os
import warnings

import numpy as np
import torch
import torch.distributed as dist

from . import ops
from .run_retrieval import Passages, Questions, _world, gather_rank_lists, get_logger, rank_files, write_run
from .utils.csr_writer import load_csr


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--ctx_embeddings_dir", type=str, default="")
    p.add_argument("--query_emb_path", type=str, default="",
                   help="if left empty, will use <ctx_embeddings_dir>/sparse_query.pkl")
    p.add_argument("--questions_tsv_path", type=str, default="")
    p.add_argument("--passages_tsv_path", type=str, default="")
    p.add_argument("--output_runfile_path", type=str, default="")
    p.add_argument("--topk", type=int, default=100)
    p.add_argument("--trec_format", action="store_true")
    p.add_argument("--run_name", type=str, default="splade")
    p.add_argument("--ignore_identical_ids", action="store_true",
                   help="this is used for BEIR Arguana and Quora datasets")
    p.add_argument("--fp32_scores", action="store_true", help="write fp32 scores instead of fp16-rounded ones")
    p.add_argument("--device", type=str, default="cuda", help="device holding the index (the kernels need CUDA)")
    return p


def _dev(a, dtype, device):
    if torch.is_tensor(a):
        return a.to(device=device, dtype=dtype)
    with warnings.catch_warnings():                     # arrays read from a file are read-only; they are only copied
        warnings.simplefilter("ignore", UserWarning)
        return torch.from_numpy(np.asarray(a)).to(device=device, dtype=dtype)


def check_terms(terms, V, what):
    if terms.size and (int(terms.min()) < 0 or int(terms.max()) >= V):
        raise ValueError(f"{what} holds term ids outside [0, {V})")


class SparseIndex:
    """An inverted SPLADE index on one device, searched with ``dprb_sparse_search``.

    Built once from a CSR passage matrix: postings sorted by term and, inside a term, by row (a stable sort on term of
    the row-ordered entries), stored as row int32 and weight fp16, with term_ptr int64 [V + 1] and the int64 id of every
    row.  Device memory: about 6 * nnz + 8 * (V + 1) + 8 * N bytes, plus the query-block accumulator of at most 2 GiB
    that ``ops.sparse_search`` keeps cached per device."""

    def __init__(self, offsets, terms, weights, V, ids=None, device="cuda"):
        """offsets int [N + 1], terms int [nnz] in [0, V), weights float [nnz] (rounded to fp16); ids int64 [N] (the
        id returned for each row, default the row).  ValueError: an empty index, term ids out of range, a row whose
        terms are not strictly ascending (a repeated term), a weight that does not fit fp16."""
        offsets = offsets.cpu().numpy() if torch.is_tensor(offsets) else np.asarray(offsets, dtype=np.int64)
        N, nnz = offsets.size - 1, int(offsets[-1]) if offsets.size else 0
        if N < 1:
            raise ValueError("the sparse index is empty: no passage rows")
        V = int(V)
        ops.sparse_search_check(V, nnz, N, 1)
        dev = self.device = torch.device(device)
        t = _dev(terms, torch.int32, dev)                                # int32 and fp16 keep the build's peak low
        if nnz and (int(t.min()) < 0 or int(t.max()) >= V):
            raise ValueError(f"the passage index holds term ids outside [0, {V})")
        w = _dev(weights, torch.float32, dev)
        if nnz and not (float(w.abs().max()) <= ops.FP16_MAX):
            raise ValueError(f"a passage weight does not fit fp16 (|w| > {ops.FP16_MAX:g} or not finite)")
        w = w.half()
        rows = torch.repeat_interleave(torch.arange(N, dtype=torch.int32, device=dev),
                                       _dev(np.diff(offsets), torch.int64, dev))
        # one posting per (term, row): the range bound of search() takes each term's largest weight once per passage
        if nnz > 1 and bool(((t[1:] <= t[:-1]) & (rows[1:] == rows[:-1])).any()):
            raise ValueError("a passage row of the sparse index repeats a term or is not sorted by term (SPLADE "
                             "rows hold each term once, in ascending order)")
        t, order = torch.sort(t, stable=True)
        pad = (nnz + 7) // 8 * 8
        self.row = torch.zeros(max(pad, 8), dtype=torch.int32, device=dev)
        self.weight = torch.zeros(max(pad, 8), dtype=torch.float16, device=dev)
        self.row[:nnz] = rows[order]
        del rows
        self.weight[:nnz] = w[order]
        del w, order
        counts = torch.bincount(t, minlength=V)
        del t
        self.term_ptr = torch.zeros(V + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=self.term_ptr[1:])
        self.term_ptr_host = self.term_ptr.cpu().numpy()
        # largest |fp16 weight| of each term (0 for a term without postings)
        tmax = torch.segment_reduce(self.weight[:nnz].float().abs(), "max", lengths=counts, unsafe=True, initial=0.0)
        self.term_max = tmax.double().cpu().numpy()
        self.ids = _dev(np.arange(N) if ids is None else ids, torch.int64, dev)
        self.N, self.V, self.nnz = N, V, nnz

    @classmethod
    def from_csr(cls, parts, device="cuda"):
        """The index of CSR shards (load_csr dicts, row order = shard order), ids = rows.  ValueError: no shard,
        shards with different V, and what the constructor refuses."""
        if not parts:
            raise ValueError("the sparse index is empty: no sparse_* shard files")
        Vs = sorted({int(d["V"]) for d in parts})
        if len(Vs) > 1:
            raise ValueError(f"the sparse shards have different vocabulary sizes {Vs}")
        offsets = [np.zeros(1, np.int64)]
        base = 0
        for d in parts:
            offsets.append(d["offsets"][1:] + base)
            base += int(d["offsets"][-1])
        offsets = np.concatenate(offsets)
        terms = np.concatenate([d["terms"] for d in parts])
        weights = np.concatenate([d["weights"] for d in parts])
        return cls(offsets, terms, weights, Vs[0], None, device)

    def search(self, offsets, terms, weights, k):
        """k best rows of every query of a CSR query matrix (offsets [Q + 1], terms [Eq], fp32 weights [Eq], host
        arrays).  Returns device (scores fp32 [Q, k], ids int64 [Q, k])."""
        ops.sparse_search_check(self.V, self.nnz, self.N, int(k))
        offsets = np.asarray(offsets, dtype=np.int64)
        terms = np.asarray(terms, dtype=np.int64)
        wq = np.asarray(weights, dtype=np.float32)
        Q = offsets.size - 1
        check_terms(terms, self.V, "the query matrix")
        if wq.size and not np.isfinite(wq).all():
            raise ValueError("a query weight is not finite")
        # range of the int64 fixed point: each query's sum of |products| stays below 2^30
        c = np.r_[0.0, np.cumsum(np.abs(wq.astype(np.float64)) * self.term_max[terms])]
        reach = c[offsets[1:]] - c[offsets[:-1]]
        if reach.size and float(reach.max()) >= ops.EXPERT_SEARCH_TERM_LIMIT:
            raise ValueError("query and passage weights are too large for the search's fixed-point sums (a query's "
                             f"sum of |w_q w_p| reaches {float(reach.max()):.3g} >= 2^30)")
        dev = self.device
        Qb = min(ops.sparse_search_block_queries(self.N), max(Q, 1))
        scores = torch.empty(Q, k, dtype=torch.float32, device=dev)
        ids = torch.empty(Q, k, dtype=torch.int64, device=dev)
        for q0 in range(0, Q, Qb):
            q1 = min(q0 + Qb, Q)
            e0, e1 = int(offsets[q0]), int(offsets[q1])
            item_end, items = ops.sparse_search_items(self.term_ptr_host, terms[e0:e1])
            seq = np.repeat(np.arange(q1 - q0, dtype=np.int32), np.diff(offsets[q0:q1 + 1]))
            s, i = ops.sparse_search(self.row, self.weight, self.term_ptr, self.nnz, self.ids,
                                     _dev(terms[e0:e1], torch.int32, dev), _dev(wq[e0:e1], torch.float32, dev),
                                     _dev(seq, torch.int32, dev), q1 - q0, _dev(item_end, torch.int32, dev), items,
                                     int(k))
            scores[q0:q1] = s
            ids[q0:q1] = i
        return scores, ids


def shard_paths(ctx_embeddings_dir):
    return sorted(p for p in glob.glob(os.path.join(ctx_embeddings_dir, "sparse_*.pkl"))
                  if os.path.basename(p)[len("sparse_"):-len(".pkl")].isdigit())


def _agree(err, N):
    """Every rank's (refused, rows), with one all-gather, so that a refusal on any rank fails every rank before the
    search's collectives.  Returns the rows of every rank."""
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    mine = torch.tensor([int(err is not None), int(N)], dtype=torch.int64, device=dev)
    every = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
    dist.all_gather(every, mine)
    every = torch.stack(every).cpu().numpy()
    if err is not None:
        raise err
    bad = np.flatnonzero(every[:, 0])
    if bad.size:
        raise ValueError(f"rank {int(bad[0])} refused its sparse shards or the queries")
    return every[:, 1]


def search_distributed(index_paths, query, topk, device="cuda"):
    """Every rank searches the block of shards it owns; the W [Q, k] lists are merged with one all-gather and
    ops.topk_merge.  Returns the global (scores, passage rows) on every rank.  ValueError (on every rank): no shard,
    shards of different V, a query V other than the index's, term ids out of range, a row that repeats a term, topk
    above the passages."""
    if not index_paths:
        raise ValueError("the sparse index is empty: no sparse_* shard files")
    world = _world()
    err, index = None, None
    try:
        parts = [load_csr(p) for p in (rank_files(index_paths, dist.get_rank(), world) if world > 1 else index_paths)]
        index = SparseIndex.from_csr(parts, device)
        if int(query["V"]) != index.V:
            raise ValueError(f"the queries' vocabulary size {int(query['V'])} differs from the index's {index.V}")
        check_terms(np.asarray(query["terms"]), index.V, "the query matrix")
    except ValueError as e:
        if world == 1:
            raise
        err = e
    if world == 1:
        return index.search(query["offsets"], query["terms"], query["weights"], int(topk))
    rows = _agree(err, 0 if index is None else index.N)
    rank = dist.get_rank()
    if int(topk) > int(rows.sum()):
        raise ValueError(f"topk={topk} exceeds the {int(rows.sum())} passages of the index")
    index.ids += int(rows[:rank].sum())                # global passage rows
    k = min(int(topk), index.N)
    s, i = index.search(query["offsets"], query["terms"], query["weights"], k)
    if k < topk:                                       # a shard smaller than topk: pad its list with rows that lose
        s = torch.cat([s, s.new_full((s.shape[0], topk - k), -float("inf"))], 1).contiguous()
        i = torch.cat([i, i.new_full((i.shape[0], topk - k), -1)], 1).contiguous()
    gs, gi = gather_rank_lists(s, i)
    return ops.topk_merge(gs, gi, int(topk))


def main(args, logger=None):
    logger = logger or get_logger()
    logger.info(args.__dict__)
    paths = shard_paths(args.ctx_embeddings_dir)
    qpath = args.query_emb_path or os.path.join(args.ctx_embeddings_dir, "sparse_query.pkl")
    print("Loading sparse query vectors.")
    query = load_csr(qpath)
    if "LOCAL_RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    print("Retrieving results...")
    scores, indexes = search_distributed(paths, query, args.topk, args.device)
    if _world() > 1 and dist.get_rank() != 0:
        return                                      # every rank holds the result; rank 0 writes the run file
    if not args.fp32_scores:
        scores = scores.to(torch.float16)
    scores = scores.float().cpu().numpy().astype(np.float64)
    indexes = indexes.cpu().numpy()
    print(f"Loading questions file {args.questions_tsv_path}")
    questions = list(Questions(args.questions_tsv_path, args.trec_format))
    print(f"Loading passages from {args.passages_tsv_path}")
    passages = Passages(args.passages_tsv_path)
    print(f"Writing output to {args.output_runfile_path}")
    write_run(args.output_runfile_path, passages, questions, scores, indexes, args.trec_format, args.run_name,
              args.ignore_identical_ids)


if __name__ == "__main__":
    main(get_parser().parse_args())
