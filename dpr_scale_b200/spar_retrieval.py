#!/usr/bin/env python3
"""SPAR retrieval with two models' embeddings: the command line and output files of the reference's
``spar/spar_retrieval.py``.

  python -m dpr_scale_b200.spar_retrieval --model_1_emb_dir dense/ --model_2_emb_dir lexical/ \\
      --tsv_passages_path psgs.tsv --jsonl_dataset_paths nq_test.jsonl --pred_filenames nq_test.json \\
      --query_reps_filenames query_reps.pkl --weights 0.7 --output_dir out/ [--pooling concat] [--shard 2]

Each model directory holds its ``reps_*`` passage pickles and one query pickle per dataset.  The two models' vectors
are pooled (``w`` is the dataset's weight; ``q*`` / ``p*`` are model 1's and model 2's vectors):
  concat  queries [q1, w q2],            passages [p1, p2]        score q1.p1 + w q2.p2
  mean    queries (q1 + w q2) / (1 + w), passages (p1 + p2) / 2
  sum     queries q1 + w q2,             passages p1 + p2
and every dataset's pooled queries go through the one brute-force search ``run_retrieval`` uses (``ops.search_topk``
per index segment, ``ops.topk_merge`` across segments and ranks).  The run file has one entry per question:
``question``, ``answers``, ``ctxs`` (``id``, ``title``, ``text``, ``score``) and ``id``.

The pooled passage store is built straight into the fp16 device buffer the search reads: each model's ``reps_*``
files are streamed, one file at a time, into their column block (concat) or pooled chunk by chunk in fp32 on the
device (mean, sum).  No host copy of the pooled corpus is made, so the device needs the bytes of the two stores
together (concat) and the host one ``reps_*`` file per model.  ``--shard`` splits the passage rows into sequential
segments searched one after another; under torchrun every rank searches its contiguous block of rows.  A pooled value
that does not fit fp16 raises.  Scores are the fp32-accumulated inner products of the fp16 vectors.

``--save_embeddings`` also writes the weighted query pickles (under each ``--query_reps_filenames`` name) and the pooled
passage vectors in fp32 as 8 ``reps_000{i}.pkl`` files of ``N // 8 + 1`` rows, so ``run_retrieval`` can search them.
"""
import argparse
import glob
import json
import os
import pickle

import numpy as np
import torch
import torch.distributed as dist

from . import ops
from . import run_retrieval as rr
from .utils.reps_writer import StreamingTensorPickle

POOLINGS = ("concat", "mean", "sum")
CHUNK_ROWS = 1 << 17          # rows moved to the device per copy while a segment is built
SAVED_SHARDS = 8


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--model_1_emb_dir", type=str, required=True)
    p.add_argument("--model_2_emb_dir", type=str, required=True)
    p.add_argument("--tsv_passages_path", type=str, required=True)
    p.add_argument("--jsonl_dataset_paths", nargs="+", help="paths to the JSONL dataset files; one for each dataset")
    p.add_argument("--output_dir", required=True,
                   help="directory for the retrieval results, and the pooled embeddings with --save_embeddings")
    p.add_argument("--save_embeddings", action="store_true", help="also write the pooled query and passage vectors")
    p.add_argument("--pred_filenames", nargs="+",
                   default=["nq_test.json", "squad1_test.json", "trivia_test.json", "webq_test.json", "trec_test.json"],
                   help="names of the JSON prediction files; one for each dataset")
    p.add_argument("--query_reps_filenames", nargs="+",
                   default=["query_reps_nq_test.pkl", "query_reps_squad1_test.pkl", "query_reps_trivia_test.pkl",
                            "query_reps_webq_test.pkl", "query_reps_trec_test.pkl"],
                   help="names of the query embedding files in both model directories; one for each dataset")
    p.add_argument("--weights", nargs="+", type=float, help="model 2's query weight; one for each dataset (default 1)")
    p.add_argument("--topk", type=int, default=100, help="top-k retrieval results will be saved in the output.")
    p.add_argument("--pooling", type=str, default="concat", help="concat, mean or sum (default: concat)")
    p.add_argument("--shard", type=int, default=1, help="search the passages in this many sequential segments")
    p.add_argument("--device", type=str, default="cuda", help="device holding the index (the kernels need CUDA)")
    return p


# ------------------------------------------------------------------ inputs
def reps_paths(emb_dir):
    paths = sorted(glob.glob(os.path.join(emb_dir, "reps_*")))
    if not paths:
        raise FileNotFoundError(f"no reps_* passage embedding files under {emb_dir}")
    return paths


def check_args(args):
    """Every refusal that needs no GPU work: list lengths, pooling mode, shard count, missing inputs."""
    pooling = args.pooling.lower()
    if pooling not in POOLINGS:
        raise ValueError(f"unknown pooling {args.pooling!r}: expected one of {', '.join(POOLINGS)}")
    n = len(args.jsonl_dataset_paths or [])
    weights = args.weights if args.weights else [1.0] * n
    lengths = {"--jsonl_dataset_paths": n, "--pred_filenames": len(args.pred_filenames),
               "--query_reps_filenames": len(args.query_reps_filenames), "--weights": len(weights)}
    if n == 0 or len(set(lengths.values())) != 1:
        raise ValueError("one entry per dataset is needed in each list: "
                         + ", ".join(f"{k} has {v}" for k, v in lengths.items()))
    if args.shard < 1:
        raise ValueError(f"--shard must be at least 1, got {args.shard}")
    needed = [args.tsv_passages_path] + list(args.jsonl_dataset_paths)
    for d in (args.model_1_emb_dir, args.model_2_emb_dir):
        reps_paths(d)
        needed += [os.path.join(d, name) for name in args.query_reps_filenames]
    for path in needed:
        if not os.path.isfile(path):
            raise FileNotFoundError(f"no such file: {path}")
    return pooling, [float(w) for w in weights]


def load_jsonl(path):
    with open(path) as f:
        return [json.loads(line) for line in f if line.strip()]


def load_tensor(path):
    with open(path, "rb") as f:
        return torch.as_tensor(pickle.load(f)).float()


class RepsRows:
    """The rows of one model's ``reps_*`` pickles in file order, holding one file in host memory at a time."""

    def __init__(self, paths):
        self.paths, self.next_file, self.cur, self.pos = list(paths), 0, None, 0

    def _fill(self):
        while self.cur is None or self.pos == self.cur.shape[0]:
            if self.next_file == len(self.paths):
                return False
            self.cur, self.pos = load_tensor(self.paths[self.next_file]), 0
            self.next_file += 1
        return True

    @property
    def width(self):
        if not self._fill():
            raise ValueError(f"the reps_* files {self.paths} hold no passage vectors")
        return self.cur.shape[1]

    def skip(self, n):
        """Pass over the next ``n`` rows; False when the files run out first."""
        while n > 0 and self._fill():
            m = min(n, self.cur.shape[0] - self.pos)
            self.pos += m
            n -= m
        return n == 0

    def take(self, n):
        """The next ``n`` rows as one fp32 CPU tensor (fewer when the files run out)."""
        parts = []
        while n > 0 and self._fill():
            m = min(n, self.cur.shape[0] - self.pos)
            parts.append(self.cur[self.pos:self.pos + m])
            self.pos += m
            n -= m
        if not parts:
            return torch.empty(0, self.cur.shape[1] if self.cur is not None else 0)
        return parts[0] if len(parts) == 1 else torch.cat(parts)


def pooled_width(d1, d2, pooling):
    if pooling == "concat":
        return d1 + d2
    if d1 != d2:
        raise ValueError(f"{pooling} pooling needs the two models' widths to agree, got {d1} and {d2}")
    return d1


def pool_queries(q1, q2, weight, pooling):
    """The reference's fp32 query pooling (weight on model 2's queries)."""
    if pooling == "concat":
        return torch.cat([q1, weight * q2], dim=-1)
    if pooling == "mean":
        return (q1 + weight * q2) / (1.0 + weight)
    return q1 + weight * q2


def pool_passages(p1, p2, pooling):
    """The reference's fp32 passage pooling (no weight)."""
    if pooling == "concat":
        return torch.cat([p1, p2], dim=-1)
    if pooling == "mean":
        return (p1 + p2) / 2.0
    return p1 + p2


def _take_exactly(stream, n, model):
    x = stream.take(n)
    if x.shape[0] != n:
        raise ValueError(f"model {model} has fewer passage vectors than the passage file has passages")
    return x


def _not_fp16(x):
    return ~(x.abs() <= ops.FP16_MAX).all()          # also true for NaN


def build_pooled_segment(s1, s2, rows, pooling, device):
    """fp16 [rows, d] device store of the next ``rows`` passages of the two streams, pooled chunk by chunk."""
    d1, d2 = s1.width, s2.width
    store = torch.empty(rows, pooled_width(d1, d2, pooling), dtype=torch.float16, device=device)
    bad = torch.zeros((), dtype=torch.bool, device=device)
    for r in range(0, rows, CHUNK_ROWS):
        n = min(CHUNK_ROWS, rows - r)
        x1 = _take_exactly(s1, n, 1).to(device)
        x2 = _take_exactly(s2, n, 2).to(device)
        if pooling == "concat":
            bad |= _not_fp16(x1) | _not_fp16(x2)
            store[r:r + n, :d1].copy_(x1)
            store[r:r + n, d1:].copy_(x2)
        else:
            x = pool_passages(x1, x2, pooling)
            bad |= _not_fp16(x)
            store[r:r + n].copy_(x)
        del x1, x2
    if bool(bad):
        raise ValueError(f"a pooled passage vector value does not fit fp16 (|x| > {ops.FP16_MAX:g} or not finite)")
    return store


def save_pooled_passages(paths_1, paths_2, n_rows, pooling, output_dir):
    """The pooled passages in fp32 as the reference's 8 ``reps_000{i}.pkl`` files of ``n_rows // 8 + 1`` rows."""
    s1, s2 = RepsRows(paths_1), RepsRows(paths_2)
    dim = pooled_width(s1.width, s2.width, pooling)
    per = n_rows // SAVED_SHARDS + 1
    for i in range(SAVED_SHARDS):
        writer = StreamingTensorPickle(os.path.join(output_dir, f"reps_000{i}.pkl"), dim)
        left = max(0, min(per, n_rows - i * per))
        while left:
            n = min(CHUNK_ROWS, left)
            writer.append(pool_passages(_take_exactly(s1, n, 1), _take_exactly(s2, n, 2), pooling).contiguous())
            left -= n
        writer.close()


# ------------------------------------------------------------------ search
def _init_distributed():
    """The rank under torchrun (NCCL, one GPU per rank), 0 otherwise."""
    if "LOCAL_RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    return dist.get_rank() if rr._world() > 1 else 0


def search_pooled(queries, paths_1, paths_2, n_rows, pooling, topk, shard=1, device="cuda"):
    """(scores fp32 [Q, k], passage rows int64 [Q, k]) of the pooled queries over the pooled store; every rank builds
    and searches its own block of rows in ``shard`` segments and gets the global result."""
    if not (queries.abs() <= ops.FP16_MAX).all():
        raise ValueError(f"a pooled query vector value does not fit fp16 (|x| > {ops.FP16_MAX:g} or not finite)")
    world = rr._world()
    rank = dist.get_rank() if world > 1 else 0
    lo, hi = n_rows * rank // world, n_rows * (rank + 1) // world
    s1, s2 = RepsRows(paths_1), RepsRows(paths_2)
    if not (s1.skip(lo) and s2.skip(lo)):
        raise ValueError("a model has fewer passage vectors than the passage file has passages")
    bounds = [lo + (hi - lo) * j // shard for j in range(shard + 1)]
    loaders = [lambda n=b - a: build_pooled_segment(s1, s2, n, pooling, device) for a, b in zip(bounds, bounds[1:])]
    s, i, rows = rr.search_loaded(queries, loaders, topk)
    if rank == world - 1 and (s1.take(1).shape[0] or s2.take(1).shape[0]):
        raise ValueError("the reps_* files hold more passage vectors than the passage file has passages")
    return rr.merge_ranks(s, i, rows, topk)


def run_spar_retrieval(args):
    pooling, weights = check_args(args)
    print("loading questions...")
    questions_list = [load_jsonl(p) for p in args.jsonl_dataset_paths]
    print("loading passages...")
    passages = rr.Passages(args.tsv_passages_path)
    n_rows = len(passages)
    paths_1, paths_2 = reps_paths(args.model_1_emb_dir), reps_paths(args.model_2_emb_dir)
    q_list = []
    for questions, name, weight in zip(questions_list, args.query_reps_filenames, weights):
        q1 = load_tensor(os.path.join(args.model_1_emb_dir, name))
        q2 = load_tensor(os.path.join(args.model_2_emb_dir, name))
        if not len(q1) == len(q2) == len(questions):
            raise ValueError(f"{name}: {len(q1)} and {len(q2)} query vectors for {len(questions)} questions")
        pooled_width(q1.shape[1], q2.shape[1], pooling)
        q_list.append(pool_queries(q1, q2, weight, pooling))
    rank = _init_distributed()
    os.makedirs(args.output_dir, exist_ok=True)
    if args.save_embeddings and rank == 0:
        for q, name in zip(q_list, args.query_reps_filenames):
            with open(os.path.join(args.output_dir, name), "wb") as f:
                pickle.dump(q, f, protocol=4)
        save_pooled_passages(paths_1, paths_2, n_rows, pooling, args.output_dir)
    print("searching...")
    scores, rows = search_pooled(torch.cat(q_list), paths_1, paths_2, n_rows, pooling, args.topk, args.shard,
                                 args.device)
    if rank != 0:
        return
    scores = scores.float().cpu().numpy().astype(np.float64)
    rows = rows.cpu().numpy()
    start = 0
    for questions, pred in zip(questions_list, args.pred_filenames):
        end = start + len(questions)
        questions = [dict(q, id=q.get("id", str(i))) for i, q in enumerate(questions)]
        path = os.path.join(args.output_dir, pred)
        print("writing results to", path)
        rr.write_run(path, passages, questions, scores[start:end], rows[start:end], trec_format=False)
        start = end


def main(argv=None):
    return run_spar_retrieval(get_parser().parse_args(argv))


if __name__ == "__main__":
    main()
