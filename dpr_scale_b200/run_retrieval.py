#!/usr/bin/env python3
"""Brute-force retrieval over the ``reps_*`` files written by GenerateEmbeddingsTask - the GPU counterpart of
/root/reference/dpr_scale/run_retrieval_pytorch.py (same command line, same output files).

What changes under the hood:
  * search_index (:141-176) is ONE fused kernel pass per 1024 queries (ops.search_topk: wgmma scoring with a
    running top-k); the [batch, N] fp16 score matrix and the torch.topk passes over it are gone, so ``--batch`` no
    longer bounds memory (it is accepted and ignored).
  * an index segment is held in HBM as fp16 exactly like build_index (:178-190); with 80 GB per GPU the 21 M x 768
    Wikipedia index (32 GB) is one segment.  ``--shard`` still splits the reps_* files into sequential segments and
    the per-segment lists are merged on the GPU (ops.topk_merge, replacing :210-230 / :272-277).
  * scores are rounded to fp16 before they are written, because the reference's scores are fp16 einsum outputs;
    ``--fp32_scores`` keeps the fp32-accumulated values instead.

Under torchrun the index is sharded over the ranks (each GPU searches the reps_* block it owns; one all-gather of the
[Q, k] lists; merge) - see search_distributed.  There is no CPU path: without the CUDA library the ops raise DprbError.
"""
import argparse
import functools
import glob
import json
import logging
import os
import pathlib
import pickle

import numpy as np
import torch
import torch.distributed as dist

from . import ops
from .datamodule.dpr import CSVDataset, QueryCSVDataset, QueryTSVDataset


def get_logger():
    logging.basicConfig(format="[%(asctime)s] [%(levelname)s]: %(message)s", level=logging.INFO)
    return logging.getLogger(__name__)


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--ctx_embeddings_dir", type=str, default="")
    p.add_argument("--query_emb_path", type=str, default="",
                   help="if left empty, will use <ctx_embeddings_dir>/query_reps.pkl")
    p.add_argument("--questions_tsv_path", type=str, default="")
    p.add_argument("--passages_tsv_path", type=str, default="")
    p.add_argument("--output_runfile_path", type=str, default="")
    p.add_argument("--topk", type=int, default=100)
    p.add_argument("--batch", type=int, default=100, help="accepted for compatibility; the fused search ignores it")
    p.add_argument("--shard", type=int, default=1)
    p.add_argument("--trec_format", action="store_true")
    p.add_argument("--run_name", type=str, default="dpr")
    p.add_argument("--ignore_identical_ids", action="store_true",
                   help="this is used for BEIR Arguana and Quora datasets")
    p.add_argument("--fp32_scores", action="store_true", help="write fp32 scores instead of fp16-rounded ones")
    p.add_argument("--reference_ranking", action="store_true",
                   help="rank by the fp16-ROUNDED score like the reference's topk over its fp16 einsum "
                        "(run_retrieval_pytorch.py:150-151): ids equal the reference's wherever its fp16 scores are "
                        "distinct.  Default: rank by the exact fp32-accumulated score (finer, deterministic order)")
    p.add_argument("--device", type=str, default="cuda", help="device holding the index (the kernels need CUDA)")
    return p


# ------------------------------------------------------------------ tab-separated inputs (datamodule/dpr.py:80-159)
Passages = CSVDataset            # id / text / title table with a header row


def Questions(path, trec_format):
    """question \\t answers (QueryCSVDataset) or, for trec, qid \\t question (QueryTSVDataset)."""
    return QueryTSVDataset(path) if trec_format else QueryCSVDataset(path)


# ------------------------------------------------------------------ search
def build_index(paths, device="cuda"):
    """fp16 index segment in HBM from reps_* pickles (build_index, run_retrieval_pytorch.py:178-190)."""
    parts = []
    for fname in paths:
        with open(fname, "rb") as f:
            vector = torch.as_tensor(pickle.load(f))
        parts.append(vector.to(device=device, dtype=torch.float16, non_blocking=True))
        print(f"Adding {tuple(vector.shape)} vectors from {fname}")
    return torch.cat(parts, dim=0) if len(parts) > 1 else parts[0].contiguous()


def search_index(query_embs, corpus_embs, batch, topk, index_offset=0, reference_ranking=False):
    """(scores [Q, k] fp32, row ids [Q, k] int64) on the GPU; argument meaning as run_retrieval_pytorch.py:141."""
    del batch
    q = torch.as_tensor(query_embs).to(device=corpus_embs.device, dtype=corpus_embs.dtype).contiguous()
    return ops.search_topk(q, corpus_embs, topk, index_offset=index_offset, reference_ranking=reference_ranking)


def search_loaded(q_repr, loaders, topk, reference_ranking=False):
    """Search index segments in row order, each built by its loader only when its turn comes (one segment in HBM at a
    time), and merge the lists -> (scores, row ids counted from the first segment's first row, rows searched)."""
    all_s, all_i, rows = [], [], 0
    for load in loaders:
        index = load()
        s, i = search_index(q_repr, index, None, topk, index_offset=rows, reference_ranking=reference_ranking)
        rows += index.shape[0]
        del index
        all_s.append(s)
        all_i.append(i)
    if len(all_s) == 1:
        return all_s[0], all_i[0], rows
    s, i = ops.topk_merge(torch.cat(all_s, dim=1).contiguous(), torch.cat(all_i, dim=1).contiguous(), topk)
    return s, i, rows


def _segment_loaders(input_paths, shard, device):
    assert len(input_paths) % shard == 0, "Invalid Shard number"
    per = len(input_paths) // shard
    return [functools.partial(build_index, input_paths[seg * per:(seg + 1) * per], device) for seg in range(shard)]


def search_segments(q_repr, input_paths, shard, batch, topk, device="cuda", reference_ranking=False):
    """Search ``shard`` sequential index segments and merge (run_retrieval_pytorch.py:204-230, :272-277)."""
    del batch
    s, i, _ = search_loaded(q_repr, _segment_loaders(input_paths, shard, device), topk, reference_ranking)
    return s, i


# ------------------------------------------------------------------ multi-GPU: index sharded over ranks
def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank_files(input_paths, rank, world):
    """Contiguous block of reps_* files owned by ``rank`` (file order = global row order = passage-file order)."""
    assert len(input_paths) % world == 0, f"{len(input_paths)} reps_* files do not divide over {world} ranks"
    per = len(input_paths) // world
    return input_paths[rank * per:(rank + 1) * per]


def global_row_offset(local_rows, device):
    """Rows held by the lower ranks (one all-gather of a single int64 per rank)."""
    world = _world()
    if world == 1:
        return 0
    mine = torch.tensor([int(local_rows)], dtype=torch.int64, device=device)
    every = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(every, mine)
    return int(sum(int(t.item()) for t in every[:dist.get_rank()]))


def gather_rank_lists(scores, indexes):
    """[Q, k] per rank -> [Q, W * k], rank-major along dim 1: the layout of all_scores / all_indexes in
    run_retrieval_pytorch.py:218-227 with ranks in place of sequential shards."""
    world = _world()
    if world == 1:
        return scores, indexes
    ss = [torch.empty_like(scores) for _ in range(world)]
    ii = [torch.empty_like(indexes) for _ in range(world)]
    dist.all_gather(ss, scores.contiguous())
    dist.all_gather(ii, indexes.contiguous())
    return torch.cat(ss, dim=1).contiguous(), torch.cat(ii, dim=1).contiguous()


def merge_ranks(scores, indexes, rows, topk):
    """Every rank's [Q, k] lists over its own ``rows`` -> the global top-k on every rank: rank-local row ids are
    shifted by the rows of the lower ranks, then one all-gather and ops.topk_merge."""
    if _world() == 1:
        return scores, indexes
    indexes = indexes + global_row_offset(rows, scores.device)
    gs, gi = gather_rank_lists(scores, indexes)
    return ops.topk_merge(gs, gi, topk)


def search_distributed(q_repr, input_paths, shard, batch, topk, device="cuda", reference_ranking=False):
    """Every rank searches its own block of the index (the reps_{rank} files it wrote in generate_embeddings) and
    the W lists are merged with one all-gather + ops.topk_merge; every rank returns the global result.  The only
    data-path collective is that all-gather of [Q, k] scores and ids (no corpus bytes move between GPUs)."""
    world = _world()
    if world == 1:
        return search_segments(q_repr, input_paths, shard, batch, topk, device, reference_ranking)
    mine = rank_files(input_paths, dist.get_rank(), world)
    s, i, rows = search_loaded(q_repr, _segment_loaders(mine, shard, device), topk, reference_ranking)
    return merge_ranks(s, i, rows, topk)


# ------------------------------------------------------------------ output (merge_results :96-137, writer :232-300)
def merge_results(passages, questions, top_doc_ids, scores_list, trec_format):
    assert len(top_doc_ids) == len(questions) == len(scores_list)
    merged = []
    for i, (question, doc_ids, scores) in enumerate(zip(questions, top_doc_ids, scores_list)):
        ctxs = []
        for doc, score in zip(doc_ids, scores):
            try:
                row = passages[doc]
                if trec_format:
                    ctxs.append({"id": row["id"], "score": float(score)})
                else:
                    ctxs.append({"id": row["id"], "title": row["title"], "text": row["text"], "score": float(score)})
            except (KeyError, IndexError, TypeError):
                if not trec_format:
                    raise
                continue                          # BEIR files contain empty lines; the reference skips them
        merged.append({"question": question["question"], "answers": question.get("answers", []), "ctxs": ctxs,
                       "id": question.get("id", i)})
    return merged


def write_run(path, passages, questions, scores, indexes, trec_format, run_name="dpr", ignore_identical_ids=False):
    pathlib.Path(path).parent.mkdir(parents=True, exist_ok=True)
    with open(path, "w") as g:
        results = merge_results(passages, questions, indexes, scores, trec_format)
        if not trec_format:
            g.write(json.dumps(results, indent=4))
            g.write("\n")
            return
        for result in results:
            for rank, ctx in enumerate(result["ctxs"], start=1):
                if ignore_identical_ids and result["id"] == ctx["id"]:
                    continue
                g.write("{} Q0 {} {} {} {}\n".format(result["id"], ctx["id"], rank, ctx["score"], run_name))


def main(args, logger=None):
    logger = logger or get_logger()
    logger.info(args.__dict__)
    input_paths = sorted(glob.glob(os.path.join(args.ctx_embeddings_dir, "reps_*")))
    assert input_paths, f"no reps_* files under {args.ctx_embeddings_dir}"
    qpath = args.query_emb_path or os.path.join(args.ctx_embeddings_dir, "query_reps.pkl")
    print("Loading question vectors.")
    with open(qpath, "rb") as f:
        q_repr = torch.as_tensor(pickle.load(f))
    print("Retrieving results...")
    if "LOCAL_RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl")
    scores, indexes = search_distributed(q_repr, input_paths, args.shard, args.batch, args.topk, args.device,
                                         getattr(args, "reference_ranking", False))
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
