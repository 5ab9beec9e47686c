"""Pieces shared by the bi-encoder rerank tasks (RerankDenseRetrieverTask, RerankMultiVecRetrieverTask): the per-batch
query dedupe and the three pickles a rank writes."""
import os
import pickle

import torch
import torch.distributed as dist


def distinct_queries(qids, q_tok, dedupe=True):
    """(query tokens, index int32 [n]): with ``dedupe`` the tokens of each distinct qid of the batch once (first
    occurrence order) and, for every row, the position of its query among them; without, every row's own tokens.
    Rows are encoded independently at the batch's padded width, so either way a row's query encodes the same."""
    n = len(qids)
    index = list(range(n))
    if dedupe:
        first, rows = {}, []
        for i, q in enumerate(qids):
            if q not in first:
                first[q] = len(rows)
                rows.append(i)
            index[i] = first[q]
        if len(rows) < n:
            q_tok = {k: v[torch.tensor(rows, device=v.device)] for k, v in q_tok.items()}
    return q_tok, torch.tensor(index, dtype=torch.int32)


def write_rerank_pickles(output_dir, rank, test_outputs):
    """``scores_/qids_/ctx_ids_{rank:04}.pkl`` (pickle protocol 4: an fp32 CPU tensor [n] and two lists) from the
    [qids, ctx_ids, scores] of every test step, then a barrier when a process group is up (rank 0 merges only once
    every shard is on disk).  Returns the scores file."""
    qids, ctx_ids, scores = [], [], []
    for b_qids, b_ctx_ids, b_scores in test_outputs:
        qids.extend(b_qids)
        ctx_ids.extend(b_ctx_ids)
        scores.append(b_scores)
    scores = torch.cat(scores, dim=0) if scores else torch.zeros(0, dtype=torch.float32)
    out = {what: os.path.join(output_dir, f"{what}_{rank:04}.pkl") for what in ("scores", "qids", "ctx_ids")}
    print(f"\nWriting scores to {out['scores']}")
    for what, obj in (("scores", scores), ("qids", qids), ("ctx_ids", ctx_ids)):
        with open(out[what], "wb") as f:
            pickle.dump(obj, f, protocol=4)
    if dist.is_available() and dist.is_initialized():
        dist.barrier()
    return out["scores"]
