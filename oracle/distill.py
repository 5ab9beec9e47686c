"""Restatement of the distillation arithmetic of DPRDistillTask (dpr_scale/task/dpr_distill_task.py): the
``MSELoss(reduction="sum")`` loss and its gradient, the in-batch evaluation scores and the rank metrics, in fp32 (what
the reference computes) and float64 (the exact value the kernels are held to)."""
import numpy as np
import torch


def sqerr(x, t, dtype=torch.float64):
    """(sum (x - t)^2, d/dx = 2 (x - t)) in ``dtype``."""
    diff = x.to(dtype) - t.to(dtype)
    return (diff * diff).sum(), 2 * diff


def eval_scores(query_repr, targets, dtype=torch.float64):
    """[2B, 2B] similarity of every query representation to every target vector (sim_score: q @ t^T)."""
    return query_repr.to(dtype) @ targets.to(dtype).T


def rank_metrics(scores, labels, k=1):
    """(sum of ranks, sum of reciprocal ranks, hits@k) - compute_rank_metrics of the reference: the position of the
    label in a stable descending sort of each row, counted from 1."""
    s = np.asarray(scores, dtype=np.float64)
    rank = mrr = score = 0
    for i, lab in enumerate(np.asarray(labels).tolist()):
        order = np.argsort(-s[i], kind="stable")
        pos = int(np.flatnonzero(order == lab)[0])
        rank += pos + 1
        mrr += 1.0 / (pos + 1)
        score += int(pos < k)
    return rank, mrr, score


def epoch_metrics(outputs, k=1, prefix="valid"):
    """_eval_epoch_end averaging: outputs = [((rank, mrr, score), n_queries, n_targets, loss), ...]."""
    tl = tm = tr = ts = tc = n = 0
    for (rank, mrr, score), nq, nt, loss in outputs:
        tr += rank
        tm += mrr
        n += nq
        tc += nt
        ts += score
        tl += float(loss)
    return {prefix + "_loss": tl / len(outputs), prefix + f"_accuracy@{k}": ts / n, prefix + "_avg_rank": tr / n,
            prefix + "_mrr": tm / n, prefix + "_ctx_count": tc / len(outputs)}
