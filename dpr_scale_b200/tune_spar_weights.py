#!/usr/bin/env python3
"""Choose SPAR's lexical weight by re-ranking two models' retrieval runs: the command line, output files and log of
the reference's ``dpr_scale/utils/tune_spar_weights.py``.

  python -m dpr_scale_b200.tune_spar_weights --emb_dir_1 dense/ --emb_dir_2 lexical/ --pred_filename nq_dev.json \\
      --query_reps_filename query_reps.pkl --output_dir tuned/ [--weights ...] [--regex] [--valid_on_k 100]

Each ``--emb_dir_*`` holds one model's ``reps_*`` passage pickles, its query pickle and its run ``pred_filename``
(passage ids are 1-based passage rows).  For every question the candidate pool is the union of the two runs' top 100
passages; both models score the pool in fp32 and, for each weight ``w``, the pool is sorted by ``s1 + w * s2`` and its
top 100 are written to ``<output_dir>/weight{w}_{pred_filename}`` (the question entry of run 1 with new ``ctxs``).
Accuracy@k is reported for every weight, and the best weight is the first with the highest accuracy@``valid_on_k``.

How it differs from running the reference: the pool does not depend on the weight, so whether each (question, pool
passage) pair contains an answer is computed once, in parallel host processes, instead of once per weight.  The pool
scores come from rows gathered out of the fp32 pickles (only the rows some pool holds) and are computed on the GPU
in bounded chunks of questions; each weight's ranking and accuracy follow from the scores and the answer flags there.
The order matches the reference's up to the order of summation inside each inner product.
"""
import argparse
import json
import multiprocessing
import os
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

from .eval_dpr import accuracy_lists, has_answers, print_accuracy
from .spar_retrieval import load_tensor, reps_paths

DEFAULT_WEIGHTS = [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0, 1.1, 1.25, 1.43, 1.67, 2, 2.5, 3.33, 5.0, 10.0]
DEFAULT_KS = [1, 5, 10, 20, 50, 100]
TOPK_IN = 100          # passages taken from each model's run
TOPK_OUT = 100         # passages written per question and weight
CHUNK_QUESTIONS = 512  # questions scored per device pass (at most 2 * TOPK_IN rows each)


def read_run(path):
    if not os.path.isfile(path):
        raise FileNotFoundError(f"no such file: {path}")
    with open(path) as f:
        return json.load(f)


def joint_pools(data_1, data_2):
    """Per question: the ascending passage rows (id - 1) of the union of the two runs' top lists, and each pool
    passage's context entry (run 2's where both runs hold it)."""
    pools, ctxs = [], []
    for q1, q2 in zip(data_1, data_2):
        if q1["question"] != q2["question"]:
            raise ValueError(f"the two runs disagree on a question: {q1['question']!r} vs {q2['question']!r}")
        by_id = {c["id"]: c for c in q1["ctxs"][:TOPK_IN]}
        by_id.update({c["id"]: c for c in q2["ctxs"][:TOPK_IN]})
        rows = sorted(int(i) - 1 for i in by_id)
        pools.append(rows)
        ctxs.append([by_id[str(r + 1)] for r in rows])
    return pools, ctxs


def _flags_of(job):
    answers, texts, regex = job
    return [has_answers(t, answers, regex) for t in texts]


def answer_flags(data_1, ctxs, regex, workers=None):
    """has_answers of every (question, pool passage), in pool order, over ``workers`` host processes."""
    jobs = [(q["answers"], [c["text"] for c in cs], regex) for q, cs in zip(data_1, ctxs)]
    workers = workers or os.cpu_count() or 1
    if workers == 1 or len(jobs) < 2 * workers:
        return [_flags_of(j) for j in jobs]
    with ProcessPoolExecutor(workers, mp_context=multiprocessing.get_context("fork")) as ex:
        return list(ex.map(_flags_of, jobs, chunksize=max(1, len(jobs) // (8 * workers))))


def gather_rows(emb_dir, rows):
    """fp32 [len(rows), d] table of the passage vectors at the ascending ``rows``, read one reps_* file at a time."""
    rows = np.asarray(rows, dtype=np.int64)
    parts, start = [], 0
    for path in reps_paths(emb_dir):
        t = load_tensor(path)
        lo, hi = np.searchsorted(rows, [start, start + t.shape[0]])
        parts.append(t[torch.from_numpy(rows[lo:hi] - start)].clone())
        start += t.shape[0]
        del t
    if rows.size and rows[-1] >= start:
        raise ValueError(f"{emb_dir}: a run names passage {rows[-1] + 1} but the reps_* files hold {start} passages")
    return torch.cat(parts)


def score_pools(pools, flags, q1, q2, table_1, table_2, table_rows, weights, max_k, device="cuda"):
    """For each weight: every question's pool sorted by s1 + w * s2 (fp32) -> (order [Q, P] into the pool,
    sorted scores [Q, P], first rank of an answer within the top min(max_k, TOPK_OUT), max_k when there is none [Q]).
    P is the largest pool; shorter pools are padded with -inf scores that sort last."""
    Q, P = len(pools), max(len(p) for p in pools)
    limit = min(max_k, TOPK_OUT)
    order = {w: torch.empty(Q, P, dtype=torch.int64) for w in weights}
    scores = {w: torch.empty(Q, P, dtype=torch.float32) for w in weights}
    first = {w: torch.empty(Q, dtype=torch.int64) for w in weights}
    t1, t2 = table_1.to(device), table_2.to(device)
    for a in range(0, Q, CHUNK_QUESTIONS):
        b = min(Q, a + CHUNK_QUESTIONS)
        n = torch.tensor([len(p) for p in pools[a:b]])
        valid = torch.arange(P)[None, :] < n[:, None]
        idx = torch.zeros(b - a, P, dtype=torch.int64)
        idx[valid] = torch.from_numpy(np.searchsorted(table_rows, np.concatenate([pools[i] for i in range(a, b)])))
        fl = torch.zeros(b - a, P, dtype=torch.bool)
        fl[valid] = torch.tensor([f for i in range(a, b) for f in flags[i]], dtype=torch.bool)
        idx, valid, fl = idx.to(device), valid.to(device), fl.to(device)
        s1 = torch.bmm(t1[idx], q1[a:b].to(device)[:, :, None])[:, :, 0]
        s2 = torch.bmm(t2[idx], q2[a:b].to(device)[:, :, None])[:, :, 0]
        pos = torch.arange(P, device=device)[None, :]
        for w in weights:
            s = (s1 + s2 * w).masked_fill(~valid, float("-inf"))
            s, o = torch.sort(s, dim=1, descending=True, stable=True)
            hit = torch.gather(fl, 1, o) & (pos < limit)
            r = torch.where(hit.any(1), hit.to(torch.int8).argmax(1), torch.full_like(n.to(device), max_k))
            order[w][a:b], scores[w][a:b], first[w][a:b] = o.cpu(), s.cpu(), r.cpu()
    return order, scores, first


def write_weight_run(path, data_1, ctxs, order, scores):
    out = []
    for i, q in enumerate(data_1):
        n = min(len(ctxs[i]), TOPK_OUT)
        ranked = []
        for j, s in zip(order[i, :n].tolist(), scores[i, :n].tolist()):
            c = ctxs[i][j]
            ranked.append({"id": c["id"], "title": c["title"], "text": c["text"], "score": s})
        out.append(dict(q, ctxs=ranked))
    if os.path.dirname(path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=4)


def grid_search_weights(emb_dir_1, emb_dir_2, pred_filename, query_reps_filename, weights=DEFAULT_WEIGHTS,
                        output_dir=None, eval_on_ks=DEFAULT_KS, valid_on_k=100, regex=False, device="cuda",
                        workers=None, timings=None):
    """Re-rank, write one run per weight, report accuracies -> (best weight, its accuracy@valid_on_k,
    {weight: {k: per-question accuracy list}}).  ``timings``, when a dict, receives seconds per stage."""
    if valid_on_k not in eval_on_ks:
        raise ValueError(f"--valid_on_k {valid_on_k} is not among --eval_on_ks {eval_on_ks}")
    if not weights:
        raise ValueError("no weights to try")
    timings = {} if timings is None else timings
    clock = time.perf_counter()

    def lap(name):
        nonlocal clock
        if torch.device(device).type == "cuda":
            torch.cuda.synchronize(device)
        now = time.perf_counter()
        timings[name] = timings.get(name, 0.0) + now - clock
        clock = now

    print("loading predictions...")
    data_1 = read_run(os.path.join(emb_dir_1, pred_filename))
    data_2 = read_run(os.path.join(emb_dir_2, pred_filename))
    q1 = load_tensor(os.path.join(emb_dir_1, query_reps_filename))
    q2 = load_tensor(os.path.join(emb_dir_2, query_reps_filename))
    if not len(data_1) == len(q1) == len(data_2) == len(q2):
        raise ValueError(f"{len(data_1)} and {len(data_2)} questions in the runs, {len(q1)} and {len(q2)} query vectors")
    pools, ctxs = joint_pools(data_1, data_2)
    table_rows = np.unique(np.concatenate([np.asarray(p, dtype=np.int64) for p in pools] or [np.zeros(0, np.int64)]))
    print("loading passage embeddings...")
    table_1, table_2 = gather_rows(emb_dir_1, table_rows), gather_rows(emb_dir_2, table_rows)
    lap("load")
    print("matching answers...")
    flags = answer_flags(data_1, ctxs, regex, workers)
    lap("answer_matching")
    print("performing joint-pool re-ranking...")
    order, scores, first = score_pools(pools, flags, q1, q2, table_1, table_2, table_rows, weights, max(eval_on_ks),
                                       device)
    lap("pool_scoring_and_accuracy")
    output_dir = output_dir or tempfile.mkdtemp(prefix="spar_weights_")
    os.makedirs(output_dir, exist_ok=True)
    best_acc, best_weight, accuracies = -1.0, -1.0, {}
    for w in weights:
        path = os.path.join(output_dir, f"weight{w}_{pred_filename}")
        write_weight_run(path, data_1, ctxs, order[w], scores[w])
        print("Accuracy for weight", w)
        acc = accuracy_lists(first[w].tolist(), eval_on_ks)
        print_accuracy(path, acc)
        accuracies[w] = acc
        acc_k = np.mean(acc[valid_on_k])
        if acc_k > best_acc:
            best_acc, best_weight = acc_k, w
    lap("write")
    print("The best weight is", best_weight, f"with top-{valid_on_k} accuracy of {best_acc}")
    return best_weight, best_acc, accuracies


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--emb_dir_1", type=str, metavar="path", help="Path to embeddings of model 1.")
    p.add_argument("--emb_dir_2", type=str, metavar="path", help="Path to embeddings of model 2.")
    p.add_argument("--pred_filename", type=str)
    p.add_argument("--query_reps_filename", type=str)
    p.add_argument("--weights", type=float, nargs="+", default=DEFAULT_WEIGHTS)
    p.add_argument("--output_dir", type=str)
    p.add_argument("--regex", action="store_true", default=False, help="regex match")
    p.add_argument("--eval_on_ks", type=int, nargs="+", default=DEFAULT_KS, help="topk to evaluate")
    p.add_argument("--valid_on_k", type=int, default=100, help="the k whose accuracy chooses the weight")
    p.add_argument("--device", type=str, default="cuda", help="device that scores the pools")
    return p


def main(argv=None):
    a = get_parser().parse_args(argv)
    return grid_search_weights(a.emb_dir_1, a.emb_dir_2, a.pred_filename, a.query_reps_filename, a.weights,
                               a.output_dir, a.eval_on_ks, a.valid_on_k, a.regex, a.device)


if __name__ == "__main__":
    main()
