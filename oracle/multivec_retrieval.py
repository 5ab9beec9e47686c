"""Float64 exhaustive scorer for retrieval from a COIL / CITADEL expert index (dpr_scale_b200.task.citadel_retrieval_task).

  score(q, d) = cls_q . cls_d                                               (only with CLS vectors)
              + sum over q's entries (x, u) of max(0, max over d's index entries (x, v) of u . v)    (max over {} = 0)

Ranking: descending score, ties towards the lower passage row.  ``bound`` gives, per (query, row), the error the
device's roundings can make: fp16 operands (2 * 2^-11 relative on every product, plus their product), fp32 accumulation
of a width-P dot product (P * 2^-24 relative of the sum of |products|), the 2^-32 fixed point of every term and the
final fp32 score (2^-24 relative).  Because max and the clamp are 1-Lipschitz, the error of a term is at most that of
its worst product sum; the bound sums those worst sums over the query's entries.
"""
import glob
import os
import pickle

import numpy as np


def read_index(ctx_embeddings_dir, passage_ids):
    """expert -> (rows int64 [n] sorted, payload float64 [n, P]) from ``expert_*/{expert}.pkl`` (shards in rank
    order) and the CLS vectors float64 [N, Pc] from ``cls_*.pkl`` (None without them)."""
    row_of = {int(p): i for i, p in enumerate(passage_ids)}
    entries = {}
    for shard in sorted(glob.glob(os.path.join(ctx_embeddings_dir, "expert_*"))):
        for name in os.listdir(shard):
            x = int(name[:-4])
            with open(os.path.join(shard, name), "rb") as f:
                ids, _w, pay = pickle.load(f)
            rows = np.array([row_of[int(i)] for i in ids.tolist()], dtype=np.int64)
            entries.setdefault(x, []).append((rows, pay.double().numpy()))
    out = {}
    for x, parts in entries.items():
        rows = np.concatenate([p[0] for p in parts])
        pay = np.concatenate([p[1] for p in parts])
        o = np.argsort(rows, kind="stable")
        out[x] = (rows[o], pay[o])
    cls_files = sorted(glob.glob(os.path.join(ctx_embeddings_dir, "cls_*.pkl")))
    cls = None
    if cls_files:
        parts = []
        for path in cls_files:
            with open(path, "rb") as f:
                parts.append(pickle.load(f).double().numpy())
        cls = np.concatenate(parts)
    return out, cls


def _run_max(rows, vals, N):
    """max of vals per row (rows sorted); -inf where a row has no value"""
    m = np.full(N, -np.inf)
    if rows.size:
        starts = np.flatnonzero(np.r_[True, rows[1:] != rows[:-1]])
        m[rows[starts]] = np.maximum.reduceat(vals, starts)
    return m


def scores(entries, queries, N, cls=None, q_cls=None):
    """entries: expert -> (rows sorted, payload [n, P]); queries: one dict per query, expert -> list of payload vectors
    [P]; cls [N, Pc] / q_cls [Q, Pc] or None.  Returns (score float64 [Q, N], bound float64 [Q, N])."""
    Q = len(queries)
    S = np.zeros((Q, N))
    A = np.zeros((Q, N))
    terms = np.zeros(Q)
    P = 0
    for q, qd in enumerate(queries):
        for x, us in qd.items():
            for u in us:
                u = np.asarray(u, dtype=np.float64).reshape(-1)
                P = u.size
                terms[q] += 1
                if x not in entries:
                    continue
                rows, pay = entries[x]
                m = _run_max(rows, pay @ u, N)
                S[q] += np.where(np.isfinite(m), np.maximum(m, 0.0), 0.0)
                a = _run_max(rows, np.abs(pay) @ np.abs(u), N)
                A[q] += np.where(np.isfinite(a), a, 0.0) * (2.0 ** -10 + 2.0 ** -21 + P * 2.0 ** -24)
    if cls is not None:
        qc = np.asarray(q_cls, dtype=np.float64)
        S += qc @ cls.T
        A += (np.abs(qc) @ np.abs(cls).T) * (2.0 ** -10 + 2.0 ** -21 + cls.shape[1] * 2.0 ** -24)
        terms += 1
    bound = A + (terms[:, None] + 1) * 2.0 ** -32 + np.abs(S) * 2.0 ** -23
    return S, bound


def topk(S, k):
    """(scores [Q, k], rows [Q, k]): descending, ties towards the lower row."""
    rows = np.empty((S.shape[0], k), dtype=np.int64)
    for q in range(S.shape[0]):
        rows[q] = np.lexsort((np.arange(S.shape[1]), -S[q]))[:k]
    return np.take_along_axis(S, rows, 1), rows
