"""float64 restatement of SPLADE first-stage retrieval (dpr_scale_b200.splade_retrieval / dprb_sparse_search) from CSR
inputs: score(q, d) = sum over the terms both hold of w_q * w_d, with the passage weights rounded to fp16 exactly as the
index stores them, then the k best rows per query, descending, ties towards the lower row."""
import numpy as np


def dense(offsets, terms, weights, V, fp16=False):
    """[N, V] float64 of a CSR matrix (a term repeated in a row adds up); fp16: round the weights to fp16 first."""
    offsets = np.asarray(offsets, dtype=np.int64)
    w = np.asarray(weights)
    w = (w.astype(np.float16) if fp16 else w).astype(np.float64)
    out = np.zeros((offsets.size - 1, V))
    rows = np.repeat(np.arange(offsets.size - 1), np.diff(offsets))
    np.add.at(out, (rows, np.asarray(terms, dtype=np.int64)), w)
    return out


def scores(index, queries, V):
    """float64 [Q, N] and the products' magnitudes [Q, N] (sum of |w_q w_d|): index / queries = (offsets, terms,
    weights) CSR triples."""
    P = dense(*index, V, fp16=True)
    Qm = dense(*queries, V)
    return Qm @ P.T, np.abs(Qm) @ np.abs(P).T


def topk(S, k):
    """(scores [Q, k], rows [Q, k]) descending, ties towards the lower row."""
    rows = np.argsort(-S, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(S, rows, 1), rows
