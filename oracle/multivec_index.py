"""float64 NumPy restatement of the reference's multi-vector index generation loops:

  passage_index  GenerateMultiVecEmbeddingsTask._eval_step + test_epoch_end (dpr_scale/task/citadel_eval_task.py:43-117):
                 for every passage, unmasked token 1.. and expert slot in order, COIL (2-D expert ids) keeps weight > 0
                 with payload w * rep; CITADEL keeps weight > weight_threshold with payload w * rep, or every slot with
                 the token id as payload under add_context_id; entries are appended per expert across batches.
  query_index    GenerateMultiVecQueryEmbeddingsTask._eval_step (:143-171): per query a dict expert -> payloads
                 (w * rep) and weights; COIL keeps every unmasked token, CITADEL weight > 0.

Inputs are the encoder's outputs as the reference's forward returns them (``expert_repr`` [N, S-1, P], ``expert_ids``
[N, S-1] or [N, S-1, K], ``expert_weights`` of the ids' shape, ``attention_mask`` [N, S-1]) as arrays, plus the
batch's ``input_ids`` [N, S].  Products are taken in float64; the product of two fp32 values is exact there, so the
results rounded to fp32 equal the reference's fp32 products.
"""
import numpy as np


def _entries(out, input_ids, query, add_context_id=False, weight_threshold=0.0):
    """Yield (n, expert, weight, payload) in the reference's iteration order."""
    reps = np.asarray(out["expert_repr"], dtype=np.float64)
    ids = np.asarray(out["expert_ids"])
    w = np.asarray(out["expert_weights"], dtype=np.float64)
    am = np.asarray(out["attention_mask"])
    coil = ids.ndim == 2
    for n in range(ids.shape[0]):
        for s in range(ids.shape[1]):
            if not am[n, s] > 0:
                continue
            if coil:
                if query or w[n, s] > 0:
                    yield n, int(ids[n, s]), w[n, s], w[n, s] * reps[n, s]
                continue
            for x, wx in zip(ids[n, s], w[n, s]):
                if not query and add_context_id:
                    yield n, int(x), wx, np.float64(input_ids[n, s + 1])
                elif wx > (0.0 if query else weight_threshold):
                    yield n, int(x), wx, wx * reps[n, s]


def passage_index(batches, add_context_id=False, weight_threshold=0.0):
    """batches: [(encoder outputs, input_ids, corpus_ids)] -> {expert: (ids int64 [n], weights float64 [n], reprs
    float64 [n, P] or [n])}, entries in the reference's order."""
    acc = {}
    for out, input_ids, corpus_ids in batches:
        for n, x, wx, pay in _entries(out, input_ids, False, add_context_id, weight_threshold):
            acc.setdefault(x, []).append((int(corpus_ids[n]), wx, pay))
    return {x: (np.array([e[0] for e in v], dtype=np.int64), np.array([e[1] for e in v], dtype=np.float64),
                np.stack([np.asarray(e[2]) for e in v]).astype(np.float64)) for x, v in acc.items()}


def query_index(out):
    """One batch's encoder outputs -> (embeddings, weights): per query a dict expert -> list of float64 payloads
    ([P]) and a dict expert -> list of float64 weights."""
    N = np.asarray(out["expert_ids"]).shape[0]
    emb, wts = [dict() for _ in range(N)], [dict() for _ in range(N)]
    for n, x, wx, pay in _entries(out, None, True):
        emb[n].setdefault(x, []).append(np.asarray(pay, dtype=np.float64))
        wts[n].setdefault(x, []).append(np.float64(wx))
    return emb, wts
