"""Shared inputs of the SPAR goldens (tests/golden/make_golden_spar.py) and the tests that compare against them: the
question and passage fixtures, and the two models' passage and query embeddings drawn from seeded generators (so the
golden stores outputs only)."""
import csv
import hashlib
import json
import os
import pickle

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
QUESTIONS = os.path.join(HERE, "golden", "data", "spar_questions.jsonl")
PASSAGES = os.path.join(HERE, "golden", "data", "spar_passages.tsv")
N_PASSAGES = 300
N_QUESTIONS = 24
DIM = 32
# each model's reps_* files split the passages differently, so the two streams do not line up file by file
SPLITS = {1: [120, 100, 80], 2: [170, 130]}
SEEDS = {1: 71, 2: 72}
QUERY_FILES = {"query_reps_a.pkl": 0, "query_reps_b.pkl": 1}
# (pooling, per-dataset weights) of the spar_retrieval goldens; the datasets are QUESTIONS twice, with the query files
# above in that order
RETRIEVAL_CASES = [("concat", [0.5, 2.0]), ("mean", [0.7, 1.0]), ("sum", [1.5, 0.3])]
TOPK = 100
EVAL_KS = [1, 5, 20, 100]
# tune_spar_weights goldens: (regex, eval_on_ks, valid_on_k); default weight grid
TUNE_CASES = [(False, [1, 5, 10, 20, 50, 100], 100), (True, [1, 5, 10, 20, 50, 100], 10)]
PRED_FILE = "nq_dev.json"
EVAL_RUN = "concat_a.json"     # the retrieval run eval_dpr's goldens evaluate
# the golden keeps every run's ids; all scores of EVAL_RUN, the models' own runs and these weights' tuned runs, and the
# first SCORE_RANKS ranks' scores of the others
TUNE_FULL_SCORES = (0.1, 1.0, 10.0)
SCORE_RANKS = 10


def sha256(data):
    """Hex digest of a text or of an array's bytes (how the golden pins files and tensors it does not store)."""
    raw = data.encode() if isinstance(data, str) else np.ascontiguousarray(data).tobytes()
    return hashlib.sha256(raw).hexdigest()


def load_passages():
    """The passage table's rows as ``{"id", "title", "text"}`` dicts in file order (ids are 1 .. N_PASSAGES)."""
    with open(PASSAGES, newline="") as f:
        rows = list(csv.reader(f, delimiter="\t"))
    col = {name: i for i, name in enumerate(rows[0])}
    return [{"id": r[col["id"]], "title": r[col["title"]], "text": r[col["text"]]} for r in rows[1:]]


def load_questions():
    with open(QUESTIONS) as f:
        return [json.loads(line) for line in f]


def run_text(ids, scores):
    """The text of a run over QUESTIONS in the reference's layout (``json.dump(..., indent=4)`` of question,
    answers, ctxs of id / title / text / score, and id) from its passage ids and fp32 scores ([questions, k]).  The
    golden keeps runs as these two arrays; its generator checks that this rebuilds the reference's files byte for
    byte."""
    passages = load_passages()
    out = []
    for i, (q, row_ids, row_scores) in enumerate(zip(load_questions(), ids, scores)):
        ctxs = [{"id": passages[j - 1]["id"], "title": passages[j - 1]["title"], "text": passages[j - 1]["text"],
                 "score": float(s)} for j, s in zip(row_ids.tolist(), np.asarray(row_scores, np.float32))]
        out.append({"question": q["question"], "answers": q.get("answers", []), "ctxs": ctxs,
                    "id": q.get("id", str(i))})
    return json.dumps(out, indent=4)


def model_vectors(model):
    """(passage vectors [N_PASSAGES, DIM], {query file: [N_QUESTIONS, DIM]}) of model 1 or 2, fp32."""
    g = torch.Generator().manual_seed(SEEDS[model])
    p = torch.randn(N_PASSAGES, DIM, generator=g)
    qs = {}
    for name, j in QUERY_FILES.items():
        qs[name] = torch.randn(N_QUESTIONS, DIM, generator=g) * (1.0 + 0.5 * j)
    return p, qs


def write_model_dir(path, model):
    """reps_XXXX.pkl (split as SPLITS[model]) and the query pickles of one model under ``path``."""
    os.makedirs(path, exist_ok=True)
    p, qs = model_vectors(model)
    start = 0
    for i, n in enumerate(SPLITS[model]):
        with open(os.path.join(path, f"reps_{i:04}.pkl"), "wb") as f:
            pickle.dump(p[start:start + n].clone(), f, protocol=4)
        start += n
    for name, q in qs.items():
        with open(os.path.join(path, name), "wb") as f:
            pickle.dump(q, f, protocol=4)
    return str(path)


def pooled_float64(pooling, weight, query_file):
    """float64 pooled (queries [N_QUESTIONS, d], passages [N_PASSAGES, d]) of the two models, pooled in fp32 as the
    reference does."""
    from dpr_scale_b200.spar_retrieval import pool_passages, pool_queries
    p1, q1 = model_vectors(1)
    p2, q2 = model_vectors(2)
    return (pool_queries(q1[query_file], q2[query_file], weight, pooling).double(),
            pool_passages(p1, p2, pooling).double())


def fp16_bound(q, p):
    """Per query: a bound on |fp16-store score - exact score| over every passage, from rounding both operands to fp16
    (relative 2^-11 each) and fp32 accumulation."""
    return (q.abs() @ p.abs().T).max(dim=1).values * (2.0 ** -10 + 2.0 ** -20) + 1e-6


def check_ranking(got_rows, got_scores, q, p, golden_rows=None, min_separated=0.2):
    """got_rows / golden_rows: [Q, k] passage rows (0-based).  Against the exact float64 order: scores within the fp16
    bound, and rows equal wherever the exact score gap to both neighbours exceeds twice that bound."""
    exact = q @ p.T
    bound = fp16_bound(q, p)
    k = got_rows.shape[1]
    s, order = torch.sort(exact, dim=1, descending=True, stable=True)
    got_rows, got_scores = torch.as_tensor(got_rows), torch.as_tensor(got_scores, dtype=torch.float64)
    assert (torch.gather(exact, 1, got_rows) - got_scores).abs().le(bound[:, None]).all()
    gaps = s[:, :-1] - s[:, 1:]
    inf = torch.full((s.shape[0], 1), float("inf"), dtype=s.dtype)
    sep = torch.minimum(torch.cat([inf, gaps], 1), torch.cat([gaps, inf], 1))[:, :k] > 2 * bound[:, None]
    assert sep.float().mean() > min_separated, f"only {float(sep.float().mean()):.2f} of the positions are separated"
    assert torch.equal(got_rows[sep], order[:, :k][sep])
    if golden_rows is not None:
        assert torch.equal(torch.as_tensor(golden_rows)[sep], order[:, :k][sep])


def golden_run_text(gold, key):
    """The text of a run the golden keeps with all its scores."""
    return run_text(gold[key + "/ids"], gold[key + "/scores"])


def write_golden_preds(gold, dirs):
    """Each model's own run (the reference's dense_search output) into its embedding directory, as tuning reads it."""
    for m, d in zip((1, 2), dirs):
        with open(os.path.join(d, PRED_FILE), "w") as f:
            f.write(golden_run_text(gold, f"tune/pred_{m}"))


def check_tuned_runs(gold, out_dir, weights):
    """Every ``weight{w}_`` run under ``out_dir`` against the golden: the reference's layout, ids, titles and texts
    exactly; scores within fp32 summation-order tolerance wherever the golden keeps them."""
    for w in weights:
        key = f"tune/weight{w}_{PRED_FILE}"
        with open(os.path.join(out_dir, f"weight{w}_{PRED_FILE}")) as f:
            run = json.load(f)
        ids = np.asarray([[int(c["id"]) for c in q["ctxs"]] for q in run])
        scores = np.asarray([[c["score"] for c in q["ctxs"]] for q in run])
        assert np.array_equal(ids, gold[key + "/ids"]), w
        kept = gold[key + "/scores"]
        np.testing.assert_allclose(scores[:, :kept.shape[1]], kept, rtol=1e-5, atol=1e-5)
        want = json.loads(run_text(gold[key + "/ids"], np.zeros(ids.shape, np.float32)))
        for q in run:
            for c in q["ctxs"]:
                c["score"] = 0.0
        assert json.dumps(run) == json.dumps(want), w


def check_saved(gold, path, name):
    """A pickle spar_retrieval --save_embeddings wrote, bit for bit against the reference's."""
    with open(path, "rb") as f:
        t = pickle.load(f).numpy()
    assert list(t.shape) == gold[f"saved/{name}/shape"].tolist() and sha256(t) == str(gold[f"saved/{name}/sha256"]), name
