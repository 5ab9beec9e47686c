#!/usr/bin/env python3
"""Writes tests/golden/spar_small.npz by running the UNMODIFIED reference SPAR tools in the authoring container:

  * ``dpr_scale.eval_dpr.evaluate_retrieval`` on a SPAR run, in token and regex matching modes, with
    ``oufname`` set (the augmented file is pinned by its SHA-256) and without;
  * ``spar.spar_retrieval.run_spar_retrieval`` for concat, mean and sum pooling over two datasets with their own
    weights (tests/spar_cases.py RETRIEVAL_CASES), concat also with ``save_embeddings``;
  * ``dpr_scale.utils.tune_spar_weights.grid_search_weights`` with the default weight grid on each model's own run
    (written by the reference's ``dense_search``), in both matching modes.

Runs are kept as their passage ids and fp32 scores, from which tests/spar_cases.run_text rebuilds each file byte for
byte (checked here for every stored run); the saved pickles and the augmented files are kept as SHA-256 digests.  It
also (re)writes the text fixtures tests/golden/data/spar_questions.jsonl and spar_passages.tsv from a seeded
generator.  The embeddings are drawn from the seeded generators of tests/spar_cases.py, which the tests share.

The reference modules import packages absent here; the generator installs stand-ins before importing them:
``faiss.IndexFlatIP`` as exact fp32 numpy search (scores ``q @ p.T``, descending, ties to the lower row), ``ujson`` as
``json``, ``tqdm.notebook`` as ``tqdm`` and ``p_tqdm.p_map`` as ``map``.  Nothing of the reference is copied here.

Run from the repo root: python tests/golden/make_golden_spar.py
"""
import contextlib
import io
import json
import os
import pickle
import random
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
from tests import spar_cases as C  # noqa: E402

WORDS = ("alpha bravo charlie delta echo foxtrot golf hotel india juliett kilo lima mike november oscar papa quebec "
         "romeo sierra tango uniform victor whiskey xray yankee zulu river stone cloud maple harbor lantern").split()
# (answers, phrases planted in passages): unicode and NFD/NFC forms, punctuation, multi-token, regex-looking answers
ANSWERS = [
    (["Zürich"], ["Zürich", "ZÜRICH", "Zürichsee"]),
    (["café au lait"], ["Café au lait", "cafe au lait"]),
    (["U.S."], ["the U.S. army", "U.S"]),
    (["AT&T"], ["at & t", "AT&T"]),
    (["rock 'n' roll"], ["Rock 'n' Roll", "rock n roll"]),
    (["New York City"], ["new york city", "new york"]),
    (["1969"], ["in 1969,", "1969s"]),
    (["naïve", "naive"], ["Naïve", "naivety"]),
    (["São Paulo"], ["SÃO PAULO", "Sao Paulo"]),
    (["C++"], ["c ++", "C+"]),
    (["well-known"], ["well - known", "wellknown"]),
    (["東京"], ["東京都", "東京"]),
    (["don't"], ["Don't", "dont"]),
    (["paris", "lutetia"], ["PARIS!", "Lutetia's"]),
    (["19[0-9]{2}"], ["1987", "19x2"]),
    (["colou?r"], ["color", "colour", "colr"]),
    (["(unclosed"], ["(unclosed"]),
    (["^alpha"], ["alpha"]),
    (["\\bmaple\\b"], ["maples", "maple"]),
    (["xylophonic quasar"], []),
    (["e=mc²"], ["E=MC²", "e = mc2"]),
    (["mike", "november"], []),
    (["  "], []),
    (["Straße"], ["STRASSE", "straße"]),
]


def write_fixtures():
    rng = random.Random(20261018)
    plants = {}
    for qi, (_, phrases) in enumerate(ANSWERS):
        for ph in phrases:
            for _ in range(rng.randint(1, 4)):
                plants.setdefault(rng.randrange(C.N_PASSAGES), []).append(ph)
    with open(C.PASSAGES, "w") as f:
        f.write("id\ttext\ttitle\n")
        for i in range(C.N_PASSAGES):
            words = [rng.choice(WORDS) for _ in range(rng.randint(12, 30))]
            for ph in plants.get(i, []):
                words.insert(rng.randrange(len(words) + 1), ph)
            text = " ".join(words).replace('"', "'")
            title = " ".join(rng.choice(WORDS) for _ in range(rng.randint(1, 3)))
            f.write(f"{i + 1}\t{text}\t{title}\n")
    assert len(ANSWERS) == C.N_QUESTIONS
    with open(C.QUESTIONS, "w") as f:
        for qi, (answers, _) in enumerate(ANSWERS):
            q = {"question": f"question {qi}: which {rng.choice(WORDS)} {rng.choice(WORDS)}?", "answers": answers}
            if qi % 3 == 0:
                q["id"] = f"q{qi}"
            f.write(json.dumps(q, ensure_ascii=False) + "\n")


def put_run(out, key, path, score_ranks=None):
    """A run file as its passage ids (int16) and fp32 scores ([questions, k]; only the first ``score_ranks`` ranks'
    scores when given), after checking that spar_cases.run_text rebuilds the file byte for byte from them."""
    with open(path) as f:
        text = f.read()
    run = json.loads(text)
    ids = np.asarray([[int(c["id"]) for c in q["ctxs"]] for q in run], np.int16)
    scores = np.asarray([[c["score"] for c in q["ctxs"]] for q in run], np.float32)
    assert C.run_text(ids, scores) == text, f"{path} is not rebuilt exactly from its ids and scores"
    out[key + "/ids"], out[key + "/scores"] = ids, scores[:, :score_ranks]
    return text


def ref_tune_weights(ref_tune):
    """The default weight grid of the reference's grid_search_weights."""
    import inspect
    return inspect.signature(ref_tune.grid_search_weights).parameters["weights"].default


def install_stubs():
    faiss = types.ModuleType("faiss")

    class IndexFlatIP:
        def __init__(self, d):
            self.d, self.xb = d, np.zeros((0, d), np.float32)

        def add(self, x):
            self.xb = np.concatenate([self.xb, np.asarray(x, np.float32)])

        def search(self, q, k):
            s = np.asarray(q, np.float32) @ self.xb.T
            order = np.argsort(-s, axis=1, kind="stable")[:, :k]
            return np.take_along_axis(s, order, 1), order
    faiss.IndexFlatIP = IndexFlatIP
    sys.modules["faiss"] = faiss
    sys.modules["ujson"] = json
    import tqdm
    tn = types.ModuleType("tqdm.notebook")
    tn.tqdm = tqdm.tqdm
    sys.modules["tqdm.notebook"] = tn
    pt = types.ModuleType("p_tqdm")
    pt.p_map = lambda f, *a, **k: list(map(f, *a))
    sys.modules["p_tqdm"] = pt
    sys.path.insert(0, REF)
    sys.path.insert(0, os.path.join(REF, "spar"))


def main():
    write_fixtures()
    install_stubs()
    import spar_retrieval as ref_spar
    from dpr_scale import eval_dpr as ref_eval
    from dpr_scale.utils import tune_spar_weights as ref_tune
    out = {}
    tmp = tempfile.mkdtemp(prefix="spar_golden_")
    try:
        dirs = {m: C.write_model_dir(os.path.join(tmp, f"m{m}"), m) for m in (1, 2)}
        names = list(C.QUERY_FILES)
        for pooling, weights in C.RETRIEVAL_CASES:
            od = os.path.join(tmp, f"out_{pooling}")
            preds = [f"{pooling}_a.json", f"{pooling}_b.json"]
            ref_spar.run_spar_retrieval([C.QUESTIONS, C.QUESTIONS], C.PASSAGES, dirs[1], dirs[2], od, preds,
                                        query_emb_names=names, weights=weights, save_embeddings=pooling == "concat",
                                        topk=C.TOPK, pooling=pooling)
            for p in preds:
                put_run(out, f"retrieval/{p}", os.path.join(od, p), None if p == C.EVAL_RUN else C.SCORE_RANKS)
            if pooling == "concat":
                for n in [f"reps_000{i}.pkl" for i in range(8)] + names:
                    with open(os.path.join(od, n), "rb") as f:
                        t = pickle.load(f).numpy()
                    out[f"saved/{n}/shape"], out[f"saved/{n}/sha256"] = np.asarray(t.shape), np.asarray(C.sha256(t))
        # eval_dpr on the concat run of dataset a
        run = os.path.join(tmp, "out_concat", C.EVAL_RUN)
        for regex in (False, True):
            tag = "regex" if regex else "tokens"
            aug = os.path.join(tmp, f"eval_{tag}.json")
            acc = ref_eval.evaluate_retrieval(run, C.EVAL_KS, regex, aug)
            plain = ref_eval.evaluate_retrieval(run, C.EVAL_KS, regex)
            assert plain == acc
            for k in C.EVAL_KS:
                out[f"eval/{tag}/top{k}"] = np.asarray(acc[k], np.int64)
            out[f"eval/{tag}/augmented_sha256"] = np.asarray(C.sha256(open(aug).read()))
        # each model's own run: the reference's dense_search over that model's vectors alone
        passages = ref_spar.load_passages_tsv(C.PASSAGES)
        questions = ref_spar.load_test_dataset(C.QUESTIONS)
        for m in (1, 2):
            index = ref_spar.build_index(ref_spar.load_passage_embeddings(dirs[m]))
            q = ref_spar.load_query_embeddings(dirs[m], names[0])
            res = ref_spar.dense_search(questions, q, passages, index, C.TOPK)
            with open(os.path.join(dirs[m], C.PRED_FILE), "w") as f:
                json.dump(res, f, indent=4)
            put_run(out, f"tune/pred_{m}", os.path.join(dirs[m], C.PRED_FILE))
        tune_runs = {}
        for ci, (regex, ks, valid_k) in enumerate(C.TUNE_CASES):
            od = os.path.join(tmp, f"tune{ci}")
            log = io.StringIO()
            with contextlib.redirect_stdout(log):
                ref_tune.grid_search_weights(dirs[1], dirs[2], C.PRED_FILE, names[0], output_dir=od,
                                             eval_on_ks=ks, valid_on_k=valid_k, regex=regex)
            lines = [ln for ln in log.getvalue().splitlines()
                     if ln.startswith(("Accuracy for weight", "Top", "The best weight"))]
            out[f"tune/{ci}/log"] = np.asarray("\n".join(lines))
            best = [ln for ln in lines if ln.startswith("The best weight")][0].split()[4]
            out[f"tune/{ci}/best_weight"] = np.float64(best)
            out[f"tune/{ci}/files"] = np.asarray(sorted(os.listdir(od)))
            for w in ref_tune_weights(ref_tune):       # the runs do not depend on the matching mode: kept once
                fn = f"weight{w}_{C.PRED_FILE}"
                text = open(os.path.join(od, fn)).read()
                if ci == 0:
                    tune_runs[w] = put_run(out, f"tune/{fn}", os.path.join(od, fn),
                                           None if w in C.TUNE_FULL_SCORES else C.SCORE_RANKS)
                assert text == tune_runs[w], fn
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(HERE, "spar_small.npz"), **out)
    print("wrote spar_small.npz", len(out), "entries")


if __name__ == "__main__":
    main()
