#!/usr/bin/env python3
"""Top-k answer accuracy of a retrieval run in the NQ-style JSON layout (``question``, ``answers``, ``ctxs`` of
``id`` / ``title`` / ``text`` / ``score``), with the command line and results of the reference's
``dpr_scale/eval_dpr.py``:

  python -m dpr_scale_b200.eval_dpr --retrieval run.json --topk 1 5 20 100 [--regex] [--output_eval_results out.json]

A context contains an answer when, after NFD normalisation of both strings,
  * (default) the answer's token sequence occurs in the context's token sequence.  Tokens are maximal runs of
    letters, numbers and marks, or any other single character that is neither a separator nor a control character,
    compared lower-cased;
  * (``--regex``) the answer, read as a Python regular expression, matches somewhere in the context
    case-insensitively; a pattern that does not compile matches nothing.
For each question the first of its top max(k) contexts that contains an answer decides: accuracy@k is 1 when that
context is among the first k, else 0.  With ``--output_eval_results`` every context looked at gets ``has_answer``
and the run is written back augmented.
"""
import argparse
import json
import re
import unicodedata

import numpy as np
import regex as uregex

# letters/numbers/marks runs, or one character that is not a separator (Z) or control (C) character
_TOKEN = uregex.compile(r"[\p{L}\p{N}\p{M}]+|[^\p{Z}\p{C}]",
                        flags=uregex.IGNORECASE | uregex.UNICODE | uregex.MULTILINE)


def tokens(text):
    """Lower-cased tokens of ``text`` (already normalised)."""
    return [m.group().lower() for m in _TOKEN.finditer(text)]


def _nfd(text):
    return unicodedata.normalize("NFD", text)


def _regex_found(text, pattern):
    try:
        compiled = re.compile(pattern, flags=re.IGNORECASE | re.UNICODE | re.MULTILINE)
    except Exception:
        return False
    return compiled.search(text) is not None


def _contains(seq, sub):
    n = len(sub)
    if n == 0:
        return True
    first = sub[0]
    return any(seq[i] == first and seq[i:i + n] == sub for i in range(len(seq) - n + 1))


def has_answers(text, answers, regex=False):
    """True when ``text`` contains one of ``answers`` under the matching rule above."""
    text = _nfd(text)
    if regex:
        return any(_regex_found(text, _nfd(a)) for a in answers)
    words = tokens(text)
    return any(_contains(words, tokens(_nfd(a))) for a in answers)


def first_answer_rank(flags, max_k):
    """Index of the first True among the first ``max_k`` flags, ``max_k`` when there is none."""
    for i, f in enumerate(flags[:max_k]):
        if f:
            return i
    return max_k


def accuracy_lists(first_ranks, topk):
    """{k: [0 or 1 per question]} from each question's first answer rank."""
    return {k: [0 if r >= k else 1 for r in first_ranks] for k in topk}


def print_accuracy(path, accuracy):
    print("Evaluating", path)
    for k, acc in accuracy.items():
        print(f"Top{k}\taccuracy: {np.mean(acc)}")


def evaluate_retrieval(retrieval_file, topk, regex=False, oufname=""):
    """Per-k accuracy lists of the run in ``retrieval_file``; with ``oufname``, also writes the run with
    ``has_answer`` on each of the top max(k) contexts."""
    with open(retrieval_file) as f:
        retrieval = json.load(f)
    max_k = max(topk)
    first = []
    for question in retrieval:
        answers = question["answers"]
        rank = max_k
        for idx, ctx in enumerate(question["ctxs"][:max_k]):
            found = has_answers(ctx["text"], answers, regex)
            if oufname:
                ctx["has_answer"] = found
            if found:
                rank = min(rank, idx)
                if not oufname:
                    break
        first.append(rank)
    accuracy = accuracy_lists(first, topk)
    print_accuracy(retrieval_file, accuracy)
    if oufname:
        with open(oufname, "w") as f:
            json.dump(retrieval, f, indent=4)
    return accuracy


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--retrieval", type=str, metavar="path", help="Path to retrieval output file.")
    p.add_argument("--topk", type=int, nargs="+", help="topk to evaluate")
    p.add_argument("--regex", action="store_true", default=False, help="regex match")
    p.add_argument("--output_eval_results", type=str, default="",
                   help="if not empty, the run augmented with a has_answer field per context is written here")
    return p


def main(argv=None):
    args = get_parser().parse_args(argv)
    return evaluate_retrieval(args.retrieval, args.topk, args.regex, args.output_eval_results)


if __name__ == "__main__":
    main()
