"""SPLADE first-stage retrieval on the H100 (dprb_sparse_search through SparseIndex):

  * the kernel against float64 (oracle/sparse_retrieval.py) on Zipf-distributed indexes with posting lists of several
    tiles, queries with repeated terms, empty queries and empty passages, k in {1, 100, 1024}, and query counts across
    the block boundary.  Every score is within nnz_q 2^-32 plus the fp32 rounding of the products and of the sum; ids
    equal the oracle's wherever the float64 gaps around a rank exceed twice that bound;
  * repeatability: two runs are byte-identical, and a query's results do not depend on the query-block split;
  * end to end: tiny BERT and RoBERTa SPLADE checkpoints -> GenerateSparseEmbeddingsTask /
    GenerateSparseQueryEmbeddingsTask -> ``python -m dpr_scale_b200.splade_retrieval``, against a float64 dense top-k
    of the oracle's SPLADE vectors;
  * two NCCL ranks give the run file of one rank (skipped with fewer than 2 GPUs).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from dpr_scale_b200 import ops
from oracle import sparse_retrieval as osr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def synth(N, V, per_row, Q, per_query, seed, empty_rows=True):
    """(index CSR, query CSR): Zipf terms, unique inside a passage, repeated terms in queries; query 0 and every 5th
    passage are empty."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(N), rng.integers(1, 2 * per_row, N))
    terms = (rng.zipf(1.25, rows.size) - 1) % V
    key = np.unique(rows.astype(np.int64) * V + terms)
    rows, terms = key // V, key % V
    if empty_rows:
        keep = rows % 5 != 3
        rows, terms = rows[keep], terms[keep]
    offsets = np.r_[0, np.cumsum(np.bincount(rows, minlength=N))]
    weights = (rng.random(terms.size) * 3).astype(np.float32)
    qn = rng.integers(1, 2 * per_query, Q)
    qn[0] = 0
    q_off = np.r_[0, np.cumsum(qn)]
    q_terms = (rng.zipf(1.25, q_off[-1]) - 1) % V
    q_terms[1::4] = q_terms[::4][:q_terms[1::4].size]                 # repeated terms
    q_w = (rng.random(q_terms.size) * 2).astype(np.float32)
    return (offsets, terms, weights), (q_off, q_terms, q_w)


def oracle_rows(index, queries, V):
    """Per query: float64 scores [N] and the products' magnitudes [N] (through a CSC of the fp16-rounded index)."""
    off, t, w = index
    N = off.size - 1
    rows = np.repeat(np.arange(N), np.diff(off))
    P = sp.csc_matrix((w.astype(np.float16).astype(np.float64), (rows, t)), shape=(N, V))
    q_off, q_t, q_w = queries
    for q in range(q_off.size - 1):
        a, b = q_off[q], q_off[q + 1]
        if a == b:
            yield np.zeros(N), np.zeros(N), 0
            continue
        cols = P[:, q_t[a:b]]
        wq = q_w[a:b].astype(np.float64)
        yield cols @ wq, abs(cols) @ np.abs(wq), b - a


def check(index, queries, V, k, s, i):
    s, i = s.cpu().numpy(), i.cpu().numpy()
    matched = 0
    for q, (S, M, nq) in enumerate(oracle_rows(index, queries, V)):
        B = nq * 2.0 ** -32 + 2.0 ** -24 * (M + np.abs(S))
        assert len(set(i[q].tolist())) == k, f"query {q}: a passage is returned twice"
        err = np.abs(s[q].astype(np.float64) - S[i[q]])
        assert (err <= B[i[q]]).all(), f"query {q}: score error {err.max():.3e} above the bound"
        order = np.argsort(-S, kind="stable")[:k + 1]
        es = S[order]
        b2 = 2 * B.max()
        for r in range(k):
            if (r == 0 or es[r - 1] - es[r] > b2) and es[r] - es[r + 1] > b2:
                assert i[q, r] == order[r], f"query {q} rank {r}: row {i[q, r]} vs float64 {order[r]}"
                matched += 1
        if nq == 0:
            assert i[q].tolist() == list(range(k)) and (s[q] == 0).all()
    return matched


def _index(index, V):
    from dpr_scale_b200.splade_retrieval import SparseIndex
    return SparseIndex(*index, V, device="cuda")


CASES = [  # (N, V, per passage, Q, per query, k, queries per block or None)
    (20000, 30522, 60, 40, 25, 100, None),
    (50000, 2000, 30, 30, 12, 1024, 7),
    (3000, 500, 20, 25, 10, 1, 4),
    (1_000_000, 30522, 20, 270, 25, 100, None),     # 268 queries per block: a second block of 2
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"N{c[0]}_V{c[1]}_Q{c[3]}_k{c[5]}_Qb{c[6]}")
def test_search_matches_float64(case, monkeypatch):
    N, V, per_row, Q, per_query, k, qb = case
    index, queries = synth(N, V, per_row, Q, per_query, seed=N + k)
    idx = _index(index, V)
    lengths = np.diff(idx.term_ptr_host)
    assert lengths.max() > 4 * ops.SPARSE_SEARCH_TILE or N < 10000, "no posting list spans several tiles"
    if qb is not None:
        monkeypatch.setattr(ops, "sparse_search_block_queries", lambda n: qb)
    else:
        assert N < 500_000 or ops.sparse_search_block_queries(N) < Q, "the queries do not cross a block boundary"
    s, i = idx.search(*queries, k)
    matched = check(index, queries, V, k, s, i)
    assert matched > 0
    print(f"{case}: nnz {idx.nnz}, longest list {lengths.max()}, {matched} of {Q * k} ranks separated and equal")


def test_repeatable_and_block_independent(monkeypatch):
    V = 30522
    index, queries = synth(100000, V, 60, 60, 25, seed=9)
    idx = _index(index, V)
    a = idx.search(*queries, 200)
    b = idx.search(*queries, 200)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])
    monkeypatch.setattr(ops, "sparse_search_block_queries", lambda n: 7)
    c = idx.search(*queries, 200)
    assert torch.equal(a[0].view(torch.int32), c[0].view(torch.int32)) and torch.equal(a[1], c[1])


def test_exact_ties_go_to_the_lower_row():
    from dpr_scale_b200.splade_retrieval import SparseIndex
    idx = SparseIndex([0, 1, 1, 2, 3, 3], [4, 4, 4], [0.5, 0.5, 0.5], 8, ids=np.arange(5) + 10, device="cuda")
    s, i = idx.search([0, 1], [4], [2.0], 5)
    assert i.tolist() == [[10, 12, 13, 11, 14]] and s.tolist() == [[1.0, 1.0, 1.0, 0.0, 0.0]]


# ---- end to end: tiny SPLADE checkpoints -> sparse embeddings -> splade_retrieval
def _tokens(cfg, n, seed):
    from tests import splade_cases
    return splade_cases.tiny_tokens(cfg, S=20, n=n, seed=seed)


def _generate(tmp_path, name):
    from dpr_scale_b200.task.splade_index_task import GenerateSparseEmbeddingsTask, GenerateSparseQueryEmbeddingsTask
    from tests import colbert_cases, splade_cases
    kind, _ = splade_cases.TINY[name]
    cfg = colbert_cases.encoder_config(kind)
    mdir = splade_cases.tiny_model_dir(str(tmp_path / "model"), name)
    sd_q, sd_c = splade_cases.tiny_state_dict(name), splade_cases.tiny_state_dict(name, 100)
    ckpt = str(tmp_path / "task.ckpt")
    state = {"query_encoder." + k: v for k, v in sd_q.items()}
    state.update({"context_encoder." + k: v for k, v in sd_c.items()})
    torch.save({"state_dict": state}, ckpt)
    kw = dict(transform={}, datamodule=None, optim={}, shared_model=False,
              model={"_target_": "dpr_scale_b200.models.citadel_models.splade_model.SPLADEEncoder",
                     "model_path": mdir, "dropout": 0.1})
    idx = str(tmp_path / "idx")
    passages = [_tokens(cfg, 6, 30), _tokens(cfg, 5, 31)]             # each batch ends with an empty passage
    gen = GenerateSparseEmbeddingsTask(ctx_embeddings_dir=idx, checkpoint_path=ckpt, **kw)
    gen.setup("test")
    gen.cuda()
    for j, t in enumerate(passages):
        gen.test_step({"contexts_ids": {k: v.cuda() for k, v in t.items()}}, j)
    gen.test_epoch_end([])
    queries = _tokens(cfg, 4, 32)
    qgen = GenerateSparseQueryEmbeddingsTask(ctx_embeddings_dir=idx, checkpoint_path=ckpt, **kw)
    qgen.setup("test")
    qgen.cuda()
    qgen.test_step({"query_ids": {k: v.cuda() for k, v in queries.items()}, "topic_ids": ["q0", "q1", "q2", "q3"]}, 0)
    qgen.test_epoch_end([])
    return idx, (sd_q, sd_c, kind), passages, queries


def _tables(tmp_path, n):
    p = tmp_path / "passages.tsv"
    p.write_text("id\ttext\ttitle\n" + "".join(f"{100 + i}\tpassage {i}\ttitle {i}\n" for i in range(n)))
    q = tmp_path / "queries.tsv"
    q.write_text("".join(f"q{i}\tquestion {i}\n" for i in range(4)))
    return str(p), str(q)


def _args(idx, p, q, out, k):
    return ["--ctx_embeddings_dir", idx, "--passages_tsv_path", p, "--questions_tsv_path", q,
            "--output_runfile_path", out, "--topk", str(k), "--trec_format", "--fp32_scores"]


def _run(path):
    got = {}
    for ln in open(path).read().splitlines():
        t, q0, doc, rank, score, tag = ln.split()
        got.setdefault(t, []).append((int(doc), int(rank), float(score)))
    return got


@pytest.mark.parametrize("name", ["splade_bert", "splade_roberta"])
def test_end_to_end_matches_float64_dense(tmp_path, name):
    from dpr_scale_b200 import splade_retrieval
    from dpr_scale_b200.utils.csr_writer import load_csr
    from oracle import splade as osp
    from tests import rerank_cases
    idx, (sd_q, sd_c, kind), passages, queries = _generate(tmp_path, name)
    ocfg = rerank_cases.ORACLE_CFG[kind]
    P = torch.cat([osp.reps(sd_c, ocfg, t) for t in passages]).double().numpy()
    Qv = osp.reps(sd_q, ocfg, queries).double().numpy()
    assert sorted(os.listdir(idx)) == ["sparse_0000.pkl", "sparse_query.pkl"]
    d = load_csr(os.path.join(idx, "sparse_0000.pkl"))
    assert d["offsets"].size == 12 and d["V"] == P.shape[1] and d["weights"].dtype == np.float16
    assert d["offsets"][6] == d["offsets"][5] and d["offsets"][11] == d["offsets"][10]    # the empty passages
    assert load_csr(os.path.join(idx, "sparse_query.pkl"))["topic_ids"] == ["q0", "q1", "q2", "q3"]
    p, q = _tables(tmp_path, 11)
    k = 8
    out = str(tmp_path / "run.trec")
    splade_retrieval.main(splade_retrieval.get_parser().parse_args(_args(idx, p, q, out, k)))
    got = _run(out)
    S = Qv @ P.T
    # encoder deviation: each SPLADE weight within 2^-7 of its row's largest (test_splade_gpu's gate), twice over
    tol = 2 * 2.0 ** -7 * (np.abs(Qv).max(1, keepdims=True) * np.abs(P).sum(1)[None, :] +
                           np.abs(Qv).sum(1, keepdims=True) * np.abs(P).max(1)[None, :]) + 1e-6
    for j in range(4):
        rows = [doc - 100 for doc, _, _ in got[f"q{j}"]]
        assert [r for _, r, _ in got[f"q{j}"]] == list(range(1, k + 1))
        for r, (_, _, sc) in zip(rows, got[f"q{j}"]):
            assert abs(sc - S[j, r]) <= tol[j, r], (j, r, sc, S[j, r])
        order = np.argsort(-S[j], kind="stable")
        t2 = 2 * tol[j].max()
        for r in range(k):
            if (r == 0 or S[j, order[r - 1]] - S[j, order[r]] > t2) and S[j, order[r]] - S[j, order[r + 1]] > t2:
                assert rows[r] == order[r], (j, r)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_match_one_rank(tmp_path):
    from dpr_scale_b200.utils.csr_writer import StreamingCSRPickle
    V = 3000
    index, queries = synth(40000, V, 40, 30, 20, seed=77)
    idx = tmp_path / "idx"
    idx.mkdir()
    off, t, w = index
    for r, (a, b) in enumerate(((0, 17001), (17001, 40000))):                 # unequal shards
        wr = StreamingCSRPickle(str(idx / f"sparse_{r:04}.pkl"), V, np.float16)
        wr.append(np.diff(off[a:b + 1]), t[off[a]:off[b]].astype(np.int32), w[off[a]:off[b]].astype(np.float16))
        wr.close()
    q_off, q_t, q_w = queries
    wr = StreamingCSRPickle(str(idx / "sparse_query.pkl"), V, np.float32)
    wr.append(np.diff(q_off), q_t.astype(np.int32), q_w)
    wr.close()
    p = tmp_path / "passages.tsv"
    p.write_text("id\ttext\ttitle\n" + "".join(f"{i}\tp\tt\n" for i in range(40000)))
    q = tmp_path / "queries.tsv"
    q.write_text("".join(f"q{i}\tquestion\n" for i in range(30)))
    env = dict(os.environ, PYTHONPATH=ROOT)
    outs = []
    for nproc in (1, 2):
        out = str(tmp_path / f"run{nproc}.trec")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m",
               "dpr_scale_b200.splade_retrieval"] + _args(str(idx), str(p), str(q), out, 100)
        subprocess.run(cmd, check=True, cwd=ROOT, env=env, timeout=600)
        outs.append(open(out).read())
    assert outs[0] == outs[1] and len(outs[0].splitlines()) == 30 * 100
