"""COIL / CITADEL retrieval from an expert index on the H100 (dprb_expert_search through ExpertIndex):

  * the kernel against the float64 oracle (oracle/multivec_retrieval.py) on synthetic indexes: P in {8, 32, 128,
    1024}, with and without CLS vectors, a dominant expert, runs longer than one tile, experts absent from the queries,
    queries with no matching expert, passages absent from every posting list, k in {1, 100, 1024}, N up to 200 000.
    Every returned score is within the derived fp16 bound of the oracle's score of that passage; ids equal the
    oracle's wherever the oracle's gaps around a rank exceed twice the bound;
  * repeatability: two runs bitwise equal; a query's results do not change with the other queries of its batch or
    with the query-block split;
  * the device-side refusals: a payload that does not fit fp16, topk above N, sums beyond the fixed-point range.
"""
import numpy as np
import pytest
import torch

from oracle import multivec_retrieval as orc

pytestmark = pytest.mark.gpu


def synth(N, P, V, n_entries, Q, seed, Pc=None, dominant=False, long_runs=False, absent_rows=0, q_entries=16,
          scale=0.25):
    """(index arrays, query arrays) of a synthetic CITADEL-shaped problem.  Experts V-4.. never occur in the index;
    the last ``absent_rows`` passages are in no posting list; query 0 only holds experts without postings."""
    rng = np.random.default_rng(seed)
    ex = rng.zipf(1.3, n_entries) % (V - 4)
    if dominant:
        ex[rng.random(n_entries) < 0.5] = 3
    rows = rng.integers(0, N - absent_rows, n_entries)
    if long_runs:                                   # one passage holds 300 (and one 150) entries of one expert
        ex[:300], rows[:300] = 1, 5
        ex[300:450], rows[300:450] = 1, 9
    pay = (rng.standard_normal((n_entries, P)) * scale).astype(np.float32)
    cls = (rng.standard_normal((N, Pc)) * scale).astype(np.float32) if Pc else None
    qn = rng.integers(1, 2 * q_entries, Q)
    q_seq = np.repeat(np.arange(Q), qn)
    q_ex = rng.zipf(1.3, q_seq.size) % (V - 4)
    if long_runs:
        q_ex[::3] = 1
    q_ex[q_seq == 0] = V - 2                        # no matching expert
    q_pay = (rng.standard_normal((q_seq.size, P)) * scale).astype(np.float32)
    q_cls = (rng.standard_normal((Q, Pc)) * scale).astype(np.float32) if Pc else None
    ids = np.arange(N, dtype=np.int64) * 3 + 7
    return (ex, rows, pay, ids, cls), (q_ex, q_seq, q_pay, q_cls)


def _oracle(index, queries, Q):
    ex, rows, pay, ids, cls = index
    q_ex, q_seq, q_pay, q_cls = queries
    N = ids.size
    entries = {}
    order = np.lexsort((rows, ex))
    exs, rs, ps = ex[order], rows[order], pay[order].astype(np.float64)
    starts = np.flatnonzero(np.r_[True, exs[1:] != exs[:-1]])
    for lo, hi in zip(starts, np.r_[starts[1:], exs.size]):
        entries[int(exs[lo])] = (rs[lo:hi], ps[lo:hi])
    qd = [dict() for _ in range(Q)]
    for x, s, u in zip(q_ex.tolist(), q_seq.tolist(), q_pay.astype(np.float64)):
        qd[s].setdefault(x, []).append(u)
    return orc.scores(entries, qd, N, None if cls is None else cls.astype(np.float64),
                      None if q_cls is None else q_cls.astype(np.float64))


def _search(idx, queries, Q, k, subset=None):
    q_ex, q_seq, q_pay, q_cls = queries
    if subset is not None:                          # a batch of some of the queries, renumbered
        keep = np.isin(q_seq, subset)
        remap = {q: i for i, q in enumerate(subset)}
        q_ex, q_pay = q_ex[keep], q_pay[keep]
        q_seq = np.array([remap[q] for q in q_seq[keep].tolist()], dtype=np.int64)
        q_cls = None if q_cls is None else q_cls[subset]
        Q = len(subset)
    order = np.lexsort((q_seq, q_ex))
    return idx.search(torch.from_numpy(q_ex[order]), torch.from_numpy(q_seq[order]),
                      torch.from_numpy(q_pay[order]).cuda(), None if q_cls is None else torch.from_numpy(q_cls).cuda(),
                      Q, k)


def _index(index, V):
    from dpr_scale_b200.task.citadel_retrieval_task import ExpertIndex
    ex, rows, pay, ids, cls = index
    return ExpertIndex(ex, rows, torch.from_numpy(pay), ids, None if cls is None else torch.from_numpy(cls), V, "cuda")


def check_against_oracle(got_s, got_ids, S, B, ids, k):
    rows = (got_ids - 7) // 3
    assert np.array_equal(rows * 3 + 7, got_ids) and rows.min() >= 0
    es, er = orc.topk(S, k + 1)
    matched = 0
    for q in range(S.shape[0]):
        assert len(set(rows[q].tolist())) == k, "a passage is returned twice"
        err = np.abs(got_s[q].astype(np.float64) - S[q, rows[q]])
        assert (err <= B[q, rows[q]]).all(), f"query {q}: score error {err.max():.3e} above the bound"
        b2 = 2 * B[q].max()
        for i in range(k):
            sep_prev = i == 0 or es[q, i - 1] - es[q, i] > b2
            sep_next = es[q, i] - es[q, i + 1] > b2
            if sep_prev and sep_next:
                assert rows[q, i] == er[q, i], f"query {q} rank {i}: row {rows[q, i]} vs oracle {er[q, i]}"
                matched += 1
    return matched


CASES = [  # (N, P, Pc, V, entries, Q, k, flags)
    (2000, 8, None, 200, 20000, 9, 100, ""),
    (5000, 32, 128, 30522, 200000, 17, 100, "dominant"),
    (3000, 128, 64, 500, 30000, 70, 1, "long"),
    (1500, 1024, None, 100, 6000, 5, 1024, "absent"),
    (200000, 32, 128, 30522, 1600000, 8, 1024, ""),
    (4000, 32, None, 64, 60000, 130, 100, "long_dominant"),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N{}_P{}_Pc{}_V{}_k{}_{}".format(c[0], c[1], c[2], c[3], c[6],
                                                                                        c[7] or "plain"))
def test_search_matches_oracle(case):
    N, P, Pc, V, n_entries, Q, k, flags = case
    index, queries = synth(N, P, V, n_entries, Q, seed=N + P, Pc=Pc, dominant="dominant" in flags,
                           long_runs="long" in flags, absent_rows=N // 10 if "absent" in flags else 0)
    idx = _index(index, V)
    with torch.no_grad():
        s, i = _search(idx, queries, Q, k)
    S, B = _oracle(index, queries, Q)
    matched = check_against_oracle(s, i, S, B, index[3], k)
    assert matched > 0, "no separated ranks to compare ids"
    print(f"{case}: {idx.tile_bounds.numel() - 1} tiles, {matched} of {Q * k} ranks separated and equal")


def test_repeatable_and_batch_independent():
    from dpr_scale_b200 import ops
    N, P, Pc, V, Q, k = 20000, 32, 128, 1000, 40, 50
    index, queries = synth(N, P, V, 300000, Q, seed=3, Pc=Pc, dominant=True, long_runs=True)
    idx = _index(index, V)
    with torch.no_grad():
        a = _search(idx, queries, Q, k)
        b = _search(idx, queries, Q, k)
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
        sub = [31, 2, 17, 5]
        c = _search(idx, queries, Q, k, subset=sub)
        assert np.array_equal(c[0].view(np.uint32), a[0][sub].view(np.uint32)) and np.array_equal(c[1], a[1][sub])
        orig = ops.expert_search_block_queries
        ops.expert_search_block_queries = lambda n: 7              # seven queries per block
        try:
            d = _search(idx, queries, Q, k)
        finally:
            ops.expert_search_block_queries = orig
        assert np.array_equal(d[0].view(np.uint32), a[0].view(np.uint32)) and np.array_equal(d[1], a[1])


def test_index_refusals_on_device():
    from dpr_scale_b200.task.citadel_retrieval_task import ExpertIndex
    ex, rows = np.array([1, 2]), np.array([0, 1])
    with pytest.raises(ValueError, match="fp16"):
        ExpertIndex(ex, rows, torch.tensor([[1e5] * 8, [0.0] * 8]), np.arange(2), None, 4, "cuda")
    idx = ExpertIndex(ex, rows, torch.full((2, 8), 6e4), np.arange(2), None, 4, "cuda")
    with pytest.raises(ValueError, match="topk"):
        idx.search(np.array([1]), np.array([0]), torch.ones(1, 8).cuda(), None, 1, 3)
    with pytest.raises(ValueError, match="fixed-point"):
        idx.search(np.array([1]), np.array([0]), torch.full((1, 8), 6e4).cuda(), None, 1, 1)


def test_exact_ties_go_to_the_lower_row():
    """equal scores on the device: three passages with identical entries, then every other passage at exactly 0"""
    from dpr_scale_b200.task.citadel_retrieval_task import ExpertIndex
    N, P = 1000, 16
    v = np.full((1, P), 0.5, np.float32)
    ex = np.array([5, 5, 5, 9])
    rows = np.array([3, 7, 500, 900])
    pay = np.concatenate([v, v, v, -v])
    idx = ExpertIndex(ex, rows, torch.from_numpy(pay), np.arange(N) + 1000, None, 16, "cuda")
    q_ex, q_seq = np.array([5, 9, 11]), np.array([0, 0, 1])          # query 1: no expert with postings
    q_pay = torch.from_numpy(np.concatenate([v, v, v])).cuda()
    with torch.no_grad():
        s, i = idx.search(q_ex, q_seq, q_pay, None, 2, 10)
    assert (i[0] - 1000).tolist() == [3, 7, 500, 0, 1, 2, 4, 5, 6, 8]
    assert s[0, 0] == s[0, 1] == s[0, 2] == np.float32(0.25 * P) and (s[0, 3:] == 0).all()
    assert (i[1] - 1000).tolist() == list(range(10)) and (s[1] == 0).all()


# ---- the task end to end on tiny encoders, against the oracle and the unmodified reference's recorded query entries
import os  # noqa: E402

from tests import multivec_cases, multivec_index_cases as icases  # noqa: E402
from tests.util import GOLDEN  # noqa: E402

RETRIEVAL = {"coil_bert": ("coil_bert", 1, False), "coil_bert_cls": ("coil_bert", 1, True),
             "citadel_bert_k1_cls": ("citadel_bert", 1, True), "citadel_bert_k2": ("citadel_bert", 2, False)}
PASSAGE_IDS = list(range(100, 107))


def _tasks(tmp_path, case, topk_out=5):
    from dpr_scale_b200.task.citadel_eval_task import GenerateMultiVecEmbeddingsTask
    from dpr_scale_b200.task.citadel_retrieval_task import CITADELRetrievalTask
    enc, topk, add_cls = RETRIEVAL[case]
    mdir = multivec_cases.model_dir(str(tmp_path / "model"), enc)
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)

    def kw():
        k = icases.task_kwargs(enc, mdir, topk, add_cls)
        k["model"]["_target_"] = "dpr_scale_b200.models.citadel_models." + \
            multivec_cases.TARGETS[multivec_cases.TINY[enc][0]]
        return k
    idx = str(tmp_path / "idx")
    gen = GenerateMultiVecEmbeddingsTask(ctx_embeddings_dir=idx, checkpoint_path=ckpt, add_context_id=False, **kw())
    gen.setup("test")
    gen.cuda()
    outs = []
    with torch.no_grad():
        for i, (toks, ids) in enumerate(icases.batches(enc, seed=5)):
            outs.append(gen.test_step({"contexts_ids": {k: v.cuda() for k, v in toks.items()}, "corpus_ids": ids}, i))
        gen.test_epoch_end(outs)
    table = tmp_path / "passages.tsv"
    table.write_text("id\ttext\ttitle\n" + "".join(f"{i}\tpassage text {i}\ttitle {i}\n" for i in PASSAGE_IDS))
    task = CITADELRetrievalTask(ctx_embeddings_dir=idx, checkpoint_path=ckpt, passages=str(table),
                                output_path=str(tmp_path / "run"), topk=topk_out, **kw())
    task.setup("test")
    task.cuda()
    return task, idx


@pytest.mark.parametrize("case", list(RETRIEVAL))
def test_task_end_to_end_matches_oracle_and_reference(tmp_path, case):
    enc, _, add_cls = RETRIEVAL[case]
    G = np.load(os.path.join(GOLDEN, "multivec_retrieval_small.npz"))
    task, idx = _tasks(tmp_path, case)
    entries, cls = orc.read_index(idx, PASSAGE_IDS)
    outs, want = [], []
    with torch.no_grad():
        for i, (toks, ids) in enumerate(icases.batches(enc, seed=6)):
            toks = {k: v.cuda() for k, v in toks.items()}
            expert, seq, payload, q_cls = task.query_entries(toks)
            n = toks["input_ids"].shape[0]
            qd = [dict() for _ in range(n)]
            for x, q, u in zip(expert.tolist(), seq.tolist(), payload.double().cpu().numpy()):
                qd[q].setdefault(x, []).append(u)
            # the query entries against the reference's _eval_step (COIL: no routing, so every entry)
            if enc.startswith("coil"):
                for j in range(n):
                    assert sorted(qd[j]) == sorted(G[f"{case}/q{i}/{j}/experts"].tolist())
                    for x in qd[j]:
                        ref = G[f"{case}/q{i}/{j}/x{x}/repr"]
                        assert np.abs(np.stack(qd[j][x]) - ref).max() <= 2.0 ** -7 * max(1e-30, np.abs(ref).max())
            S, B = orc.scores(entries, qd, len(PASSAGE_IDS), cls,
                              q_cls.double().cpu().numpy() if add_cls else None)
            want.append((S, B, ids))
            outs.append(task.test_step({"query_ids": toks, "topic_ids": ids}, i))
        path = task.test_epoch_end(outs)
    lines = open(path).read().splitlines()
    k = 5
    got = {}
    for ln in lines:
        t, q0, doc, rank, score, tag = ln.split()
        assert q0 == "Q0" and tag == "dpr-scale"
        got.setdefault(t, []).append((int(doc), int(rank), float(score)))
    for S, B, ids in want:
        es, er = orc.topk(S, k + 1)
        for j, t in enumerate(ids):
            rows = [PASSAGE_IDS.index(d) for d, _, _ in got[t]]
            assert [r for _, r, _ in got[t]] == list(range(1, k + 1))
            for r, (d, _, sc) in zip(rows, got[t]):
                assert abs(sc - S[j, r]) <= B[j, r] + 5e-7
            b2 = 2 * B[j].max()
            for p in range(k):
                if (p == 0 or es[j, p - 1] - es[j, p] > b2) and es[j, p] - es[j, p + 1] > b2:
                    assert rows[p] == er[j, p]


def test_task_refuses_grad_and_colbert(tmp_path):
    task, _ = _tasks(tmp_path, "coil_bert")
    toks = {k: v.cuda() for k, v in icases.batches("coil_bert", seed=6)[0][0].items()}
    with pytest.raises(ValueError, match="no_grad"):
        task.query_entries(toks)

    class ColBERTLike(torch.nn.Module):
        pass
    task.query_encoder = ColBERTLike()
    with torch.no_grad(), pytest.raises(ValueError, match="COIL or CITADEL"):
        task.query_entries(toks)
