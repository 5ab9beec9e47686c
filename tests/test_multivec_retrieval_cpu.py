"""COIL / CITADEL retrieval from an expert index, without a GPU:

  * the float64 oracle (oracle/multivec_retrieval.py) against a direct statement of the score on a small index, the
    tie rule (lower passage row first) and an expert index read back from the files the generation writes;
  * the host side of the search: index tiles never split one passage's entries of an expert and cover every entry
    once, work groups hold <= 64 query entries of one expert and skip experts without postings;
  * the run-file formats (TREC lines and the QA json) equal the reference's format strings;
  * the task config composes;
  * refusals raise ValueError before any GPU work: the options whose behaviour lives in the reference's missing index
    module, shapes outside the kernel limits, an id missing from the passage table, a CLS row count other than N,
    add_cls without CLS files, a payload width other than the encoder's, an add_context_id index.
"""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import multivec_retrieval as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _write_index(tmp, per_rank, cls=None):
    """per_rank: [{expert: (corpus ids, payload [n, P])}]; cls: [rank arrays] or None"""
    for r, experts in enumerate(per_rank):
        d = tmp / f"expert_{r:04}"
        d.mkdir(parents=True)
        for x, (ids, pay) in experts.items():
            pay = torch.as_tensor(pay, dtype=torch.float32)
            with open(d / f"{x}.pkl", "wb") as f:
                pickle.dump((torch.as_tensor(ids, dtype=torch.long), torch.ones(len(ids)), pay), f, protocol=4)
        if cls is not None:
            with open(tmp / f"cls_{r:04}.pkl", "wb") as f:
                pickle.dump(torch.as_tensor(cls[r], dtype=torch.float32), f, protocol=4)


def test_oracle_equals_direct_statement(tmp_path):
    g = np.random.default_rng(0)

    class rng:                                                    # the files hold fp32: state the score on fp32 values
        standard_normal = staticmethod(lambda shape: g.standard_normal(shape).astype(np.float32).astype(np.float64))
    ids = np.array([40, 41, 42, 43, 44])                         # passage table order
    P = 8
    r0 = {3: ([41, 41, 43], rng.standard_normal((3, P))), 7: ([40], rng.standard_normal((1, P)))}
    r1 = {3: ([44], rng.standard_normal((1, P))), 9: ([42, 44], rng.standard_normal((2, P)))}
    cls = [rng.standard_normal((3, 4)), rng.standard_normal((2, 4))]
    _write_index(tmp_path, [r0, r1], cls)
    entries, c = orc.read_index(str(tmp_path), ids)
    assert c.shape == (5, 4)
    q = [{3: [rng.standard_normal(P)], 9: [rng.standard_normal(P), rng.standard_normal(P)], 11: [np.ones(P)]},
         {7: [rng.standard_normal(P)]}]
    qc = rng.standard_normal((2, 4))
    S, B = orc.scores(entries, q, 5, c, qc)
    row = {int(p): i for i, p in enumerate(ids)}
    allent = {}
    for part in (r0, r1):
        for x, (cid, pay) in part.items():
            for i, v in zip(cid, pay):
                allent.setdefault(x, []).append((row[i], v))
    for qi, qd in enumerate(q):
        for d in range(5):
            want = float(qc[qi] @ c[d])
            for x, us in qd.items():
                for u in us:
                    vals = [float(u @ v) for rr, v in allent.get(x, []) if rr == d]
                    want += max(0.0, max(vals)) if vals else 0.0
            assert abs(S[qi, d] - want) <= 1e-12
    assert (B > 0).all()


def test_oracle_ties_go_to_the_lower_row():
    S = np.array([[1.0, 3.0, 3.0, 0.0, 3.0]])
    s, r = orc.topk(S, 4)
    assert r.tolist() == [[1, 2, 4, 0]] and s.tolist() == [[3.0, 3.0, 3.0, 1.0]]


def test_tiles_keep_runs_whole_and_cover_every_entry():
    from dpr_scale_b200 import ops
    rng = np.random.default_rng(1)
    ex = np.sort(rng.integers(0, 50, 20000))
    row = np.concatenate([np.sort(rng.integers(0, 300, n)) for n in np.bincount(ex, minlength=50)])
    row[:400] = 7                                                 # expert 0: one run longer than any window
    ex[:400] = 0
    order = np.lexsort((row, ex))
    ex, row = ex[order], row[order]
    tb, tp = ops.expert_search_tiles(ex, row, 50)
    assert tb[0] == 0 and tb[-1] == ex.size and (np.diff(tb) > 0).all()
    for lo in tb[1:-1]:                                           # a boundary never falls inside a run
        assert (ex[lo], row[lo]) != (ex[lo - 1], row[lo - 1])
    for x in range(50):                                           # each expert's tiles cover exactly its entries
        a, b = tp[x], tp[x + 1]
        assert (ex[tb[a]:tb[b]] == x).all() and (b == a) == (not (ex == x).any())
    assert np.diff(tb).max() >= 400


def test_groups_of_one_expert_and_no_empty_work():
    from dpr_scale_b200 import ops
    tile_ptr = np.array([0, 2, 2, 5, 6])                          # expert 1 has no postings
    q_ex = np.array([0] * 130 + [1, 1] + [3] + [9])               # expert 9 is outside the index vocabulary
    g, end, items = ops.expert_search_groups(q_ex, tile_ptr, 70, 1000)
    assert g[:, 0].tolist() == [0, 0, 0, 0, 1, 1]
    assert g[:3, 1].tolist() == [0, 64, 128] and g[:3, 2].tolist() == [64, 64, 2] and g[3].tolist() == [0, 132, 1, 5]
    assert g[4:, 1].tolist() == [0, 64] and g[4:, 2].tolist() == [64, 6]
    assert end.tolist() == [2, 4, 6, 7, 15, 23] and items == 23


class _Task:
    """merge_* of CITADELRetrievalTask without building encoders"""

    def __init__(self, index2docid_path=None, ctxs=None):
        from dpr_scale_b200.task.citadel_retrieval_task import CITADELRetrievalTask
        self.index2docid_path, self.ctxs = index2docid_path, ctxs
        self.merge_trec_results = CITADELRetrievalTask.merge_trec_results.__get__(self)
        self.merge_qa_results = CITADELRetrievalTask.merge_qa_results.__get__(self)


def test_run_file_formats(tmp_path):
    scores = [[2.5, 1.0000004], [0.0, -0.125]]
    ids = [[3, 1], [0, 2]]
    lines = _Task().merge_trec_results(["q1", "q2"], ids, scores)
    assert lines == ["q1 Q0 3 1 2.500000 dpr-scale\n", "q1 Q0 1 2 1.000000 dpr-scale\n",
                     "q2 Q0 0 1 0.000000 dpr-scale\n", "q2 Q0 2 2 -0.125000 dpr-scale\n"]
    i2d = tmp_path / "i2d.txt"
    i2d.write_text("d0\nd1\nd2\nd3\n")
    lines = _Task(str(i2d)).merge_trec_results(["q1", "q2"], ids, scores)
    assert lines[0] == "q1 Q0 d3 1 2.500000 dpr-scale\n" and lines[3] == "q2 Q0 d2 2 -0.125000 dpr-scale\n"
    table = {str(i): {"id": str(i), "title": f"t{i}", "text": f"x{i}"} for i in range(4)}
    qa = _Task(ctxs=table).merge_qa_results(["who?"], [["a"]], [[2, 0]], [[1.5, 0.25]])
    assert json.dumps(qa, indent=4) == json.dumps([{"question": "who?", "answers": ["a"], "ctxs": [
        {"id": "2", "title": "t2", "text": "x2", "score": 1.5},
        {"id": "0", "title": "t0", "text": "x0", "score": 0.25}]}], indent=4)


def test_config_composes():
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=multivec_retrieval", "task/model=citadel_model",
                             "datamodule=generate_multivec_query_emb", "datamodule.test_path=/q",
                             "task.model.model_path=/m", "+task.checkpoint_path=/c", "+task.ctx_embeddings_dir=/i",
                             "+task.passages=/p.tsv", "+task.output_path=/o", "+task.topk=10", "+task.add_cls=true"])
    assert cfg.task._target_ == "dpr_scale_b200.task.citadel_retrieval_task.CITADELRetrievalTask"
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.citadel_model.CITADELEncoder"
    assert cfg.task.topk == 10 and cfg.task.add_cls is True and cfg.task.shared_model is False


@pytest.mark.parametrize("kw, match", [({"quantizer": "pq"}, "quantizer"), ({"cuda": False}, "cuda"),
                                       ({"portion": 0.5}, "portion"), ({"hnsw_index": True}, "hnsw")])
def test_task_refuses_missing_index_options(kw, match):
    from dpr_scale_b200.task.citadel_retrieval_task import CITADELRetrievalTask
    with pytest.raises(ValueError, match=match):
        CITADELRetrievalTask(ctx_embeddings_dir="/i", checkpoint_path="/c", transform={}, datamodule=None, optim={},
                             model={}, **kw)


@pytest.mark.parametrize("args, match", [((12, None, 100, 10, 10, 1), "payload width"),
                                         ((32, 1032, 100, 10, 10, 1), "CLS width"),
                                         ((32, None, 1 << 24, 10, 10, 1), "vocabulary"),
                                         ((32, None, 100, 1 << 31, 10, 1), "index entries"),
                                         ((32, None, 100, 10, 1 << 31, 1), "passages"),
                                         ((32, None, 100, 10, 10, 11), "topk"),
                                         ((32, None, 100, 10, 5000, 1025), "topk")])
def test_search_limits(args, match):
    from dpr_scale_b200 import ops
    with pytest.raises(ValueError, match=match):
        ops.expert_search_check(*args)


def test_index_load_refusals(tmp_path):
    from dpr_scale_b200.task.citadel_retrieval_task import ExpertIndex
    ids = np.array([1, 2, 3])
    good = tmp_path / "good"
    _write_index(good, [{4: ([1, 3], np.ones((2, 8)))}], [np.ones((3, 16))])
    with pytest.raises(ValueError, match="not in the passage table"):
        ExpertIndex.load(str(good), np.array([1, 2]), device="cpu")
    with pytest.raises(ValueError, match="CLS rows"):
        ExpertIndex.load(str(good), np.array([1, 2, 3, 4]), add_cls=True, device="cpu")
    with pytest.raises(ValueError, match="8-wide payloads but the encoder's are 16"):
        ExpertIndex.load(str(good), ids, P=16, device="cpu")
    with pytest.raises(ValueError, match="CLS vectors are 16-wide"):
        ExpertIndex.load(str(good), ids, add_cls=True, P=8, Pc=32, device="cpu")
    nocls = tmp_path / "nocls"
    _write_index(nocls, [{4: ([1], np.ones((1, 8)))}])
    with pytest.raises(ValueError, match="no cls_"):
        ExpertIndex.load(str(nocls), ids, add_cls=True, device="cpu")
    ctx = tmp_path / "ctx" / "expert_0000"
    ctx.mkdir(parents=True)
    with open(ctx / "4.pkl", "wb") as f:
        pickle.dump((torch.tensor([1]), torch.ones(1), torch.tensor([7.0])), f, protocol=4)
    with pytest.raises(ValueError, match="add_context_id"):
        ExpertIndex.load(str(tmp_path / "ctx"), ids, device="cpu")


# ---- against the unmodified reference (tests/golden/make_golden_multivec_retrieval.py)
GOLD = os.path.join(ROOT, "tests", "golden", "multivec_retrieval_small.npz")
RETRIEVAL = {"coil_bert": ("coil_bert", 1, False), "coil_bert_cls": ("coil_bert", 1, True),
             "citadel_bert_k1_cls": ("citadel_bert", 1, True), "citadel_bert_k2": ("citadel_bert", 2, False)}
PASSAGE_IDS = list(range(100, 107))


def _kept(r):
    """the kept (query or passage n, expert, payload float64, weight) entries of one batch's encoder outputs, in the
    reference's (n, token, slot) order: unmasked tokens 1.. and slots with weight > 0"""
    ids, w, am, rep = r["expert_ids"], r["expert_weights"], r["attention_mask"], r["expert_repr"]
    if ids.ndim == 2:
        ids, w = ids[..., None], w[..., None]
    out = []
    for n in range(ids.shape[0]):
        for s in range(ids.shape[1]):
            if am[n, s] <= 0:
                continue
            for k in range(ids.shape[2]):
                if w[n, s, k] > 0:
                    out.append((n, int(ids[n, s, k]), w[n, s, k].astype(np.float64) * rep[n, s].astype(np.float64),
                                w[n, s, k]))
    return out


def _batch(G, case, side, i):
    return {k: G[f"{case}/{side}{i}/{k}"] for k in ("expert_ids", "expert_weights", "attention_mask", "expert_repr",
                                                     "cls_repr") if f"{case}/{side}{i}/{k}" in G}


@pytest.mark.parametrize("case", list(RETRIEVAL))
def test_oracle_equals_reference_expert_sim_score(case):
    G = np.load(GOLD)
    add_cls = RETRIEVAL[case][2]
    cb = [_batch(G, case, "c", i) for i in range(2)]
    qb = [_batch(G, case, "q", i) for i in range(2)]
    base = np.cumsum([0] + [c["expert_ids"].shape[0] for c in cb])
    N = int(base[-1])
    per_x = {}
    for ci, c in enumerate(cb):
        for n, x, v, _ in _kept(c):
            per_x.setdefault(x, []).append((base[ci] + n, v))
    entries = {}
    for x, lst in per_x.items():
        rows = np.array([r for r, _ in lst])
        o = np.argsort(rows, kind="stable")
        entries[x] = (rows[o], np.stack([v for _, v in lst])[o])
    cls = np.concatenate([c["cls_repr"].astype(np.float64) for c in cb]) if add_cls else None
    checked = 0
    for qi, q in enumerate(qb):
        qd = [dict() for _ in range(q["expert_ids"].shape[0])]
        for n, x, u, _ in _kept(q):
            qd[n].setdefault(x, []).append(u)
        S, _ = orc.scores(entries, qd, N, cls, q["cls_repr"].astype(np.float64) if add_cls else None)
        for ci, c in enumerate(cb):
            ref = G[f"{case}/score/q{qi}/c{ci}"]
            cols = c["expert_ids"].reshape(c["expert_ids"].shape[0], -1)
            for n in range(len(qd)):
                for d in range(cols.shape[0]):
                    # the clamp equivalence: every query entry's expert meets a column of another expert
                    if all((cols[d] != x).any() for x in qd[n]):
                        assert abs(S[n, base[ci] + d] - ref[n, d]) <= 1e-12 * max(1.0, abs(ref[n, d]))
                        checked += 1
    assert checked >= 20
    print(f"{case}: {checked} pairs equal the reference's expert_sim_score{' + sim_score' if add_cls else ''}")


@pytest.mark.parametrize("case", list(RETRIEVAL))
def test_reference_query_entries_follow_the_keep_rule(case):
    """what the reference's _eval_step passes to its index = unmasked tokens 1.., slots with weight > 0, payload
    w * rep (CITADEL: rounded to fp16), grouped by expert in token order - the rule dprb_expert_group applies"""
    G = np.load(GOLD)
    enc, _, add_cls = RETRIEVAL[case]
    for i in range(2):
        q = _batch(G, case, "q", i)
        want = [dict() for _ in range(q["expert_ids"].shape[0])]
        for n, x, _, w in _kept(q):
            want[n].setdefault(x, [])
        rep, ids = q["expert_repr"], q["expert_ids"]
        for n in range(len(want)):
            assert sorted(G[f"{case}/q{i}/{n}/experts"].tolist()) == sorted(want[n])
        half = not enc.startswith("coil")          # CITADEL payloads and weights are rounded to fp16
        flat_w = q["expert_weights"] if ids.ndim == 3 else q["expert_weights"][..., None]
        flat_x = ids if ids.ndim == 3 else ids[..., None]
        pays = [dict((x, []) for x in d) for d in want]
        for n in range(ids.shape[0]):
            for s in range(ids.shape[1]):
                if q["attention_mask"][n, s] <= 0:
                    continue
                for k in range(flat_x.shape[2]):
                    w = np.float32(flat_w[n, s, k])
                    if w > 0:
                        x = int(flat_x[n, s, k])
                        u = (torch.tensor(w) * torch.from_numpy(rep[n, s])).float()
                        pays[n][x].append(u.half().float().numpy() if half else u.numpy())
                        want[n][x].append(np.float32(np.float16(w)) if half else w)
        for n in range(len(want)):
            for x in want[n]:
                assert np.array_equal(G[f"{case}/q{i}/{n}/x{x}/weight"], np.array(want[n][x], dtype=np.float32))
                assert np.array_equal(G[f"{case}/q{i}/{n}/x{x}/repr"], np.stack(pays[n][x]))
                assert str(G[f"{case}/q{i}/{n}/x{x}/dtype"]) == ("torch.float16" if half else "torch.float32")
        if add_cls:
            assert np.array_equal(G[f"{case}/q{i}/batch_cls"], q["cls_repr"])


class _FilesTask(_Task):
    def __init__(self, output_path, index2docid_path, table):
        from dpr_scale_b200.datamodule.cross_encoder import IDCSVDataset
        from dpr_scale_b200.task.citadel_retrieval_task import CITADELRetrievalTask
        super().__init__(index2docid_path, IDCSVDataset(table))
        self.output_path, self.global_rank = output_path, 0
        self.test_epoch_end = CITADELRetrievalTask.test_epoch_end.__get__(self)


def test_run_files_equal_the_reference(tmp_path):
    G = np.load(GOLD)
    scores, ids = json.loads(str(G["files/results"]))
    table = tmp_path / "passages.tsv"
    table.write_text("id\ttext\ttitle\n" + "".join(f"{i}\tpassage text {i}\ttitle {i}\n" for i in PASSAGE_IDS))
    i2d = tmp_path / "i2d.txt"
    i2d.write_text("".join(f"doc{i}\n" for i in range(110)))
    for name, i2d_path, qa in (("trec", None, False), ("trec_i2d", str(i2d), False), ("qa", None, True)):
        odir = tmp_path / ("out_" + name)
        t = _FilesTask(str(odir), i2d_path, str(table))
        res = [(scores, ids, [], ["who is q1?", "what is q2?"], [["a1"], ["a2", "b2"]])] if qa else \
            [(scores, ids, ["q1", "q2"], [], [])]
        path = t.test_epoch_end(res)
        assert os.path.basename(path) == ("retrieval_0000.json" if qa else "retrieval_0000.trec")
        with open(path, "rb") as f:
            assert f.read() == G[f"files/{name}"].tobytes(), name
