"""SPLADE first-stage retrieval on the host: the CSR file writer and reader, the shard layout of the sparse embedding
tasks, every input the index and the retrieval command refuse, the search's host-side limits and the configs."""
import os
import pickle

import numpy as np
import pytest
import torch

from dpr_scale_b200 import ops
from dpr_scale_b200.utils.csr_writer import StreamingCSRPickle, load_csr


def _random_csr(rng, N, V, per_row=5, dtype=np.float16):
    counts = rng.integers(0, 2 * per_row, N).astype(np.int64)
    counts[::7] = 0                                                   # empty rows
    terms = np.concatenate([np.sort(rng.choice(V, c, replace=False)) for c in counts]).astype(np.int32)
    weights = rng.random(terms.size).astype(dtype) * 3
    return counts, terms, weights


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_csr_round_trip(tmp_path, dtype):
    rng = np.random.default_rng(1)
    path = str(tmp_path / "sparse_0000.pkl")
    w = StreamingCSRPickle(path, 300, dtype)
    want_c, want_t, want_w = [], [], []
    for b in range(5):
        c, t, x = _random_csr(rng, 1 + 3 * b, 300, dtype=dtype)
        w.append(c, t, x)
        want_c.append(c), want_t.append(t), want_w.append(x)
    topics = [f"q{i}" for i in range(sum(len(c) for c in want_c))]
    w.close(topics if dtype == np.float32 else None)
    assert sorted(os.listdir(tmp_path)) == ["sparse_0000.pkl"]        # the spools are gone
    with open(path, "rb") as f:
        assert f.read(2) == b"\x80\x04"                               # pickle protocol 4
    d = load_csr(path)
    c = np.concatenate(want_c)
    assert d["offsets"].dtype == np.int64 and np.array_equal(d["offsets"], np.r_[0, np.cumsum(c)])
    assert d["terms"].dtype == np.int32 and np.array_equal(d["terms"], np.concatenate(want_t))
    assert d["weights"].dtype == dtype and np.array_equal(d["weights"], np.concatenate(want_w))
    assert d["V"] == 300
    assert d.get("topic_ids") == (topics if dtype == np.float32 else None)


def test_empty_file_and_malformed_files(tmp_path):
    p = str(tmp_path / "e.pkl")
    StreamingCSRPickle(p, 10, np.float16).close()
    d = load_csr(p)
    assert d["offsets"].tolist() == [0] and d["terms"].size == 0 and d["V"] == 10
    bad = str(tmp_path / "bad.pkl")
    with open(bad, "wb") as f:
        pickle.dump({"offsets": np.array([0, 3]), "terms": np.zeros(2, np.int32), "weights": np.zeros(2, np.float16),
                     "V": 5}, f, protocol=4)
    with pytest.raises(ValueError, match="CSR"):
        load_csr(bad)
    with open(bad, "wb") as f:
        pickle.dump(torch.zeros(3, 4), f, protocol=4)
    with pytest.raises(ValueError, match="not a sparse embedding file"):
        load_csr(bad)


class _Fake(torch.nn.Module):
    """Stands in for SPLADEEncoder on the host: a fixed [B, V] block per call."""

    def __init__(self, block, dim):
        super().__init__()
        self.block, self.dim = block, dim

    def forward(self, tokens):
        return self.block


def _gen_task(tmp_path, query=False, **kw):
    from dpr_scale_b200.task.splade_index_task import GenerateSparseEmbeddingsTask, GenerateSparseQueryEmbeddingsTask
    cls = GenerateSparseQueryEmbeddingsTask if query else GenerateSparseEmbeddingsTask
    t = cls.__new__(cls)
    torch.nn.Module.__init__(t)
    t.ctx_embeddings_dir = str(tmp_path)
    t.trainer = None
    if query:
        t.query_emb_output_path = str(tmp_path / "sparse_query.pkl")
        t._topic_ids = []
    for k, v in kw.items():
        setattr(t, k, v)
    return t


def _use_fake(monkeypatch, task, blocks, V):
    from dpr_scale_b200.task import splade_index_task
    monkeypatch.setattr(splade_index_task, "SPLADEEncoder", _Fake)
    it = iter(blocks)
    enc = _Fake(None, V)
    enc.forward = lambda tokens: next(it)
    task.context_encoder = task.query_encoder = enc


def test_shard_layout_and_query_topic_ids(tmp_path, monkeypatch):
    rng = np.random.default_rng(4)
    V = 50
    blocks = []
    for B in (4, 3, 5):
        x = torch.from_numpy(rng.random((B, V)).astype(np.float32))
        x[x < 0.8] = 0
        blocks.append(x)
    blocks[1][2] = 0                                                  # a passage without a nonzero
    t = _gen_task(tmp_path)
    _use_fake(monkeypatch, t, blocks, V)
    for i in range(3):
        t.test_step({"contexts_ids": None}, i)
    path = t.test_epoch_end([])
    assert os.path.basename(path) == "sparse_0000.pkl"
    d = load_csr(path)
    full = torch.cat(blocks)
    nz = full.nonzero()
    assert d["V"] == V and d["weights"].dtype == np.float16 and d["terms"].dtype == np.int32
    assert np.array_equal(d["offsets"], np.r_[0, np.cumsum(np.bincount(nz[:, 0].numpy(), minlength=12))])
    assert np.array_equal(d["terms"], nz[:, 1].numpy())
    assert np.array_equal(d["weights"], full[nz[:, 0], nz[:, 1]].half().numpy())

    q = _gen_task(tmp_path, query=True)
    _use_fake(monkeypatch, q, blocks[:2], V)
    q.test_step({"query_ids": None, "topic_ids": ["a", "b", "c", "d"]}, 0)
    q.test_step({"query_ids": None, "topic_ids": ["e", "f", "g"]}, 1)
    d = load_csr(q.test_epoch_end([]))
    assert d["weights"].dtype == np.float32 and d["topic_ids"] == list("abcdefg")
    assert np.array_equal(d["weights"], torch.cat(blocks[:2])[torch.cat(blocks[:2]) != 0].numpy())


def test_generation_refusals(tmp_path, monkeypatch):
    t = _gen_task(tmp_path)
    t.context_encoder = torch.nn.Linear(2, 2)
    with pytest.raises(ValueError, match="SPLADEEncoder"):
        t.test_step({"contexts_ids": None}, 0)
    for bad in (7e4, float("inf"), float("nan")):
        t = _gen_task(tmp_path)
        _use_fake(monkeypatch, t, [torch.tensor([[0.0, 1.0, bad]])], 3)
        with pytest.raises(ValueError, match="fp16"):
            t.test_step({"contexts_ids": None}, 0)


def _write(path, offsets, terms, weights, V, dtype=np.float16):
    w = StreamingCSRPickle(path, V, dtype)
    w.append(np.diff(np.asarray(offsets)).astype(np.int64), np.asarray(terms, np.int32), np.asarray(weights, dtype))
    return w.close()


def test_index_and_command_refusals(tmp_path):
    from dpr_scale_b200.splade_retrieval import SparseIndex, search_distributed, shard_paths
    with pytest.raises(ValueError, match="empty"):
        SparseIndex([0], [], [], 10, device="cpu")
    with pytest.raises(ValueError, match="term ids outside"):
        SparseIndex([0, 2], [1, 10], [1.0, 1.0], 10, device="cpu")
    with pytest.raises(ValueError, match="term ids outside"):
        SparseIndex([0, 1], [-1], [1.0], 10, device="cpu")
    with pytest.raises(ValueError, match="fp16"):
        SparseIndex([0, 1], [3], [1e5], 10, device="cpu")
    idx = SparseIndex([0, 2, 2, 3], [1, 4, 4], [1.0, 2.0, 0.5], 10, device="cpu")
    with pytest.raises(ValueError, match="term ids outside"):
        idx.search([0, 1], [12], [1.0], 1)
    with pytest.raises(ValueError, match="fixed-point"):
        idx.search([0, 1], [4], [6e8], 1)
    with pytest.raises(ValueError, match="topk"):
        idx.search([0, 1], [4], [1.0], 4)
    # the command: no shard, shards of different V, a query V other than the index's
    q = {"offsets": np.array([0, 1]), "terms": np.array([1], np.int32), "weights": np.ones(1, np.float32), "V": 10}
    d = tmp_path / "idx"
    d.mkdir()
    with pytest.raises(ValueError, match="empty"):
        search_distributed(shard_paths(str(d)), q, 1, "cpu")
    _write(str(d / "sparse_0000.pkl"), [0, 1], [3], [1.0], 10)
    _write(str(d / "sparse_query.pkl"), [0, 1], [3], [1.0], 10, np.float32)
    assert [os.path.basename(p) for p in shard_paths(str(d))] == ["sparse_0000.pkl"]
    with pytest.raises(ValueError, match="differs"):
        search_distributed(shard_paths(str(d)), dict(q, V=11), 1, "cpu")
    _write(str(d / "sparse_0001.pkl"), [0, 1], [3], [1.0], 12)
    with pytest.raises(ValueError, match="different vocabulary"):
        search_distributed(shard_paths(str(d)), q, 1, "cpu")


def test_index_refuses_repeated_terms_in_a_row():
    """The fixed-point range bound counts each term once per passage, so a row must hold each term once."""
    from dpr_scale_b200.splade_retrieval import SparseIndex
    for terms in ([1, 4, 4], [4, 1, 5]):                            # a repeat; a row not in ascending order
        with pytest.raises(ValueError, match="repeats a term"):
            SparseIndex([0, 3, 3], terms, [1.0, 1.0, 1.0], 10, device="cpu")
    SparseIndex([0, 2, 3], [1, 4, 4], [1.0, 1.0, 1.0], 10, device="cpu")     # the same term in two rows


def test_index_layout_on_the_host():
    """Postings by term, rows ascending inside a term; fp16 weights; padded to 8; term_ptr; per-term max."""
    from dpr_scale_b200.splade_retrieval import SparseIndex
    offsets = [0, 3, 3, 5, 6]
    terms = [2, 5, 7, 0, 5, 5]
    w = [0.1, 0.2, 0.3, 0.4, 0.5, 1 / 3]
    idx = SparseIndex(offsets, terms, w, 8, ids=np.arange(4) + 100, device="cpu")
    assert idx.term_ptr.tolist() == [0, 1, 1, 2, 2, 2, 5, 5, 6]
    assert idx.row[:6].tolist() == [2, 0, 0, 2, 3, 0] and idx.row.numel() == 8
    assert idx.weight[:6].tolist() == torch.tensor([0.4, 0.1, 0.2, 0.5, 1 / 3, 0.3]).half().tolist()
    assert idx.term_max[5] == float(np.float16(0.5)) and idx.term_max[1] == 0.0
    assert idx.ids.tolist() == [100, 101, 102, 103]


def test_sparse_search_check_limits():
    ops.sparse_search_check(30522, 0, 1, 1)
    ops.sparse_search_check(2 ** 31 - 1, 2 ** 40 - 1, 2 ** 31 - 1, 1024)
    for args, what in (((0, 1, 10, 1), "vocabulary"), ((2 ** 31, 1, 10, 1), "vocabulary"),
                       ((10, -1, 10, 1), "postings"), ((10, 2 ** 40, 10, 1), "postings"),
                       ((10, 1, 0, 1), "passages"), ((10, 1, 2 ** 31, 1), "passages"),
                       ((10, 1, 10, 0), "topk"), ((10, 1, 10, 11), "topk"), ((10, 1, 5000, 1025), "topk")):
        with pytest.raises(ValueError, match=what):
            ops.sparse_search_check(*args)


def test_work_items():
    term_ptr = np.array([0, 0, 1, 1 + ops.SPARSE_SEARCH_TILE, 2 + 3 * ops.SPARSE_SEARCH_TILE], np.int64)
    end, items = ops.sparse_search_items(term_ptr, np.array([0, 1, 2, 3, 1]))
    assert end.tolist() == [0, 1, 2, 5, 6] and items == 6 and end.dtype == np.int32
    assert ops.sparse_search_items(term_ptr, np.zeros(0, np.int64))[1] == 0


@pytest.mark.parametrize("which", ["generate_sparse_embeddings", "generate_sparse_query_embeddings"])
def test_config_composes(which):
    from dpr_scale_b200.utils.config import compose
    dm = "generate" if which == "generate_sparse_embeddings" else "generate_multivec_query_emb"
    cfg = compose("config", [f"task={which}", "task/model=splade_model", f"datamodule={dm}", "datamodule.test_path=/q",
                             "task.model.model_path=/m", "+task.checkpoint_path=/c", "+task.ctx_embeddings_dir=/o"])
    cls = "GenerateSparseEmbeddingsTask" if which == "generate_sparse_embeddings" else \
        "GenerateSparseQueryEmbeddingsTask"
    assert cfg.task._target_ == "dpr_scale_b200.task.splade_index_task." + cls
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.splade_model.SPLADEEncoder"
    assert cfg.task.ctx_embeddings_dir == "/o" and cfg.task.checkpoint_path == "/c"


def test_command_flags():
    from dpr_scale_b200.splade_retrieval import get_parser
    a = get_parser().parse_args(["--ctx_embeddings_dir", "/i", "--topk", "7", "--trec_format", "--fp32_scores",
                                 "--ignore_identical_ids", "--run_name", "r", "--query_emb_path", "/q.pkl",
                                 "--questions_tsv_path", "/q.tsv", "--passages_tsv_path", "/p.tsv",
                                 "--output_runfile_path", "/o.trec"])
    assert (a.topk, a.trec_format, a.fp32_scores, a.ignore_identical_ids, a.run_name) == (7, True, True, True, "r")


def test_oracle_on_a_hand_example():
    from oracle import sparse_retrieval as osr
    index = ([0, 2, 3, 3], [1, 2, 2], [0.5, 1 / 3, 2.0])
    queries = ([0, 2, 2], [2, 2], [1.0, 0.5])                       # a repeated term adds up; query 1 is empty
    S, M = osr.scores(index, queries, 4)
    third = float(np.float16(1 / 3))
    assert np.allclose(S, [[1.5 * third, 3.0, 0.0], [0, 0, 0]], rtol=0, atol=0)
    s, r = osr.topk(S, 3)
    assert r.tolist() == [[1, 0, 2], [0, 1, 2]]
