"""COIL / CITADEL expert-index generation on the host, against goldens the unmodified reference produced
(tests/golden/make_golden_multivec_index.py):

  * the float64 oracle (oracle/multivec_index.py), given the reference's encoder outputs, reproduces every file the
    reference wrote, exactly once rounded to fp32, keys and entry order included;
  * the task and datamodule configs compose, and the query collate equals the reference's batches;
  * refusals raise ValueError without a GPU: a ColBERT encoder, a query batch without topic ids, a grad-enabled step,
    a non-integer corpus id, shapes outside the kernel's limits.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests import colbert_cases, multivec_cases, multivec_index_cases as cases, rerank_cases
from tests.util import GOLDEN

G = np.load(os.path.join(GOLDEN, "multivec_index_small.npz"))
KEYS = ("expert_repr", "expert_ids", "expert_weights", "attention_mask")


def reference_outputs(side, case, i):
    return {k: G[f"{side}/{case}/b{i}/{k}"] for k in KEYS}


@pytest.mark.parametrize("case", list(cases.PASSAGE))
def test_oracle_reproduces_reference_passage_files(case):
    from oracle import multivec_index as om
    enc, _, add_cls, ctx_id, thr = cases.PASSAGE[case]
    batches = [(reference_outputs("p", case, i), G[f"p/{case}/b{i}/input_ids"], ids)
               for i, (_, ids) in enumerate(cases.batches(enc))]
    got = om.passage_index(batches, ctx_id, thr)
    assert sorted(got) == G[f"p/{case}/experts"].tolist()
    for x, (ids, w, reps) in got.items():
        assert np.array_equal(ids, G[f"p/{case}/x{x}/ids"])
        assert np.array_equal(w.astype(np.float32), G[f"p/{case}/x{x}/weights"])
        assert np.array_equal(reps.astype(np.float32), G[f"p/{case}/x{x}/reprs"])
    assert (f"p/{case}/cls" in G) == add_cls


@pytest.mark.parametrize("case", list(cases.QUERY))
def test_oracle_reproduces_reference_query_files(case):
    from oracle import multivec_index as om
    enc, _, add_cls = cases.QUERY[case]
    emb, wts = [], []
    for i in range(len(cases.SHAPES)):
        e, w = om.query_index(reference_outputs("q", case, i))
        emb.extend(e)
        wts.extend(w)
    assert G[f"q/{case}/topic_ids"].tolist() == [t for _, ids in cases.batches(enc, seed=6) for t in ids]
    assert len(emb) == len(G[f"q/{case}/topic_ids"])
    for j, (e, w) in enumerate(zip(emb, wts)):
        assert list(e) == G[f"q/{case}/{j}/experts"].tolist()                 # the reference's key order too
        for x in e:
            assert np.array_equal(np.stack(e[x]).astype(np.float32), G[f"q/{case}/{j}/x{x}/repr"])
            assert np.array_equal(np.array(w[x]).astype(np.float32), G[f"q/{case}/{j}/x{x}/weight"])
    assert (f"q/{case}/cls" in G) == add_cls


@pytest.mark.parametrize("which", ["generate_multivec_embeddings", "generate_multivec_query_embeddings"])
def test_config_composes(which):
    from dpr_scale_b200.utils.config import compose
    dm = "generate" if which == "generate_multivec_embeddings" else "generate_multivec_query_emb"
    cfg = compose("config", [f"task={which}", "task/model=citadel_model", f"datamodule={dm}",
                             "datamodule.test_path=/q", "task.model.model_path=/m", "+task.checkpoint_path=/c",
                             "+task.ctx_embeddings_dir=/o", "+task.add_cls=true", "+task.context_topk=2",
                             "task.weight_threshold=0.5"])
    cls = "GenerateMultiVecEmbeddingsTask" if which == "generate_multivec_embeddings" else \
        "GenerateMultiVecQueryEmbeddingsTask"
    assert cfg.task._target_ == "dpr_scale_b200.task.citadel_eval_task." + cls
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.citadel_model.CITADELEncoder"
    assert cfg.task.add_context_id is False and cfg.task.weight_threshold == 0.5 and cfg.task.context_topk == 2
    if which != "generate_multivec_embeddings":
        assert cfg.datamodule._target_ == "dpr_scale_b200.datamodule.citadel.DenseRetrieverQueriesDataModule"
        assert cfg.datamodule.test_batch_size == 128 and cfg.datamodule.trec_format is False


@pytest.mark.parametrize("fmt", ["trec", "csv"])
def test_query_collate_matches_reference_batches(tmp_path, fmt):
    from dpr_scale_b200.datamodule.citadel import DenseRetrieverQueriesDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    tok_dir = rerank_cases.tokenizer_dir(str(tmp_path / "tok"))
    dm = DenseRetrieverQueriesDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                         test_path=os.path.join(rerank_cases.DATA, "questions.tsv" if fmt == "trec"
                                                                else "questions.csv"),
                                         test_batch_size=4, trec_format=fmt == "trec", prefetch_batches=0,
                                         device_prefetch=False)
    bs = list(dm.test_dataloader())
    assert len(bs) == int(G[f"dm/{fmt}/n_batches"])
    for i, b in enumerate(bs):
        pre = f"dm/{fmt}/b{i}/"
        assert sorted(b) == G[pre + "keys"].tolist()
        for k, v in b["query_ids"].items():
            assert np.array_equal(torch.as_tensor(v).numpy(), G[pre + "query_ids/" + k]), k
        for k in ("question", "topic_ids", "answers"):
            if k in b:
                assert json.loads(str(G[pre + k])) == b[k]


def _task(tmp_path, enc, query=False, **kw):
    from dpr_scale_b200.task.citadel_eval_task import (GenerateMultiVecEmbeddingsTask,
                                                       GenerateMultiVecQueryEmbeddingsTask)
    model = multivec_cases.TINY[enc][0] if enc in multivec_cases.TINY else "colbert"
    mdir = (multivec_cases.model_dir if enc in multivec_cases.TINY else colbert_cases.model_dir)(
        str(tmp_path / "model"), enc)
    ckpt = str(tmp_path / "task.ckpt")
    sd = multivec_cases.task_state_dict(enc) if enc in multivec_cases.TINY else colbert_cases.task_state_dict(enc)
    torch.save({"state_dict": sd}, ckpt)
    if enc in multivec_cases.TINY:
        kwargs = cases.task_kwargs(enc, mdir, kw.pop("topk", 1), kw.pop("add_cls", False))
        kwargs["model"]["_target_"] = "dpr_scale_b200.models.citadel_models." + multivec_cases.TARGETS[model]
    else:
        kwargs = dict(transform={}, datamodule=None, optim={}, shared_model=False,
                      model={"_target_": "dpr_scale_b200.models.citadel_models.colbert_model.ColBERTEncoder",
                             "model_path": mdir, "projection_dim": colbert_cases.TINY[enc][1]})
    cls = GenerateMultiVecQueryEmbeddingsTask if query else GenerateMultiVecEmbeddingsTask
    task = cls(ctx_embeddings_dir=str(tmp_path / "out"), checkpoint_path=ckpt, add_context_id=False, **kwargs, **kw)
    task.setup("test")
    return task


def test_refusals_without_a_gpu(tmp_path):
    toks, ids = cases.batches("citadel_bert")[0]
    task = _task(tmp_path / "cit", "citadel_bert")
    with torch.no_grad():
        with pytest.raises(ValueError):
            task.test_step({"contexts_ids": toks, "corpus_ids": ["a"] + ids[1:]}, 0)         # non-integer corpus id
        long = {k: v.repeat(1, 43)[:, :513] for k, v in toks.items()}
        with pytest.raises(ValueError):
            task.test_step({"contexts_ids": long, "corpus_ids": ids}, 0)                     # S > 512
        task.context_topk = 9
        with pytest.raises(ValueError):
            task.test_step({"contexts_ids": toks, "corpus_ids": ids}, 0)                     # K > 8
    task.context_topk = 1
    with torch.enable_grad():
        with pytest.raises(ValueError):
            task.test_step({"contexts_ids": toks, "corpus_ids": ids}, 0)
    colbert = _task(tmp_path / "col", colbert_cases.TASK_KINDS[0])
    with torch.no_grad(), pytest.raises(ValueError):
        colbert.test_step({"contexts_ids": toks, "corpus_ids": ids}, 0)
    q = _task(tmp_path / "q", "coil_bert", query=True)
    assert q.query_emb_output_dir == q.ctx_embeddings_dir
    with torch.no_grad(), pytest.raises(ValueError):
        q.test_step({"query_ids": toks, "question": ["?"] * len(ids)}, 0)


def test_expert_group_check_limits():
    from dpr_scale_b200 import ops
    ops.expert_group_check(128, 512, 8, 1024, (1 << 24) - 1)
    ops.expert_group_check(1, 2, 1, 8, 1)
    ops.expert_group_check(3, 16, 2, 0, 30522, context_id=True)                 # P is not read with token ids
    for args in ((0, 16, 1, 32, 100), (2, 1, 1, 32, 100), (2, 513, 1, 32, 100), (2, 16, 0, 32, 100),
                 (2, 16, 9, 32, 100), (2, 16, 1, 12, 100), (2, 16, 1, 1032, 100), (2, 16, 1, 0, 100),
                 (2, 16, 1, 32, 0), (2, 16, 1, 32, 1 << 24), (1 << 20, 512, 8, 32, 100)):
        with pytest.raises(ValueError):
            ops.expert_group_check(*args)
