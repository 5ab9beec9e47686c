"""Cross-encoder reranking on the host, against goldens the unmodified reference produced
(tests/golden/make_golden_rerank.py):

  * CrossEncoderRerankDataModule: every batch (qids, ctx ids, pair token tensors) equal to the reference's collate, with
    and without the background assembly thread, and the 2-rank contiguous shard split;
  * CrossEncoder state dicts: a tiny reference BERT (1 label) and RoBERTa (2 labels), rebuilt from their seeds and
    checked against the golden's checksums, load strictly, keys and shapes equal, and a checkpoint directory loads to
    the same tensors;
  * the float64 oracle against the reference's logits;
  * rerank.trec: per-query descending scores, ties in run-file order, shards merged in rank order;
  * configs that the kernels cannot run raise ValueError at construction; the YAML groups compose.
"""
import json
import os
import pickle
import types

import numpy as np
import pytest
import torch

from tests import rerank_cases
from tests.util import GOLDEN

RAW = np.load(os.path.join(GOLDEN, "rerank_small.npz"))
G = {k: torch.from_numpy(RAW[k]) for k in RAW.files if RAW[k].dtype.kind != "U"}   # numeric entries as tensors


def _golden_batches():
    out = []
    for i in range(int(G["n_batches"])):
        out.append({"qid": RAW[f"batch{i}/qid"].tolist(), "ctx_id": RAW[f"batch{i}/ctx_id"].tolist(),
                    "text_ids": {k.split("/")[-1]: G[k] for k in G if k.startswith(f"batch{i}/text_ids/")}})
    return out


def _datamodule(tmp_path, **kw):
    from dpr_scale_b200.datamodule.cross_encoder import CrossEncoderRerankDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    tok = rerank_cases.tokenizer_dir(str(tmp_path / "tok"))
    return CrossEncoderRerankDataModule(transform=HFTransform(tok, max_seq_len=rerank_cases.MAX_LEN),
                                        device_prefetch=False, **rerank_cases.datamodule_kwargs(), **kw)


def _reference_sd(kind):
    """The reference CrossEncoder's state_dict, rebuilt from the seed; its keys, shapes and checksum are the golden's."""
    sd = rerank_cases.reference_state_dict(kind)
    assert list(sd) == RAW[f"{kind}/sd_keys"].tolist()
    assert [list(v.shape) for v in sd.values()] == json.loads(str(RAW[f"{kind}/sd_shapes"]))
    assert torch.equal(rerank_cases.sd_checksum(sd), G[f"{kind}/sd_checksum"]), "seeded weights differ from the golden's"
    return sd


def _same_batch(got, want):
    assert got["qid"] == want["qid"] and got["ctx_id"] == want["ctx_id"]
    assert set(got["text_ids"]) == set(want["text_ids"])
    for k, v in want["text_ids"].items():
        assert torch.equal(got["text_ids"][k], v), k


@pytest.mark.parametrize("prefetch", [0, 3])
def test_batches_equal_reference_collate(tmp_path, prefetch):
    dm = _datamodule(tmp_path, prefetch_batches=prefetch)
    got, want = list(dm.test_dataloader()), _golden_batches()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        _same_batch(g, w)


def test_two_rank_shards_are_the_reference_sampler_rows(tmp_path):
    want_rows = [r for b in _golden_batches() for r in zip(b["qid"], b["ctx_id"])]
    seen = []
    for rank in range(2):
        dm = _datamodule(tmp_path, prefetch_batches=0)
        dm.trainer = types.SimpleNamespace(world_size=2, global_rank=rank)
        order = dm._test_order()
        assert order == G[f"shard2/rank{rank}"].tolist()
        rows = [r for b in dm.test_dataloader() for r in zip(b["qid"], b["ctx_id"])]
        assert rows == [want_rows[i] for i in order]
        seen += rows
    assert seen == want_rows


def test_readers_follow_the_reference_lookup_rules(tmp_path):
    from dpr_scale_b200.datamodule.cross_encoder import IDCSVDataset, QueryTRECDataset
    q = tmp_path / "q.tsv"
    q.write_text('a\tfirst\nb\t"quoted ""x"" y"\na\tsecond\n')
    qs = QueryTRECDataset(str(q))
    assert qs["a"]["question"] == "second" and qs["b"]["question"] == 'quoted "x" y'    # last line of an id wins
    p = tmp_path / "p.tsv"
    p.write_text("title\tid\ttext\nT1\tx7\tbody\n")
    assert IDCSVDataset(str(p))["x7"] == {"title": "T1", "id": "x7", "text": "body"}
    with pytest.raises(KeyError):
        qs["missing"]


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_reference_state_dict_loads_strictly(tmp_path, kind):
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    cfg = json.loads(str(RAW[f"{kind}/config"]))
    ref = _reference_sd(kind)
    m = CrossEncoder.from_config(cfg, seed=5)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.items()}
    m.load_state_dict(ref, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, ref[k]), k
    assert m.num_labels == cfg["num_labels"]
    # a HuggingFace checkpoint directory of the same weights loads to the same tensors
    d = rerank_cases.hf_model_dir(str(tmp_path / kind), cfg, rerank_cases.TINY[kind]["seed"])
    m2 = CrossEncoder(model_path=d)
    for k, v in m2.state_dict().items():
        assert torch.equal(v, ref[k]), k
    if kind == "roberta":
        assert not any("pooler" in k for k in m2.state_dict())


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_oracle_matches_reference_logits(kind):
    from oracle import cross_encoder as oce
    sd = _reference_sd(kind)
    toks = {k.split("/")[-1]: G[k] for k in G if k.startswith(f"{kind}/tokens/")}
    got = oce.logits(sd, rerank_cases.ORACLE_CFG[kind], toks)
    want = G[f"{kind}/logits"].double()
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max()))


def test_rerank_run_orders_by_score_and_keeps_ties_in_run_order(tmp_path):
    from dpr_scale_b200 import rerank
    # two shards as two ranks wrote them: [n, 1] scores (one label)
    shards = [(["q1", "q1", "q1", "q2"], ["a", "b", "c", "d"], [[0.5], [0.9], [0.5], [0.1]]),
              (["q2", "q0", "q2"], ["e", "f", "g"], [[0.7], [0.3], [0.1]])]
    for r, (q, c, s) in enumerate(shards):
        for what, obj in (("qids", q), ("ctx_ids", c), ("scores", torch.tensor(s))):
            with open(tmp_path / f"{what}_{r:04}.pkl", "wb") as f:
                pickle.dump(obj, f, protocol=4)
    out = rerank.merge(str(tmp_path), run_name="ce", world=2)
    lines = [ln.split() for ln in open(out).read().splitlines()]
    assert [(l[0], l[2], l[3]) for l in lines] == [
        ("q1", "b", "1"), ("q1", "a", "2"), ("q1", "c", "3"),
        ("q2", "e", "1"), ("q2", "d", "2"), ("q2", "g", "3"),
        ("q0", "f", "1")]
    assert all(l[1] == "Q0" and l[5] == "ce" for l in lines)
    assert float(lines[0][4]) == pytest.approx(0.9)
    # [n] scores (several labels) merge the same way
    rows = rerank.write_rerank_run(str(tmp_path / "x.trec"), ["q", "q"], ["u", "v"], [1.0, 2.0])
    assert [ln.split()[2] for ln in open(rows)] == ["v", "u"]


def test_unsupported_configs_raise_value_error():
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    base = rerank_cases.tiny_config("bert")
    minilm = dict(base, hidden_size=384, num_attention_heads=12, intermediate_size=1536)      # head dim 32
    for cfg in (minilm, dict(base, model_type="electra"), dict(base, model_type="deberta-v2"),
                dict(base, num_labels=17), dict(base, hidden_act="relu")):
        with pytest.raises(ValueError):
            CrossEncoder.from_config(cfg)
    # num_labels follows id2label when the config has one
    m = CrossEncoder.from_config(dict(base, num_labels=1, id2label={"0": "a", "1": "b", "2": "c"}))
    assert m.num_labels == 3 and m.transformer.classifier.weight.shape == (3, 128)


def test_rerank_configs_compose():
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=cross_encoder_rerank", "task/model=cross_encoder", "datamodule=cross_encoder_rerank",
                             "task.model.model_path=/m", "+task.output_dir=/o"])
    assert cfg.task._target_ == "dpr_scale_b200.task.cross_encoder_eval_task.RerankCrossEncoderTask"
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.cross_encoder.CrossEncoder"
    assert cfg.datamodule._target_ == "dpr_scale_b200.datamodule.cross_encoder.CrossEncoderRerankDataModule"
    assert cfg.task.transform.model_path == "/m" and cfg.task.output_dir == "/o"
