"""ColBERT (multi-vector) reranking on the host, against goldens the unmodified reference produced
(tests/golden/make_golden_colbert.py):

  * DenseRetrieverRerankDataModule: every batch (qids, ctx ids, separately tokenised questions and passages) equal to
    the reference's collate, and the 2-rank contiguous shard split;
  * ColBERTEncoder state dicts (tiny BERT / RoBERTa, a 128-wide projection or none) load strictly with the reference's
    keys and shapes; the rerank task loads a reference-keyed checkpoint strictly;
  * the float64 oracle against the reference's fp32 expert_repr, its rerank scores for both pools, and the BERT-base
    golden scores;
  * refusals raise ValueError without a GPU: a grad-enabled forward, P % 8 != 0, S < 2, S > 512, an unknown pool;
  * the YAML groups compose, and include/dprb.h defines the two MaxSim pool codes.
"""
import json
import os
import types

import numpy as np
import pytest
import torch

from tests import colbert_cases, rerank_cases
from tests.util import GOLDEN

RAW = np.load(os.path.join(GOLDEN, "colbert_small.npz"))
G = {k: torch.from_numpy(RAW[k]) for k in RAW.files if RAW[k].dtype.kind != "U"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_CFG = {"bert": rerank_cases.ORACLE_CFG["bert"], "roberta": rerank_cases.ORACLE_CFG["roberta"]}


def golden_batches():
    out = []
    for i in range(int(G["n_batches"])):
        b = {"qid": RAW[f"batch{i}/qid"].tolist(), "ctx_id": RAW[f"batch{i}/ctx_id"].tolist()}
        for side in ("query_ids", "contexts_ids"):
            b[side] = {k.split("/")[-1]: G[k] for k in G if k.startswith(f"batch{i}/{side}/")}
        out.append(b)
    return out


def _datamodule(tmp_path, **kw):
    from dpr_scale_b200.datamodule.citadel import DenseRetrieverRerankDataModule
    from dpr_scale_b200.transforms.hf_transform import HFTransform
    tok = rerank_cases.tokenizer_dir(str(tmp_path / "tok"))
    return DenseRetrieverRerankDataModule(transform=HFTransform(tok, max_seq_len=rerank_cases.MAX_LEN),
                                          device_prefetch=False, **rerank_cases.datamodule_kwargs(), **kw)


def reference_sd(name):
    """The reference ColBERTEncoder's state dict, rebuilt from the seed; its keys, shapes and checksum are the golden's."""
    sd = colbert_cases.tiny_state_dict(name)
    assert sorted(sd) == sorted(RAW[f"{name}/sd_keys"].tolist())
    shapes = dict(zip(RAW[f"{name}/sd_keys"].tolist(), json.loads(str(RAW[f"{name}/sd_shapes"]))))
    assert {k: list(v.shape) for k, v in sd.items()} == shapes
    assert torch.equal(colbert_cases.sd_checksum(sd), G[f"{name}/sd_checksum"]), "seeded weights differ from the golden's"
    return sd


@pytest.mark.parametrize("prefetch", [0, 3])
def test_batches_equal_reference_collate(tmp_path, prefetch):
    got, want = list(_datamodule(tmp_path, prefetch_batches=prefetch).test_dataloader()), golden_batches()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g["qid"] == w["qid"] and g["ctx_id"] == w["ctx_id"]
        for side in ("query_ids", "contexts_ids"):
            assert set(g[side]) == set(w[side])
            for k, v in w[side].items():
                assert torch.equal(g[side][k], v), (side, k)


def test_two_rank_shards_are_the_reference_sampler_rows(tmp_path):
    want_rows = [r for b in golden_batches() for r in zip(b["qid"], b["ctx_id"])]
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


@pytest.mark.parametrize("name", list(colbert_cases.TINY))
def test_reference_state_dict_loads_strictly(tmp_path, name):
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    kind, proj, _ = colbert_cases.TINY[name]
    ref = reference_sd(name)
    m = ColBERTEncoder.from_config(json.loads(str(RAW[f"{name}/config"])), projection_dim=proj, seed=5)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.items()}
    m.load_state_dict(ref, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, ref[k]), k
    assert m.dim == (proj or 128)
    # a HuggingFace checkpoint directory of the same body loads to the same transformer tensors
    m2 = ColBERTEncoder(model_path=colbert_cases.model_dir(str(tmp_path / name), name), projection_dim=proj)
    for k, v in m2.state_dict().items():
        if k.startswith("transformer."):
            assert torch.equal(v, ref[k]), k
    if proj:
        assert isinstance(m2.project, torch.nn.Sequential) and len(m2.project) == 1     # Linear only, no LayerNorm


def test_rerank_task_loads_a_reference_keyed_checkpoint_strictly(tmp_path):
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    name = "bert_p128"
    sd = colbert_cases.task_state_dict(name)
    ckpt = str(tmp_path / "x.ckpt")
    torch.save({"state_dict": sd}, ckpt)
    mdir = colbert_cases.model_dir(str(tmp_path / "m"), name)
    task = RerankMultiVecRetrieverTask(
        checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), query_pool="max", transform={}, datamodule=None,
        optim={}, shared_model=False, in_batch_eval=False, query_topk=1, context_topk=1, add_cls=False, tau=1.0,
        model={"_target_": "dpr_scale_b200.models.citadel_models.colbert_model.ColBERTEncoder", "model_path": mdir,
               "projection_dim": 128, "dropout": 0.1})
    task.setup("test")
    got = task.state_dict()
    assert sorted(got) == sorted(sd)
    for k, v in sd.items():
        assert torch.equal(got[k], v), k
    assert task.query_encoder is not task.context_encoder
    bad = dict(sd)
    bad.pop("context_encoder.project.0.bias")
    torch.save({"state_dict": bad}, ckpt)
    task2 = RerankMultiVecRetrieverTask(checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), transform={},
                                        datamodule=None, optim={}, shared_model=False, model=task.model_conf)
    with pytest.raises(RuntimeError):
        task2.setup("test")


@pytest.mark.parametrize("name", list(colbert_cases.TINY))
def test_oracle_matches_reference_expert_repr(name):
    from oracle import colbert as oc
    kind = colbert_cases.TINY[name][0]
    sd = reference_sd(name)
    toks = {k.split("/")[-1]: G[k] for k in G if k.startswith(f"{name}/tokens/")}
    got = oc.expert_repr(sd, ORACLE_CFG[kind], toks)
    want = G[f"{name}/expert_repr"].double()
    assert got.shape == want.shape and bool((want[toks["attention_mask"][:, 1:] == 0] == 0).all())
    assert float((got - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max()))


def oracle_scores(name, pool):
    """The float64 oracle over the fixture run's golden batches with the task's two encoders."""
    from oracle import colbert as oc
    kind = colbert_cases.TINY[name][0]
    sd = colbert_cases.task_state_dict(name)
    out = []
    for b in golden_batches():
        q = oc.expert_repr(sd, ORACLE_CFG[kind], b["query_ids"], prefix="query_encoder.")
        d = oc.expert_repr(sd, ORACLE_CFG[kind], b["contexts_ids"], prefix="context_encoder.")
        out.append(oc.maxsim(q, d, pool))
    return torch.cat(out)


@pytest.mark.parametrize("name", colbert_cases.TASK_KINDS)
@pytest.mark.parametrize("pool", colbert_cases.POOLS)
def test_oracle_matches_reference_rerank_scores(name, pool):
    want = G[f"{name}/{pool}/pkl/scores"]
    assert want.dtype == torch.float32 and want.dim() == 1
    got = oracle_scores(name, pool)
    assert float((got - want.double()).abs().max()) <= 1e-5 * float(want.abs().max())


@pytest.mark.parametrize("pool", colbert_cases.POOLS)
def test_oracle_matches_bert_base_golden(pool):
    from oracle import colbert as oc
    raw = np.load(os.path.join(GOLDEN, "colbert_bert_base.npz"))
    sd, cfg = colbert_cases.bert_base_state_dict()
    assert torch.equal(colbert_cases.sd_checksum(sd), torch.from_numpy(raw["checksum"]))
    q = {k: torch.from_numpy(raw[f"query/{k}"]) for k in ("input_ids", "token_type_ids", "attention_mask")}
    d = {k: torch.from_numpy(raw[f"passage/{k}"]) for k in ("input_ids", "token_type_ids", "attention_mask")}
    ocfg = {"layers": 12, "heads": 12, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}
    got = oc.maxsim(oc.expert_repr(sd, ocfg, q), oc.expert_repr(sd, ocfg, d), pool)
    want = torch.from_numpy(raw[f"{pool}/scores"]).double()
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())
    assert float(raw[f"{pool}/amp_max_abs"]) > 0


def test_maxsim_oracle_keeps_the_padding_quirk():
    from oracle import colbert as oc
    q = torch.tensor([[[0.0, 0.0], [1.0, 0.0], [0.5, 0.5]]])         # token 0 is skipped
    d = torch.tensor([[[9.0, 9.0], [-1.0, 0.0], [-2.0, -1.0], [5.0, 5.0]]])
    dm = torch.tensor([[1, 1, 1, 0]])                                  # the last passage token is padding
    qm = torch.tensor([[1, 1, 0]])                                     # so is the last query token
    # row 1: max(-1, -2, 0 [padded]) = 0; row 2 masked: 0
    assert oc.maxsim_tokens(q, d, qm, dm, [0], "sum").tolist() == [0.0]
    assert oc.maxsim_tokens(q, d, qm, dm, [0], "max").tolist() == [0.0]
    assert oc.maxsim_tokens(q, d, torch.ones(1, 3), torch.ones(1, 4), [0], "sum").tolist() == [5.0 + 5.0]


# ------------------------------------------------------------------ refusals without a GPU
def test_refusals_raise_value_error_without_a_gpu(tmp_path):
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    cfg = colbert_cases.encoder_config("bert")
    m = ColBERTEncoder.from_config(cfg, projection_dim=128)
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(0), 2, 8, cfg["vocab_size"], 0)
    with torch.enable_grad(), pytest.raises(ValueError, match="forward only"):
        m(toks)
    with torch.no_grad():
        for S in (1, 513):
            bad = {k: torch.zeros(2, S, dtype=torch.long) for k in toks}
            with pytest.raises(ValueError):
                m(bad)
    for proj in (100, 1032):
        with pytest.raises(ValueError):
            ColBERTEncoder.from_config(cfg, projection_dim=proj)
    with pytest.raises(ValueError):                     # head dim 32
        ColBERTEncoder.from_config(dict(cfg, hidden_size=384, num_attention_heads=12, intermediate_size=1536))
    bf = torch.bfloat16
    for q, d in (((2, 8, 100), (3, 8, 100)), ((2, 1, 64), (3, 8, 64)), ((2, 8, 64), (3, 513, 64)),
                 ((2, 8, 1032), (3, 8, 1032))):
        with pytest.raises(ValueError):
            ops.maxsim(torch.zeros(q, dtype=bf), torch.zeros(d, dtype=bf), None, None, torch.zeros(3, dtype=torch.int32))
    with pytest.raises(ValueError):                     # query index out of range
        ops.maxsim(torch.zeros(2, 8, 64, dtype=bf), torch.zeros(3, 8, 64, dtype=bf), None, None, torch.tensor([0, 1, 2]))
    with pytest.raises(ValueError):
        ops.maxsim(torch.zeros(2, 8, 64, dtype=bf), torch.zeros(3, 8, 64, dtype=bf), None, None, torch.zeros(3),
                   pool="mean")
    task = RerankMultiVecRetrieverTask(checkpoint_path="", output_dir=str(tmp_path), query_pool="mean", transform={},
                                       datamodule=None, optim={}, model={})
    with pytest.raises(NotImplementedError):
        task._scores({"qid": [], "query_ids": {}, "contexts_ids": {}})


def test_multivec_configs_compose():
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=multivec_rerank", "task/model=colbert_model", "datamodule=multivec_rerank",
                             "task.model.model_path=/m", "+task.checkpoint_path=/c", "+task.output_dir=/o",
                             "+task.query_pool=max"])
    assert cfg.task._target_ == "dpr_scale_b200.task.citadel_eval_task.RerankMultiVecRetrieverTask"
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models.colbert_model.ColBERTEncoder"
    assert cfg.task.model.projection_dim == 128 and cfg.task.shared_model is False
    assert cfg.datamodule._target_ == "dpr_scale_b200.datamodule.citadel.DenseRetrieverRerankDataModule"
    assert cfg.task.transform.model_path == "/m" and cfg.task.output_dir == "/o" and cfg.task.checkpoint_path == "/c"


def test_maxsim_pool_defines():
    header = open(os.path.join(ROOT, "include", "dprb.h")).read()
    assert "#define DPRB_MAXSIM_SUM 0" in header and "#define DPRB_MAXSIM_MAX 1" in header
