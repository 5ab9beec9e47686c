"""COIL / CITADEL reranking on the host, against goldens the unmodified reference produced
(tests/golden/make_golden_multivec.py):

  * COILEncoder / CITADELEncoder state dicts (tiny BERT / RoBERTa) load strictly with the reference's keys and shapes,
    the CITADEL decoder stays tied to the word embeddings and the head bias, and the rerank task loads a
    reference-keyed checkpoint strictly;
  * the float64 oracle (oracle/multivec.py) against the reference's expert_repr, ids, weights and cls_repr, and against
    its rerank scores for both pools;
  * refusals raise ValueError without a GPU: a grad-enabled forward, topk > 8, P or Pc out of range, an unsupported
    model type;
  * the YAML groups compose.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests import colbert_cases, multivec_cases, rerank_cases
from tests.util import GOLDEN

RAW = np.load(os.path.join(GOLDEN, "multivec_small.npz"))
G = {k: torch.from_numpy(RAW[k]) for k in RAW.files if RAW[k].dtype.kind != "U"}
NAMES = list(multivec_cases.TINY)


def reference_sd(name):
    """The reference encoder's state dict, rebuilt from the seed; its keys, shapes and checksum are the golden's."""
    sd = multivec_cases.tiny_state_dict(name)
    assert sorted(sd) == sorted(RAW[f"{name}/sd_keys"].tolist())
    shapes = dict(zip(RAW[f"{name}/sd_keys"].tolist(), json.loads(str(RAW[f"{name}/sd_shapes"]))))
    assert {k: list(v.shape) for k, v in sd.items()} == shapes
    assert torch.equal(colbert_cases.sd_checksum(sd), G[f"{name}/sd_checksum"]), "seeded weights differ from the golden's"
    return sd


@pytest.mark.parametrize("name", NAMES)
def test_reference_state_dict_loads_strictly(name):
    sd = reference_sd(name)
    m = multivec_cases.build(name, sd)
    own = m.state_dict()
    assert sorted(own) == sorted(sd)
    for k, v in sd.items():
        assert own[k].shape == v.shape and torch.equal(own[k], v), k
    if name.startswith("citadel"):
        head = "transformer.cls.predictions." if name == "citadel_bert" else "transformer.lm_head."
        body = "transformer.bert." if head.endswith("predictions.") else "transformer.roberta."
        assert own[head + "decoder.weight"].data_ptr() == own[body + "embeddings.word_embeddings.weight"].data_ptr()
        assert own[head + "decoder.bias"].data_ptr() == own[head + "bias"].data_ptr()
        with torch.no_grad():                          # the tie holds after a load that changes the embeddings
            sd2 = dict(sd)
            sd2[body + "embeddings.word_embeddings.weight"] = sd[body + "embeddings.word_embeddings.weight"] * 2
            m.load_state_dict(sd2, strict=True)
        assert torch.equal(m.state_dict()[head + "decoder.weight"], sd2[body + "embeddings.word_embeddings.weight"])
        missing = {k: v for k, v in sd.items() if not k.endswith("decoder.weight")}
        with pytest.raises(RuntimeError):
            m.load_state_dict(missing, strict=True)


@pytest.mark.parametrize("name", NAMES)
def test_task_loads_reference_keyed_checkpoint(tmp_path, name):
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    model, kind, proj, cls_proj, _ = multivec_cases.TINY[name]
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(name)}, ckpt)
    mdir = multivec_cases.model_dir(str(tmp_path / "model"), name)
    task = RerankMultiVecRetrieverTask(
        checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), add_cls=True, query_topk=2, context_topk=1,
        transform={}, datamodule=None, optim={}, shared_model=False,
        model=dict({"_target_": "dpr_scale_b200.models.citadel_models." + multivec_cases.TARGETS[model],
                    "model_path": mdir}, **multivec_cases.ctor_kwargs(model, proj, cls_proj)))
    task.setup("test")
    want = multivec_cases.task_state_dict(name)
    got = task.state_dict()
    assert sorted(got) == sorted(want)
    assert all(torch.equal(got[k], v) for k, v in want.items())
    assert (task.add_cls, task.query_topk, task.context_topk) == (True, 2, 1)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_outputs(name):
    from oracle import multivec as om
    model, kind, _, _, _ = multivec_cases.TINY[name]
    sd = reference_sd(name)
    toks = {k.split("/")[-1]: G[k] for k in G if k.startswith(f"{name}/tokens/")}
    cfg = rerank_cases.ORACLE_CFG[kind]
    for topk in ((1, 2) if model == "citadel" else (1,)):
        for add_cls in (0, 1):
            pre = f"{name}/k{topk}/cls{add_cls}/"
            if model == "coil":
                r = om.coil(sd, cfg, toks, bool(add_cls))
            else:
                r = om.citadel(sd, cfg, toks, topk, bool(add_cls))
            for k in ("expert_repr", "expert_weights", "cls_repr"):
                if pre + k not in G:
                    assert k not in r
                    continue
                want = G[pre + k].double()
                err = float((r[k].double() - want).abs().max())
                assert err <= 1e-4 * max(1.0, float(want.abs().max())), (pre + k, err)
            live = G[pre + "expert_weights"] > 0                       # ids of zero-weight experts are arbitrary
            assert torch.equal(r["expert_ids"].long()[live], G[pre + "expert_ids"].long()[live])


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("pool", multivec_cases.POOLS)
def test_oracle_matches_reference_task_scores(name, pool):
    from oracle import multivec as om
    from tests.test_colbert_cpu import golden_batches
    model, kind, _, _, _ = multivec_cases.TINY[name]
    full = multivec_cases.task_state_dict(name)
    cfg = rerank_cases.ORACLE_CFG[kind]
    qk, ck = multivec_cases.TASK_TOPK
    scores = []
    for b in golden_batches():
        if model == "coil":
            q = om.coil(full, cfg, b["query_ids"], True, "query_encoder.")
            d = om.coil(full, cfg, b["contexts_ids"], True, "context_encoder.")
        else:
            q = om.citadel(full, cfg, b["query_ids"], qk, True, "query_encoder.")
            d = om.citadel(full, cfg, b["contexts_ids"], ck, True, "context_encoder.")
        scores.append(om.expert_score(q["expert_repr"], d["expert_repr"], q["expert_ids"], q["expert_weights"],
                                      d["expert_ids"], d["expert_weights"], pool, q["cls_repr"], d["cls_repr"]))
    got = torch.cat(scores)
    want = G[f"{name}/{pool}/pkl/scores"].double()
    assert float((got - want).abs().max()) <= 1e-4 * max(1.0, float(want.abs().max()))


def test_refusals_without_a_gpu():
    from dpr_scale_b200.models.citadel_models.citadel_model import CITADELEncoder
    from dpr_scale_b200.models.citadel_models.coil_model import COILEncoder
    cfg = colbert_cases.encoder_config("bert")
    for kw in ({"tok_projection_dim": 100}, {"tok_projection_dim": 1032}, {"cls_projection_dim": 60},
               {"cls_projection_dim": 2048}):
        with pytest.raises(ValueError):
            CITADELEncoder.from_config(cfg, **kw)
    for kw in ({"projection_dim": 100}, {"cls_projection_dim": 60}, {"cls_projection_dim": 1032}):
        with pytest.raises(ValueError):
            COILEncoder.from_config(cfg, **kw)
    with pytest.raises(ValueError):
        CITADELEncoder.from_config(dict(cfg, model_type="electra"))
    with pytest.raises(ValueError):
        CITADELEncoder.from_config(dict(cfg, hidden_size=128, num_attention_heads=4))     # head dim 32
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(0), 2, 12, cfg["vocab_size"], 0)
    cit = multivec_cases.build("citadel_bert")
    coil = multivec_cases.build("coil_bert")
    with torch.enable_grad():
        with pytest.raises(ValueError):
            cit(toks)
        with pytest.raises(ValueError):
            coil(toks)
    with torch.no_grad():
        with pytest.raises(ValueError):
            cit(toks, topk=9)
        with pytest.raises(ValueError):
            cit(toks, topk=0)
        with pytest.raises(ValueError):
            cit({k: v[:, :1] for k, v in toks.items()})
        with pytest.raises(ValueError):
            coil({k: v[:, :1] for k, v in toks.items()})


@pytest.mark.parametrize("model", ["coil_model", "citadel_model"])
def test_config_composes(model):
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=multivec_rerank", f"task/model={model}", "datamodule=multivec_rerank",
                             "task.model.model_path=/m", "+task.checkpoint_path=/c", "+task.output_dir=/o",
                             "+task.add_cls=true", "+task.query_topk=2"])
    ref = {"coil_model": ("coil_model.COILEncoder", {"projection_dim": 128, "cls_projection_dim": 128}),
           "citadel_model": ("citadel_model.CITADELEncoder", {"tok_projection_dim": 32, "cls_projection_dim": 128})}
    target, dims = ref[model]
    assert cfg.task.model._target_ == "dpr_scale_b200.models.citadel_models." + target
    assert cfg.task._target_ == "dpr_scale_b200.task.citadel_eval_task.RerankMultiVecRetrieverTask"
    for k, v in dims.items():
        assert cfg.task.model[k] == v
    assert cfg.task.model.dropout == 0.1 and cfg.task.add_cls is True and cfg.task.query_topk == 2
