"""SPLADE and dense (DPR) reranking on the host, against goldens the unmodified reference produced
(tests/golden/make_golden_splade.py):

  * SPLADEEncoder state dicts (tiny BERT / RoBERTa) load strictly with the reference's keys and shapes, the decoder
    stays tied, and RerankDenseRetrieverTask loads reference-keyed checkpoints strictly for HFEncoder and SPLADEEncoder;
  * the float64 oracle (oracle/splade.py) against the reference's SPLADE reps and both encoders' rerank pickles;
  * refusals raise ValueError without a GPU (a grad-enabled forward, sequence lengths, model types, widths) and
    ops.splade_pool_check mirrors dprb_splade_pool_fwd's limits;
  * the YAML groups compose.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests import colbert_cases, rerank_cases, splade_cases
from tests.util import GOLDEN

RAW = np.load(os.path.join(GOLDEN, "splade_small.npz"))
G = {k: torch.from_numpy(RAW[k]) for k in RAW.files if RAW[k].dtype.kind != "U"}
NAMES = list(splade_cases.TINY)


def reference_sd(name):
    """The reference encoder's state dict, rebuilt from the seed; its keys, shapes and checksum are the golden's."""
    sd = splade_cases.tiny_state_dict(name)
    assert sorted(sd) == sorted(RAW[f"{name}/sd_keys"].tolist())
    shapes = dict(zip(RAW[f"{name}/sd_keys"].tolist(), json.loads(str(RAW[f"{name}/sd_shapes"]))))
    assert {k: list(v.shape) for k, v in sd.items()} == shapes
    assert torch.equal(colbert_cases.sd_checksum(sd), G[f"{name}/sd_checksum"]), "seeded weights differ from the golden's"
    return sd


def golden_tokens(name):
    return {k.split("/")[-1]: G[k] for k in G if k.startswith(f"{name}/tokens/")}


@pytest.mark.parametrize("name", NAMES)
def test_reference_state_dict_loads_strictly(name):
    sd = reference_sd(name)
    m = splade_cases.build(name, sd)
    own = m.state_dict()
    assert sorted(own) == sorted(sd)
    for k, v in sd.items():
        assert own[k].shape == v.shape and torch.equal(own[k], v), k
    head = "transformer.cls.predictions." if name == "splade_bert" else "transformer.lm_head."
    body = "transformer.bert." if name == "splade_bert" else "transformer.roberta."
    assert own[head + "decoder.weight"].data_ptr() == own[body + "embeddings.word_embeddings.weight"].data_ptr()
    assert own[head + "decoder.bias"].data_ptr() == own[head + "bias"].data_ptr()
    missing = {k: v for k, v in sd.items() if not k.endswith("decoder.weight")}
    with pytest.raises(RuntimeError):
        m.load_state_dict(missing, strict=True)


@pytest.mark.parametrize("model", list(splade_cases.TASK))
def test_task_loads_reference_keyed_checkpoint(tmp_path, model):
    from dpr_scale_b200.task.dpr_rerank_task import RerankDenseRetrieverTask
    _, _, proj, seed = splade_cases.TASK[model]
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": splade_cases.task_state_dict(model)}, ckpt)
    mdir = splade_cases.model_dir(str(tmp_path / "model"), model, seed)
    mconf = {"_target_": splade_cases.TARGETS[model].replace("dpr_scale.", "dpr_scale_b200."), "model_path": mdir}
    if proj:
        mconf["projection_dim"] = proj
    task = RerankDenseRetrieverTask(checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), transform={},
                                    datamodule=None, optim={}, shared_model=False, model=mconf)
    task.setup("test")
    want = splade_cases.task_state_dict(model)
    got = task.state_dict()
    assert sorted(got) == sorted(want)
    assert all(torch.equal(got[k], v) for k, v in want.items())


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_reps(name):
    from oracle import splade as osp
    kind, _ = splade_cases.TINY[name]
    r = osp.reps(reference_sd(name), rerank_cases.ORACLE_CFG[kind], golden_tokens(name))
    want = G[f"{name}/reps"].double()
    assert r.shape == want.shape
    assert float((r - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max()))
    assert bool((want[-1] == 0).all()) and bool((r[-1] == 0).all())        # no valid token after token 0


def test_pool_contract_equals_reps_on_compacted_rows():
    """oracle.splade.pool on the compacted head transforms equals oracle.splade.reps (the identity the kernel rests on)."""
    from oracle import multivec as om
    from oracle import splade as osp
    from oracle.colbert import _double, hidden_states
    from oracle.encoder import gelu_erf, layer_norm
    name = "splade_bert"
    sd = _double(reference_sd(name))
    cfg = rerank_cases.ORACLE_CFG["bert"]
    toks = golden_tokens(name)
    h = hidden_states(sd, cfg, toks, "transformer.bert.")
    keep = toks["attention_mask"].clone() != 0
    keep[:, 0] = False
    p = "transformer.cls.predictions."
    x = gelu_erf(h[keep] @ sd[p + "transform.dense.weight"].T + sd[p + "transform.dense.bias"])
    x = layer_norm(x, sd[p + "transform.LayerNorm.weight"], sd[p + "transform.LayerNorm.bias"], cfg["ln_eps"])
    off = torch.cat([torch.zeros(1, dtype=torch.long), keep.sum(1).cumsum(0)])
    got = osp.pool(x, sd["transformer.bert.embeddings.word_embeddings.weight"], off, x.shape[1], sd[p + "bias"])
    want = osp.reps(sd, cfg, toks)
    assert om.head_kind(sd) == "bert" and float((got - want).abs().max()) <= 1e-12


@pytest.mark.parametrize("model", list(splade_cases.TASK))
def test_oracle_matches_reference_task_scores(model):
    from oracle import splade as osp
    from tests.test_colbert_cpu import golden_batches
    full = splade_cases.task_state_dict(model)
    cfg = rerank_cases.ORACLE_CFG["bert"]
    enc = osp.dense if model == "hf" else osp.reps
    scores, qids, ctx_ids = [], [], []
    for b in golden_batches():
        q = enc(full, cfg, b["query_ids"], "query_encoder.")
        d = enc(full, cfg, b["contexts_ids"], "context_encoder.")
        scores.append(osp.rerank_score(q, d))
        qids += b["qid"]
        ctx_ids += b["ctx_id"]
    got = torch.cat(scores)
    want = G[f"{model}/pkl/scores"].double()
    assert float((got - want).abs().max()) <= 1e-5 * max(1.0, float(want.abs().max()))
    assert qids == RAW[f"{model}/pkl/qids"].tolist() and ctx_ids == RAW[f"{model}/pkl/ctx_ids"].tolist()


def test_refusals_without_a_gpu():
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.splade_model import SPLADEEncoder
    cfg = colbert_cases.encoder_config("bert")
    with pytest.raises(ValueError):
        SPLADEEncoder.from_config(dict(cfg, model_type="electra"))
    with pytest.raises(ValueError):
        SPLADEEncoder.from_config(dict(cfg, hidden_size=128, num_attention_heads=4))      # head dim 32
    with pytest.raises(ValueError):
        SPLADEEncoder.from_config(dict(cfg, hidden_size=1088, num_attention_heads=17))    # H > 1024
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(0), 2, 12, cfg["vocab_size"], 0)
    m = splade_cases.build("splade_bert")
    with torch.enable_grad():
        with pytest.raises(ValueError):
            m(toks)
    with torch.no_grad():
        with pytest.raises(ValueError):
            m({k: v[:, :1] for k, v in toks.items()})
        long = colbert_cases.seq_tokens(torch.Generator().manual_seed(0), 1, 513, cfg["vocab_size"], 0)
        with pytest.raises(ValueError):
            m(long)
    ops.splade_pool_check(3, 30522, 768, 776, 776, 30522)
    ops.splade_pool_check(1, 1, 8)
    ops.splade_pool_check(1, 50265, 1024)
    for args in ((1, 8, 100), (1, 8, 0), (1, 8, 1032), (1, 8, 64, 60), (1, 8, 64, 68), (1, 8, 64, 64, 56),
                 (1, 8, 64, 64, 72 + 4), (1, 0, 64), (0, 8, 64), (1, 8, 64, 64, 64, 7), (1, 8, 64, None, None, None, -1),
                 (1, 8, 64, None, None, None, 1 << 31)):
        with pytest.raises(ValueError):
            ops.splade_pool_check(*args)


@pytest.mark.parametrize("model", ["splade_model", "hf_model"])
def test_config_composes(model):
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["task=dpr_rerank", f"task/model={model}", "datamodule=multivec_rerank",
                             "task.model.model_path=/m", "+task.checkpoint_path=/c", "+task.output_dir=/o"])
    target = {"splade_model": "models.citadel_models.splade_model.SPLADEEncoder",
              "hf_model": "models.hf_model.HFEncoder"}[model]
    assert cfg.task.model._target_ == "dpr_scale_b200." + target
    assert cfg.task._target_ == "dpr_scale_b200.task.dpr_rerank_task.RerankDenseRetrieverTask"
    assert cfg.datamodule._target_ == "dpr_scale_b200.datamodule.citadel.DenseRetrieverRerankDataModule"
    assert cfg.task.model.dropout == 0.1 and cfg.task.shared_model is False and cfg.task.in_batch_eval is False
    assert cfg.task.checkpoint_path == "/c" and cfg.task.output_dir == "/o"
