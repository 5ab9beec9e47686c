"""Distillation and DrBoost host logic vs goldens of the UNMODIFIED reference (tests/golden/make_golden_distill.py ->
distill_small.npz): DPRDistillJsonlDataModule batches bit for bit (synchronous and threaded loaders), malformed rows,
the float64 oracle, configs, checkpoint key names, weak-checkpoint loading and distillation checkpoints in
generate_query_embeddings."""
import json
import os

import numpy as np
import pytest
import torch

from dpr_scale_b200.datamodule.dpr import DPRDistillJsonlDataModule
from dpr_scale_b200.transforms.dpr_distill_transform import DPRDistillTransform
from dpr_scale_b200.transforms.hf_transform import HFTransform
from oracle import distill as odist
from tests import distill_cases
from tests.util import BERT_TINY_CFG, sub

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "golden", "data")
JSONL = os.path.join(DATA, "distill.jsonl")
CASES = {"a": dict(batch_size=3, pos_ctx_sample=True),
         "b": dict(batch_size=4, val_batch_size=5, test_batch_size=6, pos_ctx_sample=False)}
CFG = distill_cases.CFG


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "distill_small.npz"))


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    from transformers import BertConfig
    d = tmp_path_factory.mktemp("tok")
    vocab = open(os.path.join(DATA, "vocab.txt")).read()
    BertConfig(vocab_size=len(vocab.split()), hidden_size=16, num_hidden_layers=1, num_attention_heads=1,
               intermediate_size=16).save_pretrained(d)
    (d / "vocab.txt").write_text(vocab)
    return str(d)


def _tensors(gold):
    """The numeric arrays of the golden file as tensors (the assertion messages are strings)."""
    return {k: torch.from_numpy(gold[k]) for k in gold.files if gold[k].dtype.kind != "U"}


def _model_conf(projection_dim=None):
    return {"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": CFG, "dropout": 0.0,
            "projection_dim": projection_dim}


@pytest.mark.parametrize("prefetch,fast", [(0, False), (0, True), (3, True)])
@pytest.mark.parametrize("case", sorted(CASES))
def test_batches_equal_reference(gold, model_dir, case, prefetch, fast):
    import random
    tf = HFTransform(model_path=model_dir, max_seq_len=24)
    dm = DPRDistillJsonlDataModule(transform=tf, train_path=JSONL, val_path=JSONL, test_path=JSONL,
                                   prefetch_batches=prefetch, device_prefetch=False, fast_tokenize=fast, **CASES[case])
    random.seed(5)
    for stage, loader in (("train", dm.train_dataloader()), ("valid", dm.val_dataloader()),
                          ("test", dm.test_dataloader())):
        want = int(gold[f"data/{case}/{stage}/num_batches"])
        assert len(loader) == want
        n = 0
        for i, batch in enumerate(loader):
            prefix = f"data/{case}/{stage}/{i}"
            names = sorted(k.split("/")[-1] for k in gold.files if k.startswith(prefix + "/query_ids/"))
            assert names == sorted(batch["query_ids"].keys())
            for k in names:
                assert np.array_equal(batch["query_ids"][k].numpy(), gold[f"{prefix}/query_ids/{k}"]), (prefix, k)
            tv = batch["target_vectors"]
            assert tv.dtype == torch.float32 and tv.shape[0] == batch["query_ids"]["input_ids"].shape[0]
            assert np.array_equal(tv.numpy(), gold[f"{prefix}/target_vectors"]), prefix
            n += 1
        assert n == want


def test_target_values_round_once_like_torch_tensor():
    """Every parsed value is torch.Tensor(list_of_python_floats) of the row, bit for bit."""
    rows = open(JSONL, "rb").read().splitlines()
    t = DPRDistillTransform(text_transform=torch.nn.Identity())
    _, vecs = t.select(rows, "test")
    for i, raw in enumerate(rows):
        row = json.loads(raw)
        assert np.array_equal(vecs[2 * i], torch.Tensor(row["ctx_target_vectors"][:1])[0].numpy())
        assert np.array_equal(vecs[2 * i + 1], torch.Tensor(row["qry_target_vector"]).numpy())


@pytest.mark.parametrize("name", ["no_pos", "not_vectors"])
def test_malformed_rows_fail_as_in_reference(gold, name):
    t = DPRDistillTransform(text_transform=torch.nn.Identity())
    with pytest.raises(AssertionError) as e:
        t.select([str(gold[f"data/malformed/{name}/row"])], "train")
    assert str(e.value) == str(gold[f"data/malformed/{name}/message"])


def test_oracle_agrees_with_reference_goldens(gold):
    g = _tensors(gold)
    from oracle import encoder as oenc
    sd = {k: v.double().requires_grad_(True)
          for k, v in distill_cases.encoder_state(distill_cases.CFG, distill_cases.TASK_SEED).items()}
    q = oenc.encode(sd, BERT_TINY_CFG, sub(g, "task/train/query_ids/"))
    loss, dq = odist.sqerr(q, g["task/train/target_vectors"])
    assert abs(float(loss) - float(g["task/train/loss"])) <= 1e-5 * float(g["task/train/loss"])
    q.backward(dq)
    ref = sub(g, "task/grad/")
    assert len(ref) >= 25
    for k, r in ref.items():
        got = sd[k].grad
        assert float((got - r.double()).norm()) <= 1e-3 * float(r.double().norm()) + 1e-7, k
    outs = []
    for i in range(2):
        qr, tv = g[f"task/eval/{i}/query_repr"], g[f"task/eval/{i}/target_vectors"]
        l64, _ = odist.sqerr(qr, tv)
        assert abs(float(l64) - float(g[f"task/eval/{i}/loss"])) <= 1e-5 * float(l64)
        m = odist.rank_metrics(odist.eval_scores(qr, tv).numpy(), np.arange(tv.shape[0]))
        assert m[0] == int(g[f"task/eval/{i}/rank"]) and m[2] == int(g[f"task/eval/{i}/score"])
        assert abs(m[1] - float(g[f"task/eval/{i}/mrr"])) <= 1e-9
        outs.append(((int(g[f"task/eval/{i}/rank"]), float(g[f"task/eval/{i}/mrr"]), float(g[f"task/eval/{i}/score"])),
                     qr.shape[0], tv.shape[0], g[f"task/eval/{i}/loss"]))
    for k, v in odist.epoch_metrics(outs).items():
        assert abs(v - float(g["task/metrics/" + k])) <= 1e-6 * max(1.0, abs(v)), k


def test_configs_compose_and_instantiate(model_dir):
    from dpr_scale_b200.utils.config import compose, instantiate
    cfg = compose("config", ["task=dpr_distill", "datamodule=dpr_distill", f"datamodule.train_path={JSONL}",
                             f"datamodule.val_path={JSONL}", f"datamodule.test_path={JSONL}",
                             f"task.model.model_path={model_dir}", "datamodule.device_prefetch=false"])
    assert cfg.task._target_.endswith("DPRDistillTask")
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert type(task).__name__ == "DPRDistillTask" and task.k == 1 and task.fp16_grads is False
    dm = instantiate(cfg.datamodule, transform=instantiate(cfg.task.transform))
    assert isinstance(dm, DPRDistillJsonlDataModule) and dm.drboost_distill_transform.pos_ctx_sample
    cfg = compose("config", ["task=drboost", "+task.checkpoint_paths=[/x/a.ckpt,b.ckpt]"])
    assert cfg.task.checkpoint_paths == ["/x/a.ckpt", "b.ckpt"]
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert type(task).__name__ == "DrBoostTask" and task.checkpoint_paths == ["/x/a.ckpt", "b.ckpt"]


@pytest.mark.parametrize("projection_dim", [None, 32])
def test_distill_checkpoint_keys(gold, projection_dim):
    from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask, encoder_out_dim
    task = DPRDistillTask(transform={}, model=_model_conf(projection_dim), datamodule=None, optim={})
    task.setup("fit")
    keys = set(task.state_dict())
    assert all(k.startswith("query_encoder.transformer.") or k.startswith("query_encoder.project.") for k in keys)
    ref_keys = {k for k in gold["task/state_dict_keys"].tolist() if not k.endswith("position_ids")}
    assert {k for k in keys if not k.startswith("query_encoder.project.")} == ref_keys
    assert any(k.startswith("query_encoder.project.") for k in keys) == bool(projection_dim)
    assert encoder_out_dim(task.query_encoder) == (projection_dim or 128)


def test_target_width_mismatch_raises_before_gpu_work():
    from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask
    task = DPRDistillTask(transform={}, model=_model_conf(32), datamodule=None, optim={})
    task.setup("fit")
    batch = {"query_ids": {"input_ids": torch.ones(2, 4, dtype=torch.long)}, "target_vectors": torch.zeros(2, 128)}
    with pytest.raises(ValueError, match="target width"):
        task.training_step(batch, 0)


def _weak_checkpoint(tmp_path, name, seed, shared_model=False, projection_dim=None):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    torch.manual_seed(seed)
    t = DenseRetrieverTask(transform={}, model=_model_conf(projection_dim), datamodule=None, optim={},
                           shared_model=shared_model)
    t.setup("fit")
    with torch.no_grad():
        g = torch.Generator().manual_seed(seed)
        for p in t.parameters():
            p.add_(0.01 * torch.randn(p.shape, generator=g))
    path = str(tmp_path / name)
    torch.save(ModelCheckpoint._payload(t, 0, 0), path)
    return path, t


def test_drboost_loads_checkpoint_list(tmp_path):
    from dpr_scale_b200.task.drboost_task import DrBoostTask
    a, ta = _weak_checkpoint(tmp_path, "a.ckpt", 1)
    b, tb = _weak_checkpoint(tmp_path, "b.ckpt", 2, shared_model=True, projection_dim=16)
    task = DrBoostTask(checkpoint_paths=[a, b], transform={}, model={}, datamodule=None, optim={})
    task.setup("test")
    assert len(task.weak_encoders) == 2
    for weak, ref in zip(task.weak_encoders, (ta, tb)):
        assert weak.shared_model == ref.shared_model
        got, want = weak.state_dict(), ref.state_dict()
        assert set(got) == set(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert task.weak_encoders[1].query_encoder is task.weak_encoders[1].context_encoder
    assert task.query_encoder is task.weak_encoders[0].query_encoder
    assert task.configure_optimizers() is None


def test_drboost_missing_or_corrupt_checkpoint(tmp_path):
    from dpr_scale_b200.task.drboost_task import DrBoostTask
    a, _ = _weak_checkpoint(tmp_path, "a.ckpt", 1)
    missing = str(tmp_path / "nope.ckpt")
    with pytest.raises(FileNotFoundError, match="nope.ckpt"):
        DrBoostTask(checkpoint_paths=[a, missing], transform={}, model={}, datamodule=None, optim={}).setup("test")
    bad = tmp_path / "bad.ckpt"
    bad.write_bytes(b"not a checkpoint at all")
    with pytest.raises(RuntimeError, match="bad.ckpt"):
        DrBoostTask(checkpoint_paths=[str(bad)], transform={}, model={}, datamodule=None, optim={}).setup("test")
    with pytest.raises(ValueError, match="checkpoint_paths"):
        DrBoostTask(transform={}, model={}, datamodule=None, optim={}).setup("test")


def _query_dump_task(tmp_path, ckpt):
    from dpr_scale_b200.task.dpr_eval_task import GenerateQueryEmbeddingsTask
    return GenerateQueryEmbeddingsTask(ctx_embeddings_dir=str(tmp_path / "out"), checkpoint_path=ckpt, transform={},
                                       model=_model_conf(32), datamodule=None, optim={}, shared_model=False)


def test_distill_checkpoint_drives_query_embeddings(tmp_path):
    from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    d = DPRDistillTask(transform={}, model=_model_conf(32), datamodule=None, optim={})
    d.setup("fit")
    with torch.no_grad():
        for p in d.parameters():
            p.add_(0.01)
    path = str(tmp_path / "distill.ckpt")
    payload = ModelCheckpoint._payload(d, 0, 0)
    torch.save(payload, path)
    task = _query_dump_task(tmp_path, path)
    task.setup("test")
    got = task.query_encoder.state_dict()
    for k, v in d.query_encoder.state_dict().items():
        assert torch.equal(got[k], v), k
    payload["state_dict"]["query_encoder.extra"] = torch.zeros(1)
    torch.save(payload, path)
    with pytest.raises(RuntimeError, match="query_encoder.extra"):
        _query_dump_task(tmp_path, path).setup("test")
    del payload["state_dict"]["query_encoder.extra"]
    del payload["state_dict"]["query_encoder.project.0.bias"]
    torch.save(payload, path)
    with pytest.raises(RuntimeError, match="project.0.bias"):
        _query_dump_task(tmp_path, path).setup("test")
