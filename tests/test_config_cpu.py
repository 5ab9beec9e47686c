"""CPU tests of the host-side plugin surface: config composition, `_target_` instantiation, C-ABI exports."""
import ctypes
import re
import os

from dpr_scale_b200 import _lib
from dpr_scale_b200.utils.config import compose, instantiate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_compose_defaults_and_overrides():
    cfg = compose("msmarco_baseline", ["task.model.model_path=/tmp/m", "task.warmup_steps=7", "+task.k=3"])
    assert cfg.task._target_ == "dpr_scale_b200.task.dpr_task.DenseRetrieverTask"
    assert cfg.task.model._target_ == "dpr_scale_b200.models.hf_model.HFEncoder"
    assert cfg.task.model.model_path == "/tmp/m"
    assert cfg.task.transform.model_path == "/tmp/m"  # ${task.model.model_path} interpolation
    assert cfg.task.warmup_steps == 7 and cfg.task.k == 3
    assert cfg.task.optim.lr == 2.0e-05 and cfg.task.optim._target_.endswith("FusedAdamW")
    assert cfg.trainer.gradient_clip_val == 2.0 and cfg.datamodule.num_negative == 7


def test_instantiate_task_by_target_without_recursion():
    cfg = compose("config", [])
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert type(task).__name__ == "DenseRetrieverTask"
    assert task.model_conf["_target_"].endswith("HFEncoder")  # stays a config node until setup()
    assert task.shared_model is False and task.in_batch_negatives is True


def test_signatures_match_every_header_prototype():
    """_lib.SIGNATURES binds exactly the entry points include/dprb.h declares, each with the header's return type and
    argument list: a pointer or dprb_stream_t as c_void_p or a ctypes POINTER, int / int64_t / uint64_t / float as
    their ctypes twins.  The built library exports every one of them."""
    scalar = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "float": ctypes.c_float,
              "const char*": ctypes.c_char_p}
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dprb.h")).read(), flags=re.S)
    protos = re.findall(r"^(\w[\w ]*?\**)\s*\b(dprb_\w+)\(([^)]*)\);", header, flags=re.M)
    declared = {name for _, name, _ in protos}
    assert len(declared) == len(protos)
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)

    def is_pointer(t):
        return t is ctypes.c_void_p or (isinstance(t, type) and issubclass(t, ctypes._Pointer))

    bad = []
    for ret, name, params in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        if restype is not scalar.get(ret.strip()):
            bad.append(f"{name}: returns {ret.strip()}, bound as {restype.__name__}")
        params = [] if params.strip() == "void" else [" ".join(p.split()) for p in params.split(",")]
        if len(params) != len(argtypes):
            bad.append(f"{name}: {len(params)} arguments declared, {len(argtypes)} bound")
            continue
        for i, (p, t) in enumerate(zip(params, argtypes)):
            if "*" in p or p.startswith("dprb_stream_t "):
                ok = is_pointer(t)
            else:
                ok = t is scalar.get(p.rsplit(" ", 1)[0])
            if not ok:
                bad.append(f"{name}: argument {i} `{p}` bound as {t.__name__}")
    assert not bad, "\n".join(bad)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert _lib.load().dprb_version() == 101


def test_encoder_rejects_unsupported_configs_and_cpu_execution():
    import pytest
    import torch
    from dpr_scale_b200._lib import DprbError
    from dpr_scale_b200.models.hf_model import HFEncoder
    base = dict(vocab_size=64, hidden_size=128, num_hidden_layers=1, num_attention_heads=2, intermediate_size=256,
                max_position_embeddings=40)
    with pytest.raises(ValueError):   # head_dim must be 64
        HFEncoder.from_config({**base, "num_attention_heads": 4})
    with pytest.raises(ValueError):   # erf-GELU only
        HFEncoder.from_config({**base, "hidden_act": "relu"})
    with pytest.raises(ValueError):   # absolute position embeddings only
        HFEncoder.from_config({**base, "position_embedding_type": "relative_key"})
    enc = HFEncoder.from_config(base, dropout=0.0)
    with pytest.raises(DprbError):    # no CPU fallback: the product path fails loudly without a CUDA device
        enc({"input_ids": torch.ones(2, 4, dtype=torch.long)})
    with pytest.raises(FileNotFoundError):  # hub names cannot be resolved offline: must be a local directory
        HFEncoder(model_path="bert-base-uncased")


def test_state_dict_roundtrip_keeps_arena_views():
    import torch
    from dpr_scale_b200.models.hf_model import HFEncoder
    base = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                max_position_embeddings=40)
    a, b = HFEncoder.from_config(base, seed=1), HFEncoder.from_config(base, seed=2)
    b.load_state_dict(a.state_dict())
    assert torch.equal(a.master, b.master)
    # parameters are views of ONE flat arena (Q, K, V adjacent => fused [3H, H] operand)
    lay = b.transformer.layout
    q_off = lay.by_name["encoder.layer.0.attention.self.query.weight"][1]
    k_off = lay.by_name["encoder.layer.0.attention.self.key.weight"][1]
    assert k_off - q_off == 128 * 128
    w = b.transformer.encoder.layer._modules["0"].attention.self.query.weight
    assert w.data_ptr() == b.master.data_ptr() + 4 * q_off


def test_generation_tasks_host_logic(tmp_path):
    """Writers of the two embedding-generation tasks on CPU tensors (no encoder involved): file names, pickle protocol 4
    of ONE fp32 tensor, default query path = <ctx_embeddings_dir>/query_reps.pkl (dpr_eval_task.py:36-49, :52-84)."""
    import pickle

    import torch

    from dpr_scale_b200.task.dpr_eval_task import GenerateEmbeddingsTask, GenerateQueryEmbeddingsTask
    kw = dict(transform={}, model={}, datamodule=None, optim={})
    t = GenerateEmbeddingsTask(ctx_embeddings_dir=str(tmp_path / "emb"), checkpoint_path="", **kw)
    t._encode = lambda tokens: tokens                 # stand-in for the encoder: the "tokens" are the embeddings
    # more batches than ring slots (pinned buffers are reused), ragged batch sizes
    parts = [torch.arange(3 * (2 + i % 3), dtype=torch.float32).view(-1, 3) + 10 * i for i in range(2 * t.RING + 3)]
    rows = [t.test_step({"contexts_ids": p}, i) for i, p in enumerate(parts)]
    assert rows == [p.shape[0] for p in parts]        # nothing but row counts is kept per batch
    path = t.test_epoch_end(rows)
    assert path.endswith("emb/reps_0000.pkl")
    raw = open(path, "rb").read()
    assert raw[:2] == b"\x80\x04"                                  # pickle protocol 4
    assert torch.equal(pickle.loads(raw), torch.cat(parts))
    q = GenerateQueryEmbeddingsTask(ctx_embeddings_dir=str(tmp_path / "emb"), checkpoint_path="", **kw)
    q._encode = lambda tokens: tokens
    assert q.query_emb_output_path == str(tmp_path / "emb" / "query_reps.pkl")
    out = q.test_epoch_end([q.test_step({"query_ids": p}, i) for i, p in enumerate(parts[:3])])
    assert torch.equal(pickle.load(open(out, "rb")), torch.cat(parts[:3]))
    q2 = GenerateQueryEmbeddingsTask(ctx_embeddings_dir=str(tmp_path / "emb"), checkpoint_path="",
                                     query_emb_output_path=str(tmp_path / "x" / "q.pkl"), **kw)
    q2._encode = lambda tokens: tokens
    q2.test_step({"query_ids": parts[0]}, 0)
    assert q2.test_epoch_end([2]) == str(tmp_path / "x" / "q.pkl")
    assert torch.equal(pickle.load(open(tmp_path / "x" / "q.pkl", "rb")), parts[0])


def test_generation_configs_compose():
    from dpr_scale_b200.utils.config import compose
    cfg = compose("config", ["datamodule=generate", "datamodule.test_path=/tmp/p.tsv", "task.model.model_path=/m",
                             "+task.ctx_embeddings_dir=/out"])
    assert cfg.datamodule._target_.endswith("DenseRetrieverPassagesDataModule") and cfg.datamodule.use_title is True
    assert cfg.datamodule.test_path == "/tmp/p.tsv" and cfg.task.ctx_embeddings_dir == "/out"
    assert "train_path" not in cfg.datamodule
    cfg = compose("config", ["datamodule=generate_query_emb", "datamodule.test_path=/tmp/q.tsv",
                             "+datamodule.trec_format=true"])
    assert cfg.datamodule._target_.endswith("DenseRetrieverQueriesDataModule") and cfg.datamodule.trec_format is True
    assert cfg.task.transform._target_ == "dpr_scale_b200.transforms.hf_transform.HFTransform"
    assert cfg.task.transform.model_path == cfg.task.model.model_path


def test_generation_scripts_wire_task_transform_and_datamodule(tmp_path, monkeypatch):
    """generate_embeddings / generate_query_embeddings up to the trainer call: config composition with the reference's
    override syntax, `_target_` swap, transform and datamodule instantiation (the encoder itself needs a GPU)."""
    from transformers import BertConfig

    from dpr_scale_b200 import generate_embeddings as GE
    from dpr_scale_b200 import generate_query_embeddings as GQ
    model = tmp_path / "model"
    model.mkdir()
    BertConfig(vocab_size=12, hidden_size=16, num_hidden_layers=1, num_attention_heads=1,
               intermediate_size=16).save_pretrained(model)
    (model / "vocab.txt").write_text("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "a", "b", "c", "d", "e", "f", "g"]) + "\n")
    (tmp_path / "p.tsv").write_text("id\ttext\ttitle\n" + "".join(f"{i}\ta b c\td e\n" for i in range(5)))
    (tmp_path / "q.tsv").write_text("".join(f"q{i}\tf g a\n" for i in range(3)))
    seen = {}

    class StubTrainer:
        def __init__(self, **kw):
            pass

        def test(self, task, datamodule):
            seen["task"] = type(task).__name__
            seen["dm"] = type(datamodule).__name__
            datamodule.device_prefetch = False
            seen["batches"] = [b for b in datamodule.test_dataloader()]
            seen["out"] = getattr(task, "query_emb_output_path", None) or task.ctx_embeddings_dir
            return seen
    monkeypatch.setattr(GE, "Trainer", StubTrainer)
    common = [f"task.model.model_path={model}", f"+task.ctx_embeddings_dir={tmp_path / 'emb'}", "+task.checkpoint_path="]
    GE.main(["-m", "--config-name", "msmarco_baseline.yaml", "datamodule=generate",
             f"datamodule.test_path={tmp_path / 'p.tsv'}", "datamodule.test_batch_size=2"] + common)
    assert seen["task"] == "GenerateEmbeddingsTask" and seen["dm"] == "DenseRetrieverPassagesDataModule"
    assert len(seen["batches"]) == 3 and seen["batches"][0]["corpus_ids"] == ["0", "1"]
    assert seen["batches"][0]["contexts_ids"]["input_ids"][0].tolist() == [2, 8, 9, 3, 5, 6, 7, 3]   # [CLS] d e [SEP] a b c [SEP]
    GQ.main(["datamodule=generate_query_emb", f"datamodule.test_path={tmp_path / 'q.tsv'}", "+datamodule.trec_format=true"]
            + common)
    assert seen["task"] == "GenerateQueryEmbeddingsTask" and seen["dm"] == "DenseRetrieverQueriesDataModule"
    assert seen["out"] == str(tmp_path / "emb" / "query_reps.pkl")
    assert seen["batches"][0]["query_ids"]["input_ids"].tolist() == [[2, 10, 11, 5, 3]] * 3


def test_committed_bench_line_has_the_contract_keys():
    """The bench line recorded in profiles/ (a real H100 run of `python bench.py`) carries every key of the bench
    contract, with consistent values - guards the schema against accidental edits of bench.py's output dict."""
    import json
    line = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_default_line.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert k in line, k
    assert line["unit"] == "pairs/s" and line["higher_is_better"] is True and line["scaling"] == "weak"
    assert line["config"]["workload"] == "bert-base_s128_b128_n7" and line["n_gpus"] == 1
    assert abs(line["value"] - 128 / (line["ms_per_step"] / 1e3)) < 1e-6 * line["value"]
    e2e = line["e2e"]
    assert e2e["h2d_bytes_per_step"] > 0 and e2e["d2h_bytes_per_step"] > 0 and e2e["value"] != line["value"]
    rf = line["roofline"]
    assert rf["bound"] == "tensor" and abs(rf["frac"] - rf["achieved"] / rf["peak"]) < 1e-9 and rf["unit"] == "TFLOP/s"
    cb = line["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] > 0
    assert line["gpu_launches"] > 0 and set(line["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}


def test_dragon_and_slurm_configs_compose_like_the_reference():
    """conf/dragon_aws.yaml (BASELINE config 4's recipe) and conf/trainer/slurm*.yaml mirror the reference's files of the
    same names (values from /root/reference/dpr_scale/conf/dragon_aws.yaml:6-35, conf/trainer/slurm.yaml:5-15)."""
    from dpr_scale_b200.utils.config import compose
    cfg = compose("dragon_aws", ["datamodule.corpus_path=c.tsv", "datamodule.train_path=[a.jsonl,b.jsonl]",
                                 "datamodule.val_path=d.jsonl", "datamodule.test_path=d.jsonl", "task.model.model_path=/m"])
    assert cfg.datamodule._target_.endswith("DenseRetrieverMultiJsonlDataModule")
    assert cfg.datamodule.train_path == ["a.jsonl", "b.jsonl"] and cfg.datamodule.batch_size == 64
    assert cfg.datamodule.num_negative == 1 and cfg.datamodule.pos_ctx_sample is True and cfg.datamodule.num_test_negative == 50
    assert cfg.task.optim.lr == 3e-5 and cfg.task.warmup_steps == 10000 and cfg.task.shared_model is False
    assert cfg.trainer.gpus == 8 and cfg.trainer.num_nodes == 4 and cfg.trainer.max_epochs == 20 and cfg.trainer.strategy == "ddp"
    assert cfg.trainer.gradient_clip_val == 2.0 and cfg.trainer.precision == 16
    s = compose("config", ["trainer=slurm", "task.model.model_path=/m"])
    assert s.trainer.strategy == "ddp_sharded" and s.trainer.gpus == 8 and s.trainer.max_epochs == 25
