"""Distillation and DrBoost on the H100 kernels:
  * dprb_sqerr_fwd against float64 over rows x widths, contiguous and strided: loss within 1e-5 relative, dx bitwise equal
    to torch's fp32 2 * (x - t), bitwise-repeatable loss;
  * one DPRDistillTask step on the tiny BERT against the reference's golden (loss, every gradient) and its evaluation;
    the same step at BERT-base dimensions, with and without a projection head, against the CPU oracle;
  * DrBoostTask evaluation and embedding dump against the reference's golden (two weak encoders, one projected);
  * end to end: weak checkpoints -> ensemble embeddings -> distillation JSONL -> main.py training -> the distilled
    checkpoint's query embeddings -> run_retrieval against the ensemble's passage embeddings;
  * two ranks (when two GPUs are present): gradients equal the mean of the per-rank oracle gradients.
"""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import distill as odist
from tests import distill_cases
from tests.util import cosine, rel_l2, sub

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "tests", "golden", "data")
CFG = distill_cases.CFG


@pytest.fixture(scope="module")
def g():
    z = np.load(os.path.join(ROOT, "tests", "golden", "distill_small.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files if z[k].dtype.kind != "U"}


def _conf(config=CFG, projection_dim=None, dropout=0.0):
    return {"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": config, "dropout": dropout,
            "projection_dim": projection_dim}


# ------------------------------------------------------------------ the loss kernel
@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("d", [1, 100, 160, 768, 1024])
@pytest.mark.parametrize("rows", [1, 7, 256, 65536])
def test_sqerr_kernel_against_float64(rows, d, strided):
    from dpr_scale_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(rows * 7 + d)
    pad = 3 if strided else 0
    xb = torch.randn(rows, d + pad, device="cuda", generator=gen)
    tb = torch.randn(rows, d + 2 * pad, device="cuda", generator=gen) * 0.5
    x, t = xb[:, :d], tb[:, :d]
    loss, dx = ops.sqerr(x, t)
    want = ((x.double() - t.double()) ** 2).sum()
    assert abs(float(loss[0]) - float(want)) <= 1e-5 * float(want), (float(loss[0]), float(want))
    assert torch.equal(dx, 2 * (x - t))
    again, _ = ops.sqerr(x, t)
    assert torch.equal(again, loss)
    evl, none = ops.sqerr(x, t, want_dx=False)
    assert none is None and torch.equal(evl, loss)


def test_sqerr_empty_and_refusals():
    from dpr_scale_b200 import ops
    loss, dx = ops.sqerr(torch.empty(0, 8, device="cuda"), torch.empty(0, 8, device="cuda"))
    assert float(loss[0]) == 0.0 and dx.shape == (0, 8)
    with pytest.raises(ValueError):
        ops.sqerr(torch.zeros(2, 8, device="cuda"), torch.zeros(2, 9, device="cuda"))
    with pytest.raises(ValueError):
        ops.sqerr(torch.zeros(2, 8, device="cuda", dtype=torch.half), torch.zeros(2, 8, device="cuda", dtype=torch.half))


# ------------------------------------------------------------------ the distillation step
def _distill_task(config=CFG, projection_dim=None, sd=None, dropout=0.0):
    from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask
    task = DPRDistillTask(transform={}, model=_conf(config, projection_dim, dropout), datamodule=None, optim={})
    task.setup("fit")
    if sd is not None:
        task.query_encoder.load_state_dict(sd, strict=False)
    return task.cuda()


def test_tiny_step_and_eval_match_reference_golden(g):
    task = _distill_task(sd=distill_cases.encoder_state(CFG, distill_cases.TASK_SEED))
    task.train()
    batch = {"query_ids": sub(g, "task/train/query_ids/"), "target_vectors": g["task/train/target_vectors"]}
    task.query_encoder.zero_grad()
    loss = task.training_step(batch, 0)
    want = float(g["task/train/loss"])
    assert abs(float(loss.detach()) - want) <= 1e-2 * want, (float(loss.detach()), want)
    assert task.logged["train_loss"] is loss
    loss.backward()
    torch.cuda.synchronize()
    params = dict(task.query_encoder.named_parameters())
    ref = sub(g, "task/grad/")
    top = max(float(r.norm()) for r in ref.values())
    for k, r in ref.items():
        got = params[k].grad.detach().float().cpu()
        if float(r.norm()) < 1e-5 * top:
            # analytically zero (key.bias: softmax is shift invariant): only bound the noise
            assert float(got.norm()) < 1e-2 * top, (k, float(got.norm()), top)
            continue
        assert cosine(got, r) >= 0.999 and rel_l2(got, r) <= 5e-2, (k, cosine(got, r), rel_l2(got, r))
    task.eval()
    outs = []
    with torch.no_grad():
        for i in range(2):
            b = {"query_ids": sub(g, f"task/eval/{i}/query_ids/"), "target_vectors": g[f"task/eval/{i}/target_vectors"]}
            res = task.validation_step(b, i)
            (rank, mrr, score), q, t, l = res
            assert rel_l2(q.cpu(), g[f"task/eval/{i}/query_repr"]) <= 1e-2
            assert rank == int(g[f"task/eval/{i}/rank"]) and score == int(g[f"task/eval/{i}/score"])
            assert abs(float(l) - float(g[f"task/eval/{i}/loss"])) <= 1e-2 * float(g[f"task/eval/{i}/loss"])
            outs.append(res)
        metrics = task.validation_epoch_end(outs)
    for k, v in metrics.items():
        want = float(g["task/metrics/" + k])
        assert abs(float(v) - want) <= 1e-2 * max(1.0, abs(want)), (k, float(v), want)


@pytest.mark.parametrize("projection_dim", [None, 768])
def test_bert_base_step_against_oracle(projection_dim):
    """BERT-base dimensions, 8 questions (16 rows) at S = 32: loss and sampled gradients against the CPU oracle, at the
    real-dimension step tests' tolerances (bf16 GEMMs, fp32 accumulation)."""
    from oracle import encoder as oenc
    cfg = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
               max_position_embeddings=512)
    torch.manual_seed(0)
    task = _distill_task(cfg, projection_dim)
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in task.query_encoder.state_dict().items()}
    gen = torch.Generator().manual_seed(9)
    B, S = 8, 32
    ids = torch.randint(1000, 30000, (B, S), generator=gen)
    am = torch.ones(B, S, dtype=torch.long)
    am[1::2, S // 2:] = 0
    ids[:, 0] = 101
    toks = {"input_ids": (ids * am).repeat_interleave(2, 0), "token_type_ids": torch.zeros(2 * B, S, dtype=torch.long),
            "attention_mask": am.repeat_interleave(2, 0)}
    targets = torch.randn(2 * B, projection_dim or 768, generator=gen)
    task.train()
    task.query_encoder.zero_grad()
    loss = task.training_step({"query_ids": toks, "target_vectors": targets}, 0)
    loss.backward()
    torch.cuda.synchronize()
    ocfg = {"layers": 12, "heads": 12, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}
    q = oenc.encode(sd, ocfg, toks)
    want, dq = odist.sqerr(q, targets, torch.float32)
    q.backward(dq)
    assert abs(float(loss) - float(want)) <= 1e-2 * float(want), (float(loss), float(want))
    params = dict(task.query_encoder.named_parameters())
    names = ["transformer.embeddings.word_embeddings.weight", "transformer.encoder.layer.0.attention.self.query.weight",
             "transformer.encoder.layer.5.intermediate.dense.weight", "transformer.encoder.layer.11.output.dense.bias",
             "transformer.encoder.layer.11.output.LayerNorm.weight"]
    if projection_dim:
        names += ["project.0.weight", "project.1.bias"]
    for k in names:
        got, ref = params[k].grad.detach().float().cpu(), sd[k].grad
        assert cosine(got, ref) >= 0.999 and rel_l2(got, ref) <= 5e-2, (k, cosine(got, ref), rel_l2(got, ref))


# ------------------------------------------------------------------ DrBoost
def _weak_checkpoints(tmp_path):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    paths = []
    wcfg = distill_cases.WEAK_CFG
    for i, (shared, pd, seed_q, seed_c) in enumerate(distill_cases.WEAK):
        t = DenseRetrieverTask(transform={}, model=_conf(wcfg, pd), datamodule=None, optim={}, shared_model=shared)
        t.setup("fit")
        t.query_encoder.load_state_dict(distill_cases.encoder_state(wcfg, seed_q, pd))
        if not shared:
            t.context_encoder.load_state_dict(distill_cases.encoder_state(wcfg, seed_c, pd))
        paths.append(str(tmp_path / f"weak{i}.ckpt"))
        torch.save(ModelCheckpoint._payload(t, 0, 0), paths[-1])
    return paths


def test_drboost_eval_and_dump_match_reference_golden(g, tmp_path):
    from dpr_scale_b200.task.drboost_task import DrBoostGenerateEmbeddingsTask, DrBoostTask
    paths = _weak_checkpoints(tmp_path)
    task = DrBoostTask(checkpoint_paths=paths, transform={}, model={}, datamodule=None, optim={}, in_batch_eval=False)
    task.setup("test")
    task = task.cuda().eval()
    q_ids, c_ids = sub(g, "drboost/query_ids/"), sub(g, "drboost/contexts_ids/")
    with torch.no_grad():
        q, c = task(q_ids, c_ids)
    assert q.shape == g["drboost/query_repr"].shape and c.shape == g["drboost/contexts_repr"].shape
    assert rel_l2(q.cpu(), g["drboost/query_repr"]) <= 1e-2 and rel_l2(c.cpu(), g["drboost/contexts_repr"]) <= 1e-2
    labels = torch.tensor([0, 1, 3, 4, 6])
    batch = {"query_ids": q_ids, "contexts_ids": c_ids, "pos_ctx_indices": labels, "ctx_mask": torch.zeros(7, dtype=torch.bool)}
    with torch.no_grad():
        metrics = task.test_epoch_end([task.test_step(batch, 0)])
    rank, mrr, _ = odist.rank_metrics(odist.eval_scores(q.cpu(), c.cpu()).numpy(), labels.numpy())
    assert abs(metrics["test_avg_rank"] - rank / 5) <= 1e-9 and abs(metrics["test_mrr"] - mrr / 5) <= 1e-6
    dump = DrBoostGenerateEmbeddingsTask(ctx_embeddings_dir=str(tmp_path / "emb"), checkpoint_path=None,
                                         checkpoint_paths=paths, transform={}, model={}, datamodule=None, optim={})
    dump.setup("test")
    dump = dump.cuda().eval()
    dump.test_step({"contexts_ids": c_ids}, 0)
    out = dump.test_epoch_end([7])
    with open(out, "rb") as f:
        reps = pickle.load(f)
    assert reps.shape == c.shape and rel_l2(reps, c.cpu()) <= 1e-5


# ------------------------------------------------------------------ end to end
def _tiny_model_dir(path):
    from transformers import BertConfig, BertModel
    vocab = open(os.path.join(DATA, "vocab.txt")).read()
    torch.manual_seed(3)
    BertModel(BertConfig(vocab_size=len(vocab.split()), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256, max_position_embeddings=40)).save_pretrained(path)
    with open(os.path.join(path, "vocab.txt"), "w") as f:
        f.write(vocab)
    return str(path)


def _run(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return res.stdout


def test_end_to_end_drboost_distill_retrieval(tmp_path):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    mdir = _tiny_model_dir(tmp_path / "model")
    paths = []
    for i, (shared, pd) in enumerate(((False, None), (True, 16))):
        t = DenseRetrieverTask(transform={}, model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder",
                                                    "model_path": mdir, "dropout": 0.0, "projection_dim": pd},
                               datamodule=None, optim={}, shared_model=shared)
        t.setup("fit")
        with torch.no_grad():
            gen = torch.Generator().manual_seed(40 + i)
            for p in t.parameters():
                p.add_(0.02 * torch.randn(p.shape, generator=gen))
        paths.append(str(tmp_path / f"weak{i}.ckpt"))
        torch.save(ModelCheckpoint._payload(t, 0, 0), paths[-1])
    width = 128 + 16
    common = [f"task.model.model_path={mdir}", "task.transform.max_seq_len=32"]
    ens, student = tmp_path / "ensemble", tmp_path / "student"
    drb = ["task=drboost", f"+task.checkpoint_paths=[{','.join(paths)}]", f"+task.ctx_embeddings_dir={ens}"] + common
    passages, questions = os.path.join(DATA, "passages.tsv"), os.path.join(DATA, "questions.tsv")
    _run(["dpr_scale_b200.generate_embeddings", "datamodule=generate", f"datamodule.test_path={passages}",
          "datamodule.test_batch_size=4"] + drb)
    _run(["dpr_scale_b200.generate_query_embeddings", "datamodule=generate_query_emb", f"datamodule.test_path={questions}",
          "+datamodule.trec_format=true", "datamodule.test_batch_size=3"] + drb)
    with open(ens / "reps_0000.pkl", "rb") as f:
        preps = pickle.load(f)
    with open(ens / "query_reps.pkl", "rb") as f:
        qreps = pickle.load(f)
    assert preps.shape == (11, width) and qreps.shape == (7, width)
    jsonl = tmp_path / "distill.jsonl"
    qs = [ln.split("\t")[1] for ln in open(questions).read().splitlines()]
    with open(jsonl, "w") as f:
        for i, q in enumerate(qs):
            f.write(json.dumps({"question": q, "qry_target_vector": qreps[i].tolist(),
                                "ctx_target_vectors": [preps[i].tolist(), preps[i + 1].tolist()]}) + "\n")
    ckdir = tmp_path / "ckpt"
    out = _run(["dpr_scale_b200.main", "task=dpr_distill", "datamodule=dpr_distill", f"datamodule.train_path={jsonl}",
                f"datamodule.val_path={jsonl}", f"datamodule.test_path={jsonl}", "datamodule.batch_size=4",
                f"task.model.projection_dim={width}", "task.optim.lr=1.0e-04", "trainer.max_steps=3",
                "trainer.log_every_n_steps=1", f"checkpoint_callback.dirpath={ckdir}"] + common)
    assert "train_loss" in out
    ckpt = torch.load(ckdir / "last.ckpt", map_location="cpu", weights_only=False)
    assert ckpt["global_step"] == 2 or ckpt["global_step"] == 3
    assert all(k.startswith("query_encoder.") for k in ckpt["state_dict"])
    _run(["dpr_scale_b200.generate_query_embeddings", "datamodule=generate_query_emb", f"datamodule.test_path={questions}",
          "+datamodule.trec_format=true", f"+task.ctx_embeddings_dir={student}",
          f"+task.checkpoint_path={ckdir / 'last.ckpt'}", f"task.model.projection_dim={width}"] + common)
    with open(student / "query_reps.pkl", "rb") as f:
        sreps = pickle.load(f)
    assert sreps.shape == (7, width) and torch.isfinite(sreps).all()
    run = tmp_path / "run.trec"
    _run(["dpr_scale_b200.run_retrieval", f"--ctx_embeddings_dir={ens}", f"--query_emb_path={student / 'query_reps.pkl'}",
          f"--questions_tsv_path={questions}", f"--passages_tsv_path={passages}", f"--output_runfile_path={run}",
          "--trec_format", "--topk=5"])
    lines = open(run).read().splitlines()
    assert len(lines) == 7 * 5
    assert {ln.split()[0] for ln in lines} == {f"q{i}" for i in range(7)}


# ------------------------------------------------------------------ two ranks
_CHILD = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from dpr_scale_b200.utils.dist_init import init_process_group
init_process_group()
r = dist.get_rank()
from dpr_scale_b200.task.dpr_distill_task import DPRDistillTask
from dpr_scale_b200.trainer import Trainer
from oracle import encoder as oenc, distill as odist
cfg = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
           max_position_embeddings=40)
torch.manual_seed(0)
task = DPRDistillTask(transform={}, model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                      "config": cfg, "dropout": 0.0}, datamodule=None,
                      optim={"_target_": "dpr_scale_b200.optim.FusedAdamW", "lr": 0.0}, )
tr = Trainer(max_steps=1, gradient_clip_val=0.0)
tr.attach(task, None, "fit")
sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in task.query_encoder.state_dict().items()}
out = {}
for rank in range(2):
    gen = torch.Generator().manual_seed(100 + rank)
    ids = torch.randint(5, 64, (6, 12), generator=gen)
    toks = {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": torch.ones_like(ids)}
    t = torch.randn(6, 128, generator=gen)
    if rank == r:
        batch = {"query_ids": toks, "target_vectors": t}
    s = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    q = oenc.encode(s, {"layers": 2, "heads": 2, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}, toks)
    _, dq = odist.sqerr(q, t, torch.float32)
    q.backward(dq)
    for k, v in s.items():
        if v.grad is not None:
            out[k] = out.get(k, 0) + v.grad / 2
tr.training_step(batch, 0)
torch.cuda.synchronize()
params = dict(task.query_encoder.named_parameters())
worst = 0.0
for k, ref in out.items():
    got = params[k].grad.detach().float().cpu() * tr.optimizer.grad_scale
    a, b = got.double().flatten(), ref.double().flatten()
    worst = max(worst, float((a - b).norm() / (b.norm() + 1e-30)))
if r == 0:
    print("WORST", worst)
dist.destroy_process_group()
"""


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_gradients_equal_mean_of_rank_oracles(tmp_path):
    script = tmp_path / "child.py"
    script.write_text(_CHILD)
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node=2",
                          str(script), ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    worst = float(res.stdout.split("WORST")[1].split()[0])
    assert worst <= 5e-2, worst
