#!/usr/bin/env python3
"""Golden vectors for query-encoder distillation and DrBoost ensembles: runs the UNMODIFIED reference
(dpr_scale/datamodule/dpr.py DPRDistillJsonlDataModule, transforms/dpr_distill_transform.py DPRDistillTransform,
task/dpr_distill_task.py DPRDistillTask, task/drboost_task.py DrBoostTask) on a seeded synthetic fixture.

  python tests/golden/make_golden_distill.py    # writes tests/golden/data/distill.jsonl and distill_small.npz

hydra / pytorch_lightning / ujson are not installed: the reference modules are imported through the stub modules of
make_golden.py and make_golden_data.py, with two additions the DrBoost task needs from Lightning:
LightningModule.load_from_checkpoint (rebuild from ``hyper_parameters``, build through ``on_load_checkpoint``, strict
``load_state_dict``) and ``device``.  The reference's DPRDistillTransform calls its text transform as
``tt({"text": texts})["token_ids"]``, which HFTransform does not accept, so the data cases wrap HFTransform in that
interface; the tokens are HFTransform's.  Cases:
  data/*      DPRDistillJsonlDataModule batches (train / valid / test) for two keyword sets, random.seed(5) before each;
              the reference's assertion messages for a row without positives and for positives that are not vectors.
  task/*      DPRDistillTask on the tiny BERT (vocab 64, H128, L2, A2, I256), dropout 0, 3 questions (6 rows):
              training_step loss and the query-encoder gradients tests/distill_cases.kept_gradient names; _eval_step on
              two batches and the epoch-end metrics; the task's state_dict keys.
  drboost/*   DrBoostTask over the weak DenseRetrieverTask checkpoints of tests/distill_cases.WEAK (one-layer tiny BERT;
              shared_model false, then true with projection_dim 16): encode_queries / encode_contexts.
The encoder weights are not stored: tests/distill_cases.encoder_state draws them from a seeded generator, here and in
the tests.
"""
import inspect
import json
import os
import random
import shutil
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "data")
sys.path.insert(0, HERE)
import make_golden  # noqa: E402
import make_golden_data  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import distill_cases  # noqa: E402

D_FIXTURE = 12


def write_fixture():
    rnd = random.Random(11)
    words = make_golden_data.WORDS

    def vec():
        return [rnd.gauss(0.0, 1.0) * 10 ** rnd.randint(-6, 1) for _ in range(D_FIXTURE)]

    rows = []
    for r in range(10):
        pos = [vec() for _ in range(1 + (r * 7) % 4)]
        q = vec()
        if r == 3:
            q = [rnd.randint(-3, 3) for _ in range(D_FIXTURE)]      # JSON integers
        rows.append({"question": " ".join(rnd.choice(words) for _ in range(rnd.randint(2, 9))),
                     "qry_target_vector": q, "ctx_target_vectors": pos})
    path = os.path.join(DATA, "distill.jsonl")
    with open(path, "w") as f:
        for row in rows:
            f.write(json.dumps(row) + "\n")
    return path, len(rows)


def install_stubs():
    make_golden.install_stubs()
    sys.modules["ujson"] = json
    sys.path.insert(0, make_golden.REF)
    pl = sys.modules["pytorch_lightning"]
    Base = pl.LightningModule

    class LightningModule(Base):
        def save_hyperparameters(self):
            frame = inspect.currentframe().f_back
            args = inspect.getargvalues(frame)
            self.hparams = {k: args.locals[k] for k in args.args if k != "self"}
            if args.keywords and args.keywords in args.locals:
                self.hparams.update(args.locals[args.keywords])

        @property
        def device(self):
            p = next(self.parameters(), None)
            return p.device if p is not None else torch.device("cpu")

        @classmethod
        def load_from_checkpoint(cls, checkpoint_path, map_location=None, **kw):
            ckpt = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
            model = cls(**dict(ckpt["hyper_parameters"], **kw))
            model.on_load_checkpoint(ckpt)
            model.load_state_dict(ckpt["state_dict"])
            return model.to(map_location) if map_location is not None else model

    class LightningDataModule:
        def __init__(self):
            self.trainer = None

    pl.LightningModule = LightningModule
    pl.LightningDataModule = LightningDataModule


def dump_batch(out, prefix, batch):
    for k in batch["query_ids"].keys():
        out[f"{prefix}/query_ids/{k}"] = batch["query_ids"][k].numpy()
    out[f"{prefix}/target_vectors"] = batch["target_vectors"].numpy()


def data_cases(out, path, tmp):
    from dpr_scale.datamodule.dpr import DPRDistillJsonlDataModule
    from dpr_scale.transforms.dpr_distill_transform import DPRDistillTransform
    from dpr_scale.transforms.hf_transform import HFTransform
    hf = HFTransform(model_path=make_golden_data.model_dir(os.path.join(tmp, "vocab_model")), max_seq_len=24)

    class TokenIdsTransform(torch.nn.Module):
        """The text-transform interface DPRDistillTransform._transform calls: {"text": [...]} -> {"token_ids": ...}."""

        def forward(self, batch):
            return {"token_ids": hf(batch["text"])}

    tf = TokenIdsTransform()
    cases = {"a": dict(batch_size=3, pos_ctx_sample=True),
             "b": dict(batch_size=4, val_batch_size=5, test_batch_size=6, pos_ctx_sample=False)}
    for name, kw in cases.items():
        dm = DPRDistillJsonlDataModule(transform=tf, train_path=path, val_path=path, test_path=path, **kw)
        random.seed(5)
        for stage, loader in (("train", dm.train_dataloader()), ("valid", dm.val_dataloader()),
                              ("test", dm.test_dataloader())):
            n = 0
            for i, batch in enumerate(loader):
                dump_batch(out, f"data/{name}/{stage}/{i}", batch)
                n += 1
            out[f"data/{name}/{stage}/num_batches"] = n
    bad = {"no_pos": {"question": "empty one", "qry_target_vector": [1.0, 2.0], "ctx_target_vectors": []},
           "not_vectors": {"question": "flat one", "qry_target_vector": [1.0, 2.0], "ctx_target_vectors": [1.0, 2.0]}}
    t = DPRDistillTransform(tf)
    for name, row in bad.items():
        try:
            t([json.dumps(row)], "train")
            raise SystemExit(f"the reference accepted the malformed row {name}")
        except AssertionError as e:
            out[f"data/malformed/{name}/message"] = np.array(str(e))
            out[f"data/malformed/{name}/row"] = np.array(json.dumps(row))


def load_weights(encoder, sd):
    """Seeded weights (tests/distill_cases.py) into a reference HFEncoder; only HF's buffers may stay unset."""
    missing, unexpected = encoder.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)


def task_cases(out, tmp):
    from dpr_scale.task.dpr_distill_task import DPRDistillTask
    mdir = make_golden.make_model_dir("bert", 21)
    conf = {"_target_": "dpr_scale.models.hf_model.HFEncoder", "model_path": mdir, "dropout": 0.0}
    task = DPRDistillTask(transform={}, model=conf, datamodule=None, optim={})
    task.setup("fit")
    load_weights(task.query_encoder, distill_cases.encoder_state(distill_cases.CFG, distill_cases.TASK_SEED))
    out["task/state_dict_keys"] = np.array(sorted(task.state_dict()))
    gen = torch.Generator().manual_seed(77)

    def batch(B):
        q = make_golden.make_tokens(gen, B, 12, 64, 0, 4)
        toks = {k: v.repeat_interleave(2, dim=0) for k, v in q.items()}      # every question twice
        return {"query_ids": toks, "target_vectors": 0.5 * torch.randn(2 * B, 128, generator=gen)}

    train = batch(3)
    for k, v in train["query_ids"].items():
        out[f"task/train/query_ids/{k}"] = v.numpy()
    out["task/train/target_vectors"] = train["target_vectors"].numpy()
    task.train()
    loss = task.training_step(train, 0)
    loss.backward()
    out["task/train/loss"] = loss.detach().numpy()
    out["task/train/train_loss_logged"] = np.asarray(float(task.logged["train_loss"]))
    for k, p in task.query_encoder.named_parameters():
        if p.grad is not None and distill_cases.kept_gradient(k, p.numel()):
            out["task/grad/" + k] = p.grad.numpy()
    task.eval()
    outs = []
    with torch.no_grad():
        for i, B in enumerate((3, 2)):
            b = batch(B)
            for k, v in b["query_ids"].items():
                out[f"task/eval/{i}/query_ids/{k}"] = v.numpy()
            out[f"task/eval/{i}/target_vectors"] = b["target_vectors"].numpy()
            res = task._eval_step(b, i)
            (rank, mrr, score), q, t, l = res
            out[f"task/eval/{i}/rank"] = np.asarray(rank)
            out[f"task/eval/{i}/mrr"] = np.asarray(mrr)
            out[f"task/eval/{i}/score"] = np.asarray(float(score))
            out[f"task/eval/{i}/query_repr"] = q.numpy()
            out[f"task/eval/{i}/loss"] = l.numpy()
            outs.append(res)
        task._eval_epoch_end(outs, "valid")
    for k, v in task.logged.items():
        if k.startswith("valid_"):
            out["task/metrics/" + k] = np.asarray(float(v))


def drboost_cases(out, tmp):
    from dpr_scale.task.dpr_task import DenseRetrieverTask
    from dpr_scale.task.drboost_task import DrBoostTask
    from transformers import BertConfig, BertModel
    paths = []
    for i, (shared, pd, seed_q, seed_c) in enumerate(distill_cases.WEAK):
        mdir = os.path.join(tmp, f"weak_model{i}")
        BertModel(BertConfig(**distill_cases.WEAK_CFG)).save_pretrained(mdir)
        conf = {"_target_": "dpr_scale.models.hf_model.HFEncoder", "model_path": mdir, "dropout": 0.0,
                "projection_dim": pd}
        t = DenseRetrieverTask(transform={}, model=conf, datamodule=None, optim={}, shared_model=shared)
        t.setup("fit")
        load_weights(t.query_encoder, distill_cases.encoder_state(distill_cases.WEAK_CFG, seed_q, pd))
        if not shared:
            load_weights(t.context_encoder, distill_cases.encoder_state(distill_cases.WEAK_CFG, seed_c, pd))
        path = os.path.join(tmp, f"weak{i}.ckpt")
        torch.save({"state_dict": t.state_dict(), "hyper_parameters": dict(t.hparams)}, path)
        paths.append(path)
    task = DrBoostTask(checkpoint_paths=paths, transform={}, model={}, datamodule=None, optim={})
    task.setup("test")
    task.eval()
    gen = torch.Generator().manual_seed(88)
    q = make_golden.make_tokens(gen, 5, 12, 64, 0, 4)
    c = make_golden.make_tokens(gen, 7, 16, 64, 0, 5)
    for k in q:
        out[f"drboost/query_ids/{k}"] = q[k].numpy()
        out[f"drboost/contexts_ids/{k}"] = c[k].numpy()
    with torch.no_grad():
        qr, cr = task(q, c)
    out["drboost/query_repr"] = qr.numpy()
    out["drboost/contexts_repr"] = cr.numpy()


def main():
    path, n_rows = write_fixture()
    install_stubs()
    torch.manual_seed(0)
    out = {"n_rows": np.asarray(n_rows)}
    tmp = tempfile.mkdtemp()
    try:
        data_cases(out, path, tmp)
        task_cases(out, tmp)
        drboost_cases(out, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(HERE, "distill_small.npz"), **out)
    print(f"wrote {len(out)} arrays to distill_small.npz")


if __name__ == "__main__":
    main()
