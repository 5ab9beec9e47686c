#!/usr/bin/env python3
"""Golden vectors at BASELINE.json's REAL model dimensions, produced by the UNMODIFIED reference (/root/reference).

  python tests/golden/make_golden_realdims.py          # writes tests/golden/realdims_<case>.npz  (~1 min, 6 GB RAM)

Same machinery as make_golden.py (stub `hydra` / `pytorch_lightning`, the reference's own HFEncoder +
DenseRetrieverTask.training_step).  The weights come from the seeded recipe of tests/realdims.py and are
NOT stored - only their fp64 checksums, so the GPU test can prove it rebuilt the same weights.  Stored per case:
query / context embeddings, logits, loss, the reference's own bf16-autocast loss and gradient deviation (the yardstick of
the GPU parity gates), and a sample of the fp32 parameter gradients of (i) the contrastive step and (ii) a linear probe
L = sum(rep * P) on the context encoder (well conditioned: no cancellation between rows).
"""
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import REF, flat, install_stubs  # noqa: E402
from tests import realdims  # noqa: E402


def probe_for(n, d):
    return torch.randn(n, d, generator=torch.Generator().manual_seed(3))


def run_case(name):
    kind, cfg, B, n, S, T = realdims.CASES[name]
    DDPStrategy = install_stubs()
    sys.path.insert(0, REF)
    from dpr_scale.models.hf_model import HFEncoder
    from dpr_scale.task.dpr_task import DenseRetrieverTask
    qm, cm = realdims.hf_models(kind, cfg)
    out = {"sum_q": realdims.checksums(qm).numpy(), "sum_c": realdims.checksums(cm).numpy()}
    qdir, cdir = tempfile.mkdtemp(), tempfile.mkdtemp()
    qm.save_pretrained(qdir)
    cm.save_pretrained(cdir)
    del qm, cm
    task = DenseRetrieverTask(transform={}, model={"_target_": "dpr_scale.models.hf_model.HFEncoder",
                                                  "model_path": qdir, "dropout": 0.0},
                              datamodule=None, optim={}, shared_model=False, softmax_temperature=T)
    task.trainer = types.SimpleNamespace(strategy=None)
    task.setup("fit")
    task.context_encoder = HFEncoder(model_path=cdir, dropout=0.0)
    task.eval()
    batch = realdims.batch(name)
    loss = task.training_step(batch, 0)
    loss.backward()
    flat("batch/", {k: (dict(v) if isinstance(v, dict) else v) for k, v in batch.items()}, out)
    out["loss"] = loss.detach().numpy()
    names = realdims.sampled_grad_names(cfg)
    fp32 = {}
    for side, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        params = dict(enc.named_parameters())
        for k in names:
            g = params["transformer." + k].grad
            out[f"grad_{side}/{k}"] = realdims.sample(k, g).numpy().copy()
        for k, p in params.items():
            if p.grad is not None:
                fp32[f"{side}/{k}"] = p.grad.clone()
    with torch.no_grad():
        q, c = task(batch["query_ids"], batch["contexts_ids"])
        logits = task.sim_score(q, c, batch["ctx_mask"].repeat(q.shape[0], 1)) / T
    out["q_emb"], out["c_emb"], out["logits"] = q.numpy(), c.numpy(), logits.numpy()
    # the reference's own mixed-precision deviation on this batch (bf16 autocast; fp16 matmul does not exist on CPU)
    task.zero_grad()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        amp_loss = task.training_step(batch, 0)
    amp_loss.backward()
    out["amp_loss"] = amp_loss.detach().float().numpy()
    num = den = 0.0
    for side, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        for k, p in enc.named_parameters():
            if p.grad is None:
                continue
            a, b = p.grad.double().flatten(), fp32[f"{side}/{k}"].double().flatten()
            num += float(((a - b) ** 2).sum())
            den += float((b ** 2).sum())
            if k[len("transformer."):] in names:
                out[f"amp_rel_{side}/{k[len('transformer.'):]}"] = np.float64((a - b).norm() / (b.norm() + 1e-30))
    out["amp_global_rel"] = np.float64((num / den) ** 0.5)
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
        qa, ca = task(batch["query_ids"], batch["contexts_ids"])
    out["amp_emb_rel"] = np.float64(float((ca.float() - c).norm() / c.norm()))
    # linear probe on the context encoder
    task.zero_grad()
    rep = task.encode_contexts(batch["contexts_ids"])
    (rep * probe_for(*rep.shape)).sum().backward()
    params = dict(task.context_encoder.named_parameters())
    for k in names:
        out[f"probe_c/{k}"] = realdims.sample(k, params["transformer." + k].grad).numpy().copy()
    np.savez_compressed(os.path.join(HERE, f"realdims_{name}.npz"), **out)
    print(name, "loss", float(out["loss"]), "amp loss", float(out["amp_loss"]), "amp global grad rel",
          float(out["amp_global_rel"]), "amp emb rel", float(out["amp_emb_rel"]),
          "logits", float(logits[torch.isfinite(logits)].min()), float(logits.max()))
    for d in (qdir, cdir):
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    for case in (sys.argv[1:] or list(realdims.CASES)):
        run_case(case)
