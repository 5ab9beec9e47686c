"""The fused LAMB and MADGRAD steps on the H100:
  * kernels against the float64 oracles (oracle/optim.py) on a synthetic arena of many uneven segments, with clipping,
    grad_scale and weight decay;
  * the optimizers on the golden_1rank task against a per-tensor fp32 restatement (projection head included);
  * bitwise repeatability, and a short training run from the config."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import optim as oopt
from oracle import task as otask
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "golden", "data")
# one segment per "parameter tensor": LayerNorm-sized, tiny, chunk-sized, one past a chunk, multi-chunk, large
SEGMENTS = [768, 4, 8192, 8196, 36, 3 * 8192 + 4, 768 * 3, 100004, 20, 2304 * 8, 12, 65536]


def _arena(seed, n):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g), g


def _segments(t):
    out, lo = [], 0
    for n in SEGMENTS:
        out.append(t[lo:lo + n])
        lo += n
    return out


@pytest.mark.parametrize("kw", [dict(), dict(debias=True, clamp_value=2.0), dict(adam=True)])
def test_lamb_kernel_matches_oracle_on_uneven_segments(kw):
    from dpr_scale_b200 import ops
    n = sum(SEGMENTS)
    p, g = _arena(11, n)
    p[sum(SEGMENTS[:4]):sum(SEGMENTS[:5])] = 0.0                 # a zero-norm tensor: trust 1
    pd, md, vd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    plan = ops.LambPlan(SEGMENTS, DEV)
    pr, mr, vr = p.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    lr, wd = 1e-2, 0.01
    for step in range(1, 4):
        gr = torch.randn(n, generator=g) * 3
        gd = gr.to(DEV)
        ss = torch.zeros(1, device=DEV)
        ops.sumsq(gd, ss)
        ops.lamb_step(pd, gd, md, vd, shadow, plan, lr, 0.9, 0.999, 1e-6, wd, kw.get("clamp_value", 10.0),
                      kw.get("adam", False), kw.get("debias", False), step, 0.5, ss, 2.0)
        coef, _ = otask.clip_coef([gr * 0.5], 2.0)
        assert coef < 1.0                                       # the clip is active
        trusts = [oopt.lamb_step(ps, 0.5 * coef * gs, ms, vs, step, lr, 0.9, 0.999, 1e-6, wd, **kw)
                  for ps, gs, ms, vs in zip(_segments(pr), _segments(gr.double()), _segments(mr), _segments(vr))]
        b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))    # the betas as the kernel receives them
        step_size = lr * (math.sqrt(1 - b2 ** step) / (1 - b1 ** step) if kw.get("debias") else 1.0)
        got = plan.trust_scale().double().cpu() / step_size
        assert torch.allclose(got, torch.tensor(trusts, dtype=torch.float64), rtol=1e-5, atol=0), (got, trusts)
        assert torch.equal(gd.cpu(), gr)                       # the gradient arena is read only
        if step == 1:
            assert trusts[4] == 1.0                              # ||p|| = 0
    assert torch.allclose(pd.cpu().double(), pr, rtol=1e-5, atol=1e-6), float((pd.cpu().double() - pr).abs().max())
    assert torch.allclose(md.cpu().double(), mr, rtol=1e-4, atol=1e-7)
    assert torch.allclose(vd.cpu().double(), vr, rtol=1e-4, atol=1e-9)
    assert torch.allclose(shadow.float(), pd, rtol=2 ** -8, atol=0)


@pytest.mark.parametrize("momentum", [0.9, 0.0])
def test_madgrad_kernel_matches_oracle_with_warmup_step(momentum):
    from dpr_scale_b200 import ops
    n = 100003                                                   # not a multiple of 4: the scalar tail runs too
    p, g = _arena(12, n)
    pd, nud, sd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    x0d = pd.clone() if momentum else None
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    pr = p.double()
    st = oopt.madgrad_state(pr, momentum)
    wd, eps = 0.01, 1e-6
    for k, lr in enumerate([0.0, 1e-2, 5e-3, 1e-2]):             # k = 0: the LambdaLR warmup holds lr at 0
        gr = torch.randn(n, generator=g) * 3
        gd = gr.to(DEV)
        ss = torch.zeros(1, device=DEV)
        ops.sumsq(gd, ss)
        ops.madgrad_step(pd, gd, nud, sd, x0d, shadow, lr, momentum, wd, eps, k, 0.5, ss, 2.0)
        coef, _ = otask.clip_coef([gr * 0.5], 2.0)
        assert coef < 1.0
        oopt.madgrad_step(pr, 0.5 * coef * gr.double(), st, k, lr, momentum, wd, eps)
        err = float((pd.cpu().double() - pr).abs().max())
        assert torch.allclose(pd.cpu().double(), pr, rtol=1e-5, atol=2e-6), (k, err)
        if k == 0:
            assert not torch.equal(pd.cpu(), p)                  # lr + eps: the warmup step still moves p
    assert torch.allclose(nud.cpu().double(), st["grad_sum_sq"], rtol=1e-5, atol=1e-12)
    assert torch.allclose(sd.cpu().double(), st["s"], rtol=1e-5, atol=1e-9)
    assert torch.allclose(shadow.float(), pd, rtol=2 ** -8, atol=0)


def test_lamb_and_madgrad_are_bitwise_repeatable():
    from dpr_scale_b200 import ops
    n = sum(SEGMENTS) * 8
    sizes = SEGMENTS * 8

    def lamb():
        p, g = _arena(21, n)
        pd, md, vd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        plan = ops.LambPlan(sizes, DEV)
        for step in range(1, 4):
            gd = (torch.randn(n, generator=g) * 3).to(DEV)
            ss = (gd.double() ** 2).sum().float().view(1)       # dprb_sumsq_f32 adds with atomics: not repeatable
            ops.lamb_step(pd, gd, md, vd, None, plan, 1e-2, 0.9, 0.999, 1e-6, 0.01, 10.0, False, False, step, 0.5,
                          ss, 2.0)
        return pd.cpu()

    def madgrad():
        p, g = _arena(22, n)
        pd, nud, sd = p.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        x0 = pd.clone()
        for k in range(3):
            gd = (torch.randn(n, generator=g) * 3).to(DEV)
            ss = (gd.double() ** 2).sum().float().view(1)
            ops.madgrad_step(pd, gd, nud, sd, x0, None, 1e-2, 0.9, 0.01, 1e-6, k, 0.5, ss, 2.0)
        return pd.cpu()

    for fn in (lamb, madgrad):
        assert torch.equal(fn(), fn()), fn.__name__


# ------------------------------------------------------------------ on the golden_1rank task
CFG = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
           max_position_embeddings=40)


def _task_with_projection():
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from tests.test_task_gpu import _batch
    g = load_golden("golden_1rank.npz")
    task = DenseRetrieverTask(transform={}, model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config",
                                                  "config": CFG, "dropout": 0.0, "projection_dim": 64},
                              datamodule=None, optim={}, shared_model=False,
                              softmax_temperature=float(g["temperature"]))
    task.trainer = None
    task.setup("fit")
    return task.cuda(), _batch(g)


def _lamb_restated(params, grads, states, step, lr, wd, eps=1e-6, b1=0.9, b2=0.999, clamp=10.0):
    for p, g, st in zip(params, grads, states):
        st[0].mul_(b1).add_(g, alpha=1 - b1)
        st[1].mul_(b2).addcmul_(g, g, value=1 - b2)
        u = st[0] / (st[1].sqrt() + eps) + wd * p
        w_norm, u_norm = float(p.norm().clamp(0, clamp)), float(u.norm())
        trust = 1.0 if (w_norm == 0 or u_norm == 0) else w_norm / u_norm
        p.sub_(lr * trust * u)


def _madgrad_restated(params, grads, states, k, lr, momentum, wd, eps=1e-6):
    lamb = (lr + eps) * math.sqrt(k + 1)
    for p, g, st in zip(params, grads, states):
        g = g + wd * p
        st["grad_sum_sq"].addcmul_(g, g, value=lamb)
        st["s"].add_(g, alpha=lamb)
        z = st["x0"] - st["s"] / (st["grad_sum_sq"].pow(1 / 3) + eps)
        p.mul_(momentum).add_(z, alpha=1 - momentum)


@pytest.mark.parametrize("which", ["lamb", "madgrad"])
def test_fused_optimizer_matches_per_tensor_restatement_on_task(which):
    """clip(2.0) + LAMB / MADGRAD over the flat arenas and the projection heads == the per-tensor fp32 restatement after
    torch's clip_grad_norm_, over three steps on the same gradients (the kernels leave the gradient arena unchanged)."""
    from dpr_scale_b200.optim import FusedLamb, FusedMADGRAD
    task, batch = _task_with_projection()
    if which == "lamb":
        opt = FusedLamb(task.parameters(), lr=1e-2, eps=1e-6, weight_decay=0.01, max_grad_norm=2.0)
    else:
        opt = FusedMADGRAD(task.parameters(), lr=1e-3, momentum=0.9, weight_decay=0.01, max_grad_norm=2.0)
    ref_params = [p.detach().clone() for p in task.parameters()]
    opt.attach_encoders([task.query_encoder, task.context_encoder])
    opt.zero_grad()
    task.training_step(batch, 0).backward()
    live = [p for p in task.parameters() if p.grad is not None]
    assert any(not any(p is q for _, q, _ in e.transformer.arena_params())
               for p in live for e in (task.query_encoder, task.context_encoder))   # projection heads take part
    ref = [torch.nn.Parameter(r) for r, p in zip(ref_params, task.parameters()) if p.grad is not None]
    for rp, p in zip(ref, live):
        rp.grad = p.grad.detach().clone()
    torch.nn.utils.clip_grad_norm_(ref, 2.0)
    grads = [rp.grad for rp in ref]
    if which == "lamb":
        states = [[torch.zeros_like(rp), torch.zeros_like(rp)] for rp in ref]
    else:
        states = [{"grad_sum_sq": torch.zeros_like(rp), "s": torch.zeros_like(rp), "x0": rp.detach().clone()}
                  for rp in ref]
    with torch.no_grad():
        for k in range(3):
            opt.step()
            if which == "lamb":
                _lamb_restated([rp.data for rp in ref], grads, states, k + 1, 1e-2, 0.01)
            else:
                _madgrad_restated([rp.data for rp in ref], grads, states, k, 1e-3, 0.9, 0.01)
    torch.cuda.synchronize()
    for rp, p in zip(ref, live):
        err = float((p.detach() - rp.detach()).abs().max())
        assert torch.allclose(p.detach(), rp.detach(), atol=2e-6, rtol=1e-5), err
    for enc in (task.query_encoder, task.context_encoder):
        assert torch.allclose(enc.shadow.float(), enc.master, atol=0, rtol=2 ** -8)


# ------------------------------------------------------------------ a short run from the config
def _model_dir(path):
    from transformers import BertConfig, BertModel
    vocab = open(os.path.join(DATA, "vocab.txt")).read()
    torch.manual_seed(0)
    BertModel(BertConfig(vocab_size=len(vocab.split()), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256, max_position_embeddings=64)).save_pretrained(path)
    with open(os.path.join(path, "vocab.txt"), "w") as f:
        f.write(vocab)
    with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "BertTokenizer", "do_lower_case": True}, f)
    return str(path)


def test_main_with_lamb_trains_and_lowers_the_loss(tmp_path, monkeypatch):
    from dpr_scale_b200 import main as dmain
    from dpr_scale_b200.optim import FusedLamb
    from dpr_scale_b200.trainer import Trainer
    model = _model_dir(tmp_path / "model")
    jsonl = os.path.join(DATA, "synth.jsonl")
    losses, opts = [], []
    step = Trainer.training_step

    def recording_step(self, batch, batch_idx=0):
        loss = step(self, batch, batch_idx)
        losses.append(float(loss))
        opts.append(type(self.optimizer))
        return loss
    monkeypatch.setattr(Trainer, "training_step", recording_step)
    monkeypatch.chdir(tmp_path)
    epochs = 8
    np.random.seed(0)
    torch.manual_seed(0)
    dmain.main(["task/optim=lamb", "task.optim.lr=0.01", f"task.model.model_path={model}", "task.model.dropout=0.0",
                "task.transform.max_seq_len=32", f"datamodule.train_path={jsonl}", f"datamodule.val_path={jsonl}",
                f"datamodule.test_path={jsonl}", "datamodule.batch_size=4", "datamodule.num_negative=1",
                f"trainer.max_epochs={epochs}", f"checkpoint_callback.dirpath={tmp_path / 'ckpt'}"])
    assert opts and set(opts) == {FusedLamb}
    assert len(losses) >= 3 * epochs and np.isfinite(losses).all()
    assert np.mean(losses[-4:]) < np.mean(losses[:4]), losses
