#!/usr/bin/env python3
"""Generate golden vectors by running the UNMODIFIED reference (/root/reference) in the authoring container.

  python tests/golden/make_golden.py          # writes tests/golden/*.npz

The reference cannot travel to the GPU box, so the vectors are committed.  What runs here:
  * dpr_scale.models.hf_model.HFEncoder               (imported as is)
  * dpr_scale.task.dpr_task.DenseRetrieverTask        (imported as is, through stub `hydra` /
    `pytorch_lightning` modules because neither library is installed).
    The stub LightningModule.all_gather reproduces PL 1.6.4 semantics: per tensor dist.all_gather ->
    torch.stack(dim=0) under no_grad; identity when not distributed.
Cases:
  golden_1rank.npz  BERT (vocab 64, H128, L2, A2, I256), 4 queries, 1 pos + 1 neg, padded sequences,
                    one dummy (masked) negative, temperature 8 (keeps the tiny random model's logits O(10),
                    away from the saturated-softmax regime where a 0.3 % bf16 logit error swings probabilities by e^1) — embeddings, logits, loss, all grads.
  golden_2rank.npz  same model, world_size 2 (gloo): per-rank loss and per-rank grads (global in-batch negatives).
  golden_roberta.npz RoBERTa-style (pad_id 1, position ids from cumsum) encoder forward only.
  golden_world4.npz / golden_world8.npz  (`python make_golden.py world 4 8`) same model and per-rank batches at world
                    size 4 / 8 (gloo): per-rank batch + loss and the SUM over ranks of every parameter gradient - what
                    the trainer's all-reduce must produce.  bench.py's multi-GPU self-check compares against these
                    (and against golden_2rank.npz at N = 2) before timing, so NCCL parity is on record in every
                    scaling run even though the 1-GPU test box skips the NCCL pytest.
"""
import importlib
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def install_stubs():
    hydra = types.ModuleType("hydra")
    hu = types.ModuleType("hydra.utils")

    def instantiate(conf, *args, **kw):
        conf = dict(conf)
        mod, _, name = conf.pop("_target_").rpartition(".")
        return getattr(importlib.import_module(mod), name)(*args, **conf, **kw)

    hu.instantiate = instantiate
    hydra.utils = hu
    sys.modules["hydra"] = hydra
    sys.modules["hydra.utils"] = hu

    pl = types.ModuleType("pytorch_lightning")
    st = types.ModuleType("pytorch_lightning.strategies")

    class DDPStrategy:
        pass

    class DDPShardedStrategy:
        pass

    st.DDPStrategy, st.DDPShardedStrategy = DDPStrategy, DDPShardedStrategy

    class LightningModule(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.trainer = None
            self.logged = {}

        def save_hyperparameters(self):
            pass

        def log(self, k, v, **kw):
            self.logged[k] = v

        def log_dict(self, d, **kw):
            self.logged.update(d)

        @property
        def global_rank(self):
            return dist.get_rank() if dist.is_initialized() else 0

        def all_gather(self, data):
            def one(t):
                if not dist.is_initialized():
                    return t
                with torch.no_grad():
                    src = t.to(torch.uint8) if t.dtype == torch.bool else t
                    outs = [torch.zeros_like(src) for _ in range(dist.get_world_size())]
                    dist.all_gather(outs, src.contiguous())
                    res = torch.stack(outs, dim=0)
                    return res.to(torch.bool) if t.dtype == torch.bool else res
            return tuple(one(t) for t in data) if isinstance(data, (tuple, list)) else one(data)

    pl.LightningModule = LightningModule
    pl.strategies = st
    sys.modules["pytorch_lightning"] = pl
    sys.modules["pytorch_lightning.strategies"] = st
    return DDPStrategy


def make_model_dir(kind, seed, perturb_seed=None):
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    torch.manual_seed(seed)
    if kind == "bert":
        cfg = BertConfig(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256, max_position_embeddings=40)
        model = BertModel(cfg)
    else:
        cfg = RobertaConfig(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                            intermediate_size=256, max_position_embeddings=42, type_vocab_size=1,
                            layer_norm_eps=1e-5, pad_token_id=1)
        model = RobertaModel(cfg)
    # exercise bias / LayerNorm-affine paths: HF init leaves them at 0 / 1
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith("bias"):
                p.copy_(0.02 * torch.randn(p.shape, generator=g))
            elif "LayerNorm.weight" in n:
                p.copy_(1.0 + 0.02 * torch.randn(p.shape, generator=g))
        if perturb_seed is not None:
            g2 = torch.Generator().manual_seed(perturb_seed)
            for p in model.parameters():
                p.add_(0.01 * torch.randn(p.shape, generator=g2))
    d = tempfile.mkdtemp()
    model.save_pretrained(d)
    return d


def make_tokens(gen, n, S, vocab, pad_id, min_len):
    lens = torch.randint(min_len, S + 1, (n,), generator=gen)
    lens[0] = S  # at least one full-length row (the transform pads to the longest)
    ids = torch.randint(5, vocab, (n, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    ids = ids * am + pad_id * (1 - am)
    ids[:, 0] = 3
    return {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": am}


def make_batch(rank, B=4, n_neg=1, Sq=12, Sc=16):
    gen = torch.Generator().manual_seed(1234 + rank)
    C = B * (1 + n_neg)
    ctx_mask = torch.zeros(C, dtype=torch.bool)
    ctx_mask[3] = True  # a dummy negative (never a positive slot)
    return {
        "query_ids": make_tokens(gen, B, Sq, 64, 0, 4),
        "contexts_ids": make_tokens(gen, C, Sc, 64, 0, 5),
        "pos_ctx_indices": torch.arange(B) * (1 + n_neg),
        "ctx_mask": ctx_mask,
    }


def build_task(qdir, cdir, DDPStrategy, distributed, temperature):
    sys.path.insert(0, REF)
    from dpr_scale.task.dpr_task import DenseRetrieverTask
    model_conf = {"_target_": "dpr_scale.models.hf_model.HFEncoder", "model_path": qdir, "dropout": 0.0}
    task = DenseRetrieverTask(transform={}, model=model_conf, datamodule=None, optim={}, shared_model=False,
                              softmax_temperature=temperature)
    task.trainer = types.SimpleNamespace(strategy=DDPStrategy() if distributed else None)
    task.setup("fit")
    # context encoder gets its own weights (shared_model: false in every shipped YAML)
    from dpr_scale.models.hf_model import HFEncoder
    task.context_encoder = HFEncoder(model_path=cdir, dropout=0.0)
    task.eval()  # dropout is 0 anyway
    return task


def flat(prefix, d, out):
    for k, v in d.items():
        if isinstance(v, dict):
            flat(prefix + k + "/", v, out)
        else:
            out[prefix + k] = v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)


def run_rank(rank, world, qdir, cdir, port, ret):
    DDPStrategy = install_stubs()
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)
    T = 8.0
    task = build_task(qdir, cdir, DDPStrategy, world > 1, T)
    batch = make_batch(rank)
    loss = task.training_step(batch, 0)
    loss.backward()
    out = {}
    flat("batch/", {k: (dict(v) if isinstance(v, dict) else v) for k, v in batch.items()}, out)
    out["loss"] = loss.detach().numpy()
    for name, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
        for k, p in enc.named_parameters():
            if p.grad is not None:
                out[f"grad_{name}/{k}"] = p.grad.numpy()
    if world == 1:
        with torch.no_grad():
            q, c = task(batch["query_ids"], batch["contexts_ids"])
            m = batch["ctx_mask"].repeat(q.shape[0], 1)
            logits = task.sim_score(q, c, m) / T
        out["q_emb"], out["c_emb"], out["logits"] = q.numpy(), c.numpy(), logits.numpy()
        for name, enc in (("q", task.query_encoder), ("c", task.context_encoder)):
            for k, v in enc.state_dict().items():
                out[f"sd_{name}/{k}"] = v.numpy()
        out["temperature"] = np.float32(T)
        # The reference's OWN mixed-precision deviation on this batch (Lightning `precision: 16` analogue; bf16
        # autocast because fp16 matmul is not available on CPU): same weights, same batch, gradients compared
        # with the fp32 run above.  Stored so the CUDA-path tolerances can be stated relative to it.
        fp32_grads = {f"{n}/{k}": p.grad.clone() for n, e in (("q", task.query_encoder), ("c", task.context_encoder))
                      for k, p in e.named_parameters() if p.grad is not None}
        task.zero_grad()
        with torch.autocast("cpu", dtype=torch.bfloat16):
            amp_loss = task.training_step(batch, 0)
        amp_loss.backward()
        out["amp_loss"] = amp_loss.detach().float().numpy()
        num = den = 0.0
        for n, e in (("q", task.query_encoder), ("c", task.context_encoder)):
            for k, p in e.named_parameters():
                if p.grad is None:
                    continue
                a, b = p.grad.double().flatten(), fp32_grads[f"{n}/{k}"].double().flatten()
                out[f"amp_cos_{n}/{k}"] = np.float64((a @ b) / (a.norm() * b.norm() + 1e-30))
                out[f"amp_rel_{n}/{k}"] = np.float64((a - b).norm() / (b.norm() + 1e-30))
                num += float(((a - b) ** 2).sum())
                den += float((b ** 2).sum())
        out["amp_global_rel"] = np.float64((num / den) ** 0.5)
    ret[rank] = out
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def make_world(worlds):
    import torch.multiprocessing as mp
    qdir = make_model_dir("bert", 0)
    cdir = make_model_dir("bert", 0, perturb_seed=1)
    for W in worlds:
        shared = mp.Manager().dict()
        mp.spawn(run_rank, args=(W, qdir, cdir, 29540 + W, shared), nprocs=W, join=True)
        out = {}
        for r in range(W):
            for k, v in shared[r].items():
                if k.startswith("batch/") or k == "loss":
                    out[f"rank{r}/{k}"] = v
                elif k.startswith("grad_"):
                    key = "gradsum_" + k[len("grad_"):]
                    out[key] = out[key] + v.astype(np.float64) if key in out else v.astype(np.float64)
        out = {k: (v.astype(np.float32) if k.startswith("gradsum_") else v) for k, v in out.items()}
        np.savez_compressed(os.path.join(HERE, f"golden_world{W}.npz"), **out)
        print(f"world {W} losses", [float(shared[r]["loss"]) for r in range(W)])
    for d in (qdir, cdir):
        shutil.rmtree(d, ignore_errors=True)


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "world":
        return make_world([int(x) for x in sys.argv[2:]])
    qdir = make_model_dir("bert", 0)
    cdir = make_model_dir("bert", 0, perturb_seed=1)
    ret = {}
    run_rank(0, 1, qdir, cdir, 0, ret)
    np.savez_compressed(os.path.join(HERE, "golden_1rank.npz"), **ret[0])
    print("1-rank loss", ret[0]["loss"])

    import torch.multiprocessing as mp
    mgr = mp.Manager()
    shared = mgr.dict()
    mp.spawn(run_rank, args=(2, qdir, cdir, 29533, shared), nprocs=2, join=True)
    out = {}
    for r in (0, 1):
        for k, v in shared[r].items():
            out[f"rank{r}/{k}"] = v
    np.savez_compressed(os.path.join(HERE, "golden_2rank.npz"), **out)
    print("2-rank losses", shared[0]["loss"], shared[1]["loss"])

    # RoBERTa-style forward (position ids from the padding mask)
    install_stubs()
    sys.path.insert(0, REF)
    from dpr_scale.models.hf_model import HFEncoder
    rdir = make_model_dir("roberta", 7)
    enc = HFEncoder(model_path=rdir, dropout=0.0).eval()
    gen = torch.Generator().manual_seed(99)
    tok = make_tokens(gen, 5, 14, 64, 1, 4)
    tok.pop("token_type_ids")
    with torch.no_grad():
        rep = enc(tok)
    o = {"rep": rep.numpy()}
    flat("tokens/", tok, o)
    for k, v in enc.state_dict().items():
        o["sd/" + k] = v.numpy()
    np.savez_compressed(os.path.join(HERE, "golden_roberta.npz"), **o)
    print("roberta rep norm", float(rep.norm()))
    for d in (qdir, cdir, rdir):
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
