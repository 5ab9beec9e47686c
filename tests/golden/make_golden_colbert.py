#!/usr/bin/env python3
"""Golden vectors for ColBERT (multi-vector) reranking, produced by the UNMODIFIED reference (/root/reference).

  python tests/golden/make_golden_colbert.py        # writes tests/golden/colbert_small.npz, colbert_bert_base.npz

The reference is imported as make_golden_rerank.install_reference sets it up (hydra / pytorch_lightning stubs, the
citadel TRECDataset binding), plus ``pytorch_lightning.utilities.cloud_io.load`` = ``torch.load``, which
RerankMultiVecRetrieverTask.setup reads its checkpoint with.  No reference source is edited.

colbert_small.npz:
  * batches of ``DenseRetrieverRerankDataModule`` (use_title, batch 5, max_seq_len 24, the fixture BERT vocabulary)
    over tests/golden/data/rerank_run.trec; the rows of ``ContiguousDistributedSamplerForTest`` at 2 ranks;
  * for tiny BERT and RoBERTa ColBERT encoders with a 128-wide projection and without one (tests/colbert_cases.py):
    config, the reference ``ColBERTEncoder``'s state_dict keys, shapes and fp64 checksum (not its weights), and
    ``expert_repr`` on padded random tokens;
  * the three pickles ``RerankMultiVecRetrieverTask.test_epoch_end`` writes for the fixture run, for query_pool "sum"
    and "max", from a checkpoint file holding two seeded encoders (shared_model: false).
colbert_bert_base.npz: a seeded BERT-base-dims ColBERT (P = 128; weight checksums, not weights) on 16 pairs, queries of
  at most 32 tokens and passages of at most 256, each side padded to its longest: fp32 scores and the reference's own
  bf16-autocast scores, both pools.
"""
import json
import os
import pickle
import shutil
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_rerank import install_reference  # noqa: E402
from tests import colbert_cases, rerank_cases  # noqa: E402


def install():
    install_reference()
    ut = types.ModuleType("pytorch_lightning.utilities")
    cio = types.ModuleType("pytorch_lightning.utilities.cloud_io")
    cio.load = lambda path, map_location=None: torch.load(path, map_location=map_location, weights_only=False)
    ut.cloud_io = cio
    sys.modules["pytorch_lightning"].utilities = ut
    sys.modules["pytorch_lightning.utilities"] = ut
    sys.modules["pytorch_lightning.utilities.cloud_io"] = cio


def main():
    install()
    from dpr_scale.datamodule.citadel import DenseRetrieverRerankDataModule
    from dpr_scale.models.citadel_models.colbert_model import ColBERTEncoder
    from dpr_scale.task.citadel_eval_task import RerankMultiVecRetrieverTask
    from dpr_scale.transforms.hf_transform import HFTransform
    from dpr_scale.utils.utils import ContiguousDistributedSamplerForTest
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29562")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()

    # -- datamodule batches
    tok_dir = rerank_cases.tokenizer_dir(os.path.join(tmp, "tok"))
    dm = DenseRetrieverRerankDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                        **rerank_cases.datamodule_kwargs())
    batches = list(dm.test_dataloader())
    out["n_batches"] = np.int64(len(batches))
    for i, b in enumerate(batches):
        out[f"batch{i}/qid"] = np.array(b["qid"])
        out[f"batch{i}/ctx_id"] = np.array(b["ctx_id"])
        for side in ("query_ids", "contexts_ids"):
            for k, v in b[side].items():
                out[f"batch{i}/{side}/{k}"] = v.numpy()
    for r in range(2):
        out[f"shard2/rank{r}"] = np.array(list(ContiguousDistributedSamplerForTest(
            dm.datasets["test"], num_replicas=2, rank=r, shuffle=False)), dtype=np.int64)
    print("rows", len(dm.datasets["test"]), "batches", len(batches))

    # -- tiny encoders: expert_repr on random tokens
    for name, (kind, proj, _) in colbert_cases.TINY.items():
        cfg = colbert_cases.encoder_config(kind)
        mdir = colbert_cases.model_dir(os.path.join(tmp, name), name)
        enc = ColBERTEncoder(model_path=mdir, dropout=0.0, projection_dim=proj).eval()
        want = colbert_cases.tiny_state_dict(name)
        enc.load_state_dict(want, strict=True)
        sd = enc.state_dict()
        out[f"{name}/config"] = np.array(json.dumps(cfg))
        out[f"{name}/sd_keys"] = np.array(list(sd))
        out[f"{name}/sd_shapes"] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out[f"{name}/sd_checksum"] = colbert_cases.sd_checksum(sd).numpy()
        assert torch.equal(colbert_cases.sd_checksum(want), colbert_cases.sd_checksum(sd))
        toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(17), 6, 20, cfg["vocab_size"], cfg["pad_token_id"])
        with torch.no_grad():
            rep = enc(toks)["expert_repr"]
        for k, v in toks.items():
            out[f"{name}/tokens/{k}"] = v.numpy()
        out[f"{name}/expert_repr"] = rep.numpy()
        print(name, "expert_repr", tuple(rep.shape))

    # -- the rerank task's pickles
    for name in colbert_cases.TASK_KINDS:
        kind, proj, _ = colbert_cases.TINY[name]
        mdir = colbert_cases.model_dir(os.path.join(tmp, name + "_task"), name)
        ckpt = os.path.join(tmp, name + ".ckpt")
        torch.save({"state_dict": colbert_cases.task_state_dict(name)}, ckpt)
        for pool in colbert_cases.POOLS:
            odir = os.path.join(tmp, f"{name}_{pool}_out")
            task = RerankMultiVecRetrieverTask(
                checkpoint_path=ckpt, output_dir=odir, query_pool=pool, transform={}, datamodule=None, optim={},
                shared_model=False, in_batch_eval=False,
                model={"_target_": "dpr_scale.models.citadel_models.colbert_model.ColBERTEncoder", "model_path": mdir,
                       "projection_dim": proj, "dropout": 0.1})
            task.setup("test")
            task.eval()
            with torch.no_grad():
                outs = [task.test_step(b, i) for i, b in enumerate(dm.test_dataloader())]
            task.test_epoch_end(outs)
            for what in ("scores", "qids", "ctx_ids"):
                with open(os.path.join(odir, f"{what}_0000.pkl"), "rb") as f:
                    obj = pickle.load(f)
                out[f"{name}/{pool}/pkl/{what}"] = obj.numpy() if torch.is_tensor(obj) else np.array(obj)
            print(name, pool, "scores", out[f"{name}/{pool}/pkl/scores"][:4])
    np.savez_compressed(os.path.join(HERE, "colbert_small.npz"), **out)

    # -- BERT-base dims
    sd, cfg = colbert_cases.bert_base_state_dict()
    mdir = os.path.join(tmp, "bert_base")
    from transformers import BertConfig, BertModel
    BertModel(BertConfig(**cfg)).save_pretrained(mdir)
    enc = ColBERTEncoder(model_path=mdir, dropout=0.0, projection_dim=colbert_cases.BASE_P).eval()
    enc.load_state_dict(sd, strict=True)
    big = {"checksum": colbert_cases.sd_checksum(sd).numpy()}
    q, d = colbert_cases.bert_base_tokens()
    for side, toks in (("query", q), ("passage", d)):
        for k, v in toks.items():
            big[f"{side}/{k}"] = v.numpy()
    with torch.no_grad():
        qr, dr = enc(q), enc(d)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            qa, da = enc(q), enc(d)
    for pool in colbert_cases.POOLS:
        fake = types.SimpleNamespace(query_pool=pool)
        s = RerankMultiVecRetrieverTask.expert_sim_score(fake, qr, dr).float()
        with torch.autocast("cpu", dtype=torch.bfloat16):
            a = RerankMultiVecRetrieverTask.expert_sim_score(fake, qa, da).float()
        big[f"{pool}/scores"], big[f"{pool}/amp_scores"] = s.numpy(), a.numpy()
        big[f"{pool}/amp_max_abs"] = np.float64((a - s).abs().max())
        print("bert-base", pool, "scores", s[:4].tolist(), "amp max|dscore|", float(big[f"{pool}/amp_max_abs"]),
              "max|score|", float(s.abs().max()))
    np.savez_compressed(os.path.join(HERE, "colbert_bert_base.npz"), **big)
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
