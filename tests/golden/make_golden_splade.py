#!/usr/bin/env python3
"""Golden vectors for SPLADE and dense (DPR) reranking, produced by the UNMODIFIED reference.

  python tests/golden/make_golden_splade.py        # writes tests/golden/splade_small.npz, splade_bert_base.npz

The reference is imported as make_golden_colbert.install sets it up.  No reference source is edited.

splade_small.npz:
  * for tiny BERT and RoBERTa SPLADE encoders (tests/splade_cases.py): config, the reference encoder's state_dict keys,
    shapes and fp64 checksum (not its weights), and its output on padded random tokens (the last row has no valid token
    after token 0);
  * the three pickles RerankDenseRetrieverTask.test_epoch_end writes for the fixture run (tests/colbert_cases.py's
    datamodule settings), with HFEncoder (a 64-wide projection) and with SPLADEEncoder, each from a checkpoint file
    holding two seeded encoders.
splade_bert_base.npz: a seeded BERT-base-dims SPLADE encoder on 16 pairs (queries of at most 32 tokens, passages of at
  most 256): the reps' every 16th vocabulary column and the rerank scores in fp32, the same from the reference's own
  bf16-autocast run, and the largest deviations of that run (over every column of the reps, and over the scores).
"""
import json
import os
import pickle
import shutil
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_colbert import install  # noqa: E402
from tests import colbert_cases, rerank_cases, splade_cases  # noqa: E402


def main():
    install()
    from dpr_scale.datamodule.citadel import DenseRetrieverRerankDataModule
    from dpr_scale.models.citadel_models.splade_model import SPLADEEncoder
    from dpr_scale.task.dpr_rerank_task import RerankDenseRetrieverTask
    from dpr_scale.transforms.hf_transform import HFTransform
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29564")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()
    tok_dir = rerank_cases.tokenizer_dir(os.path.join(tmp, "tok"))
    dm = DenseRetrieverRerankDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                        **rerank_cases.datamodule_kwargs())

    # -- tiny encoders
    for name, (kind, _) in splade_cases.TINY.items():
        cfg = colbert_cases.encoder_config(kind)
        mdir = splade_cases.tiny_model_dir(os.path.join(tmp, name), name)
        enc = SPLADEEncoder(mdir, 0.0).eval()
        want = splade_cases.tiny_state_dict(name)
        enc.load_state_dict(want, strict=True)
        sd = enc.state_dict()
        out[f"{name}/config"] = np.array(json.dumps(cfg))
        out[f"{name}/sd_keys"] = np.array(list(sd))
        out[f"{name}/sd_shapes"] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out[f"{name}/sd_checksum"] = colbert_cases.sd_checksum(sd).numpy()
        assert torch.equal(colbert_cases.sd_checksum(want), colbert_cases.sd_checksum(sd))
        toks = splade_cases.tiny_tokens(cfg)
        for k, v in toks.items():
            out[f"{name}/tokens/{k}"] = v.numpy()
        with torch.no_grad():
            r = enc(toks)
        out[f"{name}/reps"] = r.numpy()
        print(name, tuple(r.shape), "row maxima", r.max(1).values.tolist())

    # -- the rerank task's pickles
    for model, (_, _, proj, seed) in splade_cases.TASK.items():
        mdir = splade_cases.model_dir(os.path.join(tmp, model + "_task"), model, seed)
        ckpt = os.path.join(tmp, model + ".ckpt")
        torch.save({"state_dict": splade_cases.task_state_dict(model)}, ckpt)
        odir = os.path.join(tmp, f"{model}_out")
        mconf = {"_target_": splade_cases.TARGETS[model], "model_path": mdir, "dropout": 0.1}
        if proj:
            mconf["projection_dim"] = proj
        task = RerankDenseRetrieverTask(checkpoint_path=ckpt, output_dir=odir, transform={}, datamodule=None, optim={},
                                        shared_model=False, in_batch_eval=False, model=mconf)
        task.setup("test")
        task.eval()
        with torch.no_grad():
            outs = [task.test_step(b, i) for i, b in enumerate(dm.test_dataloader())]
        task.test_epoch_end(outs)
        for what in ("scores", "qids", "ctx_ids"):
            with open(os.path.join(odir, f"{what}_0000.pkl"), "rb") as f:
                obj = pickle.load(f)
            out[f"{model}/pkl/{what}"] = obj.numpy() if torch.is_tensor(obj) else np.array(obj)
        print(model, "scores", out[f"{model}/pkl/scores"][:4])
    np.savez_compressed(os.path.join(HERE, "splade_small.npz"), **out)

    # -- BERT-base dims
    big = {}
    q, d = splade_cases.bert_base_tokens()
    for side, toks in (("query", q), ("passage", d)):
        for k, v in toks.items():
            big[f"{side}/{k}"] = v.numpy()
    from transformers import BertConfig, BertForMaskedLM
    sd, cfg = splade_cases.bert_base_state_dict()
    mdir = os.path.join(tmp, "bert_base_splade")
    BertForMaskedLM(BertConfig(**cfg)).save_pretrained(mdir)
    enc = SPLADEEncoder(mdir, 0.0).eval()
    enc.load_state_dict(sd, strict=True)
    big["checksum"] = colbert_cases.sd_checksum(sd).numpy()
    cs = splade_cases.BASE_COL_STRIDE
    with torch.no_grad():
        qr, dr = enc(q), enc(d)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            qa, da = enc(q).float(), enc(d).float()
    for side, r, a in (("query", qr, qa), ("passage", dr, da)):
        big[f"{side}/reps_cols"], big[f"{side}/amp_reps_cols"] = r[:, ::cs].numpy(), a[:, ::cs].numpy()
        big[f"{side}/amp_reps_max_abs"] = np.float64((a - r).abs().max())
    s, sa = (qr * dr).sum(1), (qa * da).sum(1)
    big["scores"], big["amp_scores"] = s.numpy(), sa.numpy()
    big["amp_max_abs"] = np.float64((sa - s).abs().max())
    print("bert-base scores", s[:4].tolist(), "amp max|dscore|", float(big["amp_max_abs"]), "max|score|",
          float(s.abs().max()), "amp max|drep|", float(big["query/amp_reps_max_abs"]),
          float(big["passage/amp_reps_max_abs"]))
    np.savez_compressed(os.path.join(HERE, "splade_bert_base.npz"), **big)
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
