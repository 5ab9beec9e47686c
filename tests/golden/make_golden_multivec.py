#!/usr/bin/env python3
"""Golden vectors for COIL and CITADEL reranking, produced by the UNMODIFIED reference.

  python tests/golden/make_golden_multivec.py        # writes tests/golden/multivec_small.npz, multivec_bert_base.npz

The reference is imported as make_golden_colbert.install sets it up.  No reference source is edited.

multivec_small.npz, for tiny BERT and RoBERTa COIL and CITADEL encoders (tests/multivec_cases.py):
  * config, the reference encoder's state_dict keys, shapes and fp64 checksum (not its weights);
  * on padded random tokens, with add_cls off and on and (CITADEL) topk 1 and 2: expert_repr, expert_ids,
    expert_weights and cls_repr;
  * the three pickles RerankMultiVecRetrieverTask.test_epoch_end writes for the fixture run (tests/colbert_cases.py's
    datamodule settings), query_pool "sum" and "max", add_cls on, query_topk 2 / context_topk 1, from a checkpoint file
    holding two seeded encoders.
multivec_bert_base.npz: a seeded BERT-base-dims COIL (projections 128 / 128) and CITADEL (token 32, CLS 128) on 16
  pairs (queries of at most 32 tokens, passages of at most 256) with add_cls on and one expert per token: fp32 scores
  and the reference's own bf16-autocast scores, both pools; for CITADEL also each token's float32 top-1 logit and the
  gap to its second-best logit (so tests know which tokens are near ties) and the largest top-1 logit deviation of the
  bf16-autocast run.
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

from make_golden_colbert import install  # noqa: E402
from tests import colbert_cases, multivec_cases, rerank_cases  # noqa: E402


def reference_encoder(name_or_model, mdir, proj, cls_proj):
    from dpr_scale.models.citadel_models.citadel_model import CITADELEncoder
    from dpr_scale.models.citadel_models.coil_model import COILEncoder
    cls = COILEncoder if name_or_model == "coil" else CITADELEncoder
    return cls(mdir, 0.0, **multivec_cases.ctor_kwargs(name_or_model, proj, cls_proj)).eval()


def main():
    install()
    from dpr_scale.datamodule.citadel import DenseRetrieverRerankDataModule
    from dpr_scale.task.citadel_eval_task import RerankMultiVecRetrieverTask
    from dpr_scale.transforms.hf_transform import HFTransform
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29563")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()
    tok_dir = rerank_cases.tokenizer_dir(os.path.join(tmp, "tok"))
    dm = DenseRetrieverRerankDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                        **rerank_cases.datamodule_kwargs())

    # -- tiny encoders
    for name, (model, kind, proj, cls_proj, _) in multivec_cases.TINY.items():
        cfg = colbert_cases.encoder_config(kind)
        mdir = multivec_cases.model_dir(os.path.join(tmp, name), name)
        enc = reference_encoder(model, mdir, proj, cls_proj)
        want = multivec_cases.tiny_state_dict(name)
        enc.load_state_dict(want, strict=True)
        sd = enc.state_dict()
        out[f"{name}/config"] = np.array(json.dumps(cfg))
        out[f"{name}/sd_keys"] = np.array(list(sd))
        out[f"{name}/sd_shapes"] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out[f"{name}/sd_checksum"] = colbert_cases.sd_checksum(sd).numpy()
        assert torch.equal(colbert_cases.sd_checksum(want), colbert_cases.sd_checksum(sd))
        toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(19), 6, 20, cfg["vocab_size"], cfg["pad_token_id"])
        for k, v in toks.items():
            out[f"{name}/tokens/{k}"] = v.numpy()
        for topk in ((1, 2) if model == "citadel" else (1,)):
            for add_cls in (False, True):
                with torch.no_grad():
                    r = enc(toks, topk=topk, add_cls=add_cls)
                for k in ("expert_repr", "expert_ids", "expert_weights", "cls_repr"):
                    if k in r:
                        out[f"{name}/k{topk}/cls{int(add_cls)}/{k}"] = r[k].numpy()
        print(name, {k: tuple(v.shape) for k, v in r.items()})

    # -- the rerank task's pickles
    qk, ck = multivec_cases.TASK_TOPK
    for name, (model, kind, proj, cls_proj, _) in multivec_cases.TINY.items():
        mdir = multivec_cases.model_dir(os.path.join(tmp, name + "_task"), name)
        ckpt = os.path.join(tmp, name + ".ckpt")
        torch.save({"state_dict": multivec_cases.task_state_dict(name)}, ckpt)
        for pool in multivec_cases.POOLS:
            odir = os.path.join(tmp, f"{name}_{pool}_out")
            task = RerankMultiVecRetrieverTask(
                checkpoint_path=ckpt, output_dir=odir, query_pool=pool, add_cls=True, query_topk=qk, context_topk=ck,
                transform={}, datamodule=None, optim={}, shared_model=False, in_batch_eval=False,
                model=dict({"_target_": "dpr_scale.models.citadel_models." + multivec_cases.TARGETS[model],
                            "model_path": mdir, "dropout": 0.1}, **multivec_cases.ctor_kwargs(model, proj, cls_proj)))
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
    np.savez_compressed(os.path.join(HERE, "multivec_small.npz"), **out)

    # -- BERT-base dims
    big = {}
    q, d = multivec_cases.bert_base_tokens()
    for side, toks in (("query", q), ("passage", d)):
        for k, v in toks.items():
            big[f"{side}/{k}"] = v.numpy()
    from transformers import BertConfig, BertForMaskedLM, BertModel
    for model in ("coil", "citadel"):
        sd, cfg = multivec_cases.bert_base_state_dict(model)
        mdir = os.path.join(tmp, f"bert_base_{model}")
        (BertModel if model == "coil" else BertForMaskedLM)(BertConfig(**cfg)).save_pretrained(mdir)
        enc = reference_encoder(model, mdir, *multivec_cases.BASE[model])
        enc.load_state_dict(sd, strict=True)
        big[f"{model}/checksum"] = colbert_cases.sd_checksum(sd).numpy()
        with torch.no_grad():
            qr, dr = enc(q, topk=1, add_cls=True), enc(d, topk=1, add_cls=True)
            with torch.autocast("cpu", dtype=torch.bfloat16):
                qa, da = enc(q, topk=1, add_cls=True), enc(d, topk=1, add_cls=True)
            if model == "citadel":
                dev = 0.0
                for side, toks in (("query", q), ("passage", d)):
                    logits = enc.transformer(**toks, return_dict=True).logits[:, 1:].float()
                    top2 = logits.topk(2, dim=-1).values
                    with torch.autocast("cpu", dtype=torch.bfloat16):
                        la = enc.transformer(**toks, return_dict=True).logits[:, 1:].float()
                    ids = logits.argmax(-1, keepdim=True)
                    am = toks["attention_mask"][:, 1:] != 0
                    dev = max(dev, float((la.gather(-1, ids) - top2[..., :1]).abs().squeeze(-1)[am].max()))
                    big[f"citadel/{side}/top1"] = top2[..., 0].numpy()
                    big[f"citadel/{side}/gap"] = (top2[..., 0] - top2[..., 1]).numpy()
                    del logits, la
                big["citadel/amp_logit_max_abs"] = np.float64(dev)
        for pool in multivec_cases.POOLS:
            fake = types.SimpleNamespace(query_pool=pool)
            s = (RerankMultiVecRetrieverTask.expert_sim_score(fake, qr, dr) +
                 (qr["cls_repr"] * dr["cls_repr"]).sum(1)).float()
            with torch.autocast("cpu", dtype=torch.bfloat16):
                a = (RerankMultiVecRetrieverTask.expert_sim_score(fake, qa, da) +
                     (qa["cls_repr"] * da["cls_repr"]).sum(1)).float()
            big[f"{model}/{pool}/scores"], big[f"{model}/{pool}/amp_scores"] = s.numpy(), a.numpy()
            big[f"{model}/{pool}/amp_max_abs"] = np.float64((a - s).abs().max())
            print("bert-base", model, pool, "scores", s[:4].tolist(), "amp max|dscore|",
                  float(big[f"{model}/{pool}/amp_max_abs"]), "max|score|", float(s.abs().max()))
    np.savez_compressed(os.path.join(HERE, "multivec_bert_base.npz"), **big)
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
