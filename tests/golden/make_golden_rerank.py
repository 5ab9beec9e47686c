#!/usr/bin/env python3
"""Golden vectors for cross-encoder reranking, produced by the UNMODIFIED reference (/root/reference).

  python tests/golden/make_golden_rerank.py        # writes tests/golden/rerank_small.npz, rerank_bert_base.npz

The reference's datamodule/cross_encoder.py imports TRECDataset from datamodule/dpr.py, where it does not exist; it lives
in datamodule/citadel.py.  This script binds ``dpr_scale.datamodule.dpr.TRECDataset`` to the citadel class before the
import and edits no reference source.  `hydra` and `pytorch_lightning` are stubbed (neither is installed).

rerank_small.npz:
  * batches of ``CrossEncoderRerankDataModule`` (use_title, batch 5, max_seq_len 24, the fixture BERT vocabulary) over
    tests/golden/data/rerank_run.trec with questions.tsv (TREC format) and passages.tsv; the rows of
    ``ContiguousDistributedSamplerForTest`` at 2 ranks;
  * for a tiny BERT (1 label) and a tiny RoBERTa (2 labels), seeded (tests/rerank_cases.py): the config, the reference
    ``CrossEncoder``'s state_dict keys, shapes and fp64 checksum (not its weights), pair tokens (padding, segment-B token
    types) and logits;
  * the three pickles ``RerankCrossEncoderTask.test_epoch_end`` writes for the fixture run with either model.
rerank_bert_base.npz: a seeded BERT-base-dims ``BertForSequenceClassification(num_labels=1)`` (tests/realdims.py recipe:
  weight checksums, not weights) on 16 pairs at S = 256: fp32 logits and the reference's own bf16-autocast logits.
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
DATA = os.path.join(HERE, "data")
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import install_stubs  # noqa: E402
from tests import rerank_cases  # noqa: E402


def install_reference():
    install_stubs()
    pl = sys.modules["pytorch_lightning"]

    class LightningDataModule:
        def __init__(self):
            self.trainer = None
    pl.LightningDataModule = LightningDataModule
    sys.modules["ujson"] = json
    sys.path.insert(0, REF)
    import dpr_scale.datamodule.citadel as citadel
    import dpr_scale.datamodule.dpr as refdpr
    refdpr.TRECDataset = citadel.TRECDataset


def main():
    install_reference()
    from dpr_scale.datamodule.cross_encoder import CrossEncoderRerankDataModule
    from dpr_scale.models.citadel_models.cross_encoder import CrossEncoder
    from dpr_scale.task.cross_encoder_eval_task import RerankCrossEncoderTask
    from dpr_scale.transforms.hf_transform import HFTransform
    from dpr_scale.utils.utils import ContiguousDistributedSamplerForTest
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29561")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()

    # -- datamodule batches
    tok_dir = rerank_cases.tokenizer_dir(os.path.join(tmp, "tok"))
    dm = CrossEncoderRerankDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                      **rerank_cases.datamodule_kwargs())
    batches = list(dm.test_dataloader())
    out["n_batches"] = np.int64(len(batches))
    for i, b in enumerate(batches):
        out[f"batch{i}/qid"] = np.array(b["qid"])
        out[f"batch{i}/ctx_id"] = np.array(b["ctx_id"])
        for k, v in b["text_ids"].items():
            out[f"batch{i}/text_ids/{k}"] = v.numpy()
    n = len(dm.datasets["test"])
    for r in range(2):
        out[f"shard2/rank{r}"] = np.array(list(ContiguousDistributedSamplerForTest(
            dm.datasets["test"], num_replicas=2, rank=r, shuffle=False)), dtype=np.int64)
    print("rows", n, "batches", len(batches), "shards", [len(out[f"shard2/rank{r}"]) for r in range(2)])

    # -- tiny models: logits on random pair tokens, and the rerank pickles of the fixture run
    for kind in rerank_cases.TINY:
        cfg = rerank_cases.tiny_config(kind)
        mdir = rerank_cases.hf_model_dir(os.path.join(tmp, kind), cfg, rerank_cases.TINY[kind]["seed"])
        model = CrossEncoder(model_path=mdir).eval()
        out[f"{kind}/config"] = np.array(json.dumps(cfg))
        sd = model.state_dict()
        out[f"{kind}/sd_keys"] = np.array(list(sd))
        out[f"{kind}/sd_shapes"] = np.array(json.dumps([list(v.shape) for v in sd.values()]))
        out[f"{kind}/sd_checksum"] = rerank_cases.sd_checksum(sd).numpy()
        assert torch.equal(rerank_cases.sd_checksum(rerank_cases.reference_state_dict(kind)),
                           rerank_cases.sd_checksum(sd)), "the seeded rebuild differs from the loaded checkpoint"
        toks = rerank_cases.pair_tokens(torch.Generator().manual_seed(17), 6, 20, cfg["vocab_size"], cfg["pad_token_id"])
        logits = model(toks)
        for k, v in toks.items():
            out[f"{kind}/tokens/{k}"] = v.numpy()
        out[f"{kind}/logits"] = logits.numpy()
        odir = os.path.join(tmp, kind + "_out")
        task = RerankCrossEncoderTask(output_dir=odir, transform={}, datamodule=None, optim={},
                                      model={"_target_": "dpr_scale.models.citadel_models.cross_encoder.CrossEncoder",
                                             "model_path": mdir})
        task.setup("test")
        task.eval()
        outs = [task.test_step(b, i) for i, b in enumerate(dm.test_dataloader())]
        task.test_epoch_end(outs)
        for what in ("scores", "qids", "ctx_ids"):
            with open(os.path.join(odir, f"{what}_0000.pkl"), "rb") as f:
                obj = pickle.load(f)
            out[f"{kind}/pkl/{what}"] = obj.numpy() if torch.is_tensor(obj) else np.array(obj)
        print(kind, "logits", logits.shape, "scores", tuple(out[f"{kind}/pkl/scores"].shape))
    np.savez_compressed(os.path.join(HERE, "rerank_small.npz"), **out)

    # -- BERT-base dims, S = 256
    model, cfg = rerank_cases.bert_base_seqcls()
    big = {"checksum": rerank_cases.checksums(model).numpy()}
    mdir = os.path.join(tmp, "bert_base")
    model.save_pretrained(mdir)
    del model
    ce = CrossEncoder(model_path=mdir).eval()
    toks = rerank_cases.pair_tokens(torch.Generator().manual_seed(1234), rerank_cases.BASE_PAIRS, rerank_cases.BASE_S,
                                    cfg["vocab_size"], 0, lo=1000, cls_id=101, sep_id=102)
    logits = ce(toks)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        amp = ce(toks).float()
    for k, v in toks.items():
        big[f"tokens/{k}"] = v.numpy()
    big["logits"], big["amp_logits"] = logits.numpy(), amp.numpy()
    big["amp_max_abs"] = np.float64((amp - logits).abs().max())
    np.savez_compressed(os.path.join(HERE, "rerank_bert_base.npz"), **big)
    print("bert-base logits", logits.flatten()[:4].tolist(), "amp max|dlogit|", float(big["amp_max_abs"]),
          "max|logit|", float(logits.abs().max()))
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
