#!/usr/bin/env python3
"""Golden vectors for COIL / CITADEL expert-index generation, produced by the UNMODIFIED reference.

  python tests/golden/make_golden_multivec_index.py        # writes tests/golden/multivec_index_small.npz

The reference is imported as make_golden_colbert.install sets it up.  No reference source is edited.  For every case of
tests/multivec_index_cases.py the reference's GenerateMultiVecEmbeddingsTask (passages) or
GenerateMultiVecQueryEmbeddingsTask (queries) loads a checkpoint holding two seeded tiny encoders
(multivec_cases.task_state_dict), runs test_step on the case's two token batches and test_epoch_end.  Recorded:
  * per batch, the encoder outputs the step used (expert_repr, expert_ids, expert_weights, attention_mask, cls_repr)
    and the batch's input_ids;
  * passages: every expert_0000/{expert}.pkl (ids, weights, reprs) and cls_0000.pkl;
  * queries: query_id.pkl, and per query the experts of its query_repr.pkl / query_weight.pkl dicts in the
    reference's key order with their stacked payloads and weights, and query_cls.pkl.
Also the batches of the reference's citadel DenseRetrieverQueriesDataModule over the fixture question files (TREC
format: topic ids; CSV format: answers), batch size 4, with the fixture tokenizer.
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
from tests import multivec_cases, multivec_index_cases as cases, rerank_cases  # noqa: E402

KEYS = ("expert_repr", "expert_ids", "expert_weights", "attention_mask", "cls_repr")


def load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def main():
    install()
    from dpr_scale.task.citadel_eval_task import GenerateMultiVecEmbeddingsTask, GenerateMultiVecQueryEmbeddingsTask
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29564")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()
    ckpts, mdirs = {}, {}
    for enc in multivec_cases.TINY:
        mdirs[enc] = multivec_cases.model_dir(os.path.join(tmp, enc), enc)
        ckpts[enc] = os.path.join(tmp, enc + ".ckpt")
        torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpts[enc])

    def model_conf(enc, kw):
        model = multivec_cases.TINY[enc][0]
        kw["model"]["_target_"] = "dpr_scale.models.citadel_models." + multivec_cases.TARGETS[model]
        return kw

    for case, (enc, topk, add_cls, ctx_id, thr) in cases.PASSAGE.items():
        odir = os.path.join(tmp, "p_" + case)
        task = GenerateMultiVecEmbeddingsTask(ctx_embeddings_dir=odir, checkpoint_path=ckpts[enc],
                                              add_context_id=ctx_id, weight_threshold=thr,
                                              **model_conf(enc, cases.task_kwargs(enc, mdirs[enc], topk, add_cls)))
        task.setup("test")
        task.eval()
        outs = []
        with torch.no_grad():
            for i, (toks, ids) in enumerate(cases.batches(enc)):
                r = task(toks)
                for k in KEYS:
                    if k in r:
                        out[f"p/{case}/b{i}/{k}"] = r[k].numpy()
                out[f"p/{case}/b{i}/input_ids"] = toks["input_ids"].numpy()
                outs.append(task.test_step({"contexts_ids": toks, "corpus_ids": ids}, i))
        task.test_epoch_end(outs)
        edir = os.path.join(odir, "expert_0000")
        experts = sorted(int(f[:-4]) for f in os.listdir(edir))
        out[f"p/{case}/experts"] = np.array(experts, dtype=np.int64)
        for x in experts:
            ids, w, reps = load(os.path.join(edir, f"{x}.pkl"))
            assert ids.dtype == torch.int64 and w.dtype == reps.dtype == torch.float32
            out[f"p/{case}/x{x}/ids"], out[f"p/{case}/x{x}/weights"] = ids.numpy(), w.numpy()
            out[f"p/{case}/x{x}/reprs"] = reps.numpy()
        if os.path.exists(os.path.join(odir, "cls_0000.pkl")):
            out[f"p/{case}/cls"] = load(os.path.join(odir, "cls_0000.pkl")).numpy()
        n = sum(len(out[f"p/{case}/x{x}/ids"]) for x in experts)
        print("passages", case, "experts", len(experts), "entries", n)

    for case, (enc, topk, add_cls) in cases.QUERY.items():
        odir = os.path.join(tmp, "q_" + case)
        task = GenerateMultiVecQueryEmbeddingsTask(ctx_embeddings_dir=odir, checkpoint_path=ckpts[enc],
                                                   add_context_id=False, query_emb_output_dir=odir,
                                                   **model_conf(enc, cases.task_kwargs(enc, mdirs[enc], topk, add_cls)))
        task.setup("test")
        task.eval()
        outs = []
        with torch.no_grad():
            for i, (toks, ids) in enumerate(cases.batches(enc, seed=6)):
                r = task(toks)
                for k in KEYS:
                    if k in r:
                        out[f"q/{case}/b{i}/{k}"] = r[k].numpy()
                out[f"q/{case}/b{i}/input_ids"] = toks["input_ids"].numpy()
                outs.append(task.test_step({"query_ids": toks, "topic_ids": ids}, i))
        task.test_epoch_end(outs)
        out[f"q/{case}/topic_ids"] = np.array(load(os.path.join(odir, "query_id.pkl")))
        reprs, weights = load(os.path.join(odir, "query_repr.pkl")), load(os.path.join(odir, "query_weight.pkl"))
        assert len(reprs) == len(weights) == len(out[f"q/{case}/topic_ids"])
        for j, (e, w) in enumerate(zip(reprs, weights)):
            assert list(e) == list(w)
            out[f"q/{case}/{j}/experts"] = np.array(list(e), dtype=np.int64)
            for x in e:
                assert all(t.dtype == torch.float32 for t in e[x] + w[x]) and all(t.dim() == 0 for t in w[x])
                out[f"q/{case}/{j}/x{x}/repr"] = torch.stack(e[x]).numpy()
                out[f"q/{case}/{j}/x{x}/weight"] = torch.stack(w[x]).numpy()
        if os.path.exists(os.path.join(odir, "query_cls.pkl")):
            out[f"q/{case}/cls"] = load(os.path.join(odir, "query_cls.pkl")).numpy()
        print("queries", case, [len(e) for e in reprs])
    from dpr_scale.datamodule.citadel import DenseRetrieverQueriesDataModule
    from dpr_scale.transforms.hf_transform import HFTransform
    tok_dir = rerank_cases.tokenizer_dir(os.path.join(tmp, "tok"))
    for fmt, path in (("trec", "questions.tsv"), ("csv", "questions.csv")):
        dm = DenseRetrieverQueriesDataModule(transform=HFTransform(tok_dir, max_seq_len=rerank_cases.MAX_LEN),
                                             test_path=os.path.join(rerank_cases.DATA, path), test_batch_size=4,
                                             trec_format=fmt == "trec")
        bs = list(dm.test_dataloader())
        out[f"dm/{fmt}/n_batches"] = np.int64(len(bs))
        for i, b in enumerate(bs):
            for k, v in b["query_ids"].items():
                out[f"dm/{fmt}/b{i}/query_ids/{k}"] = v.numpy()
            for k in ("question", "topic_ids", "answers"):
                if k in b:
                    out[f"dm/{fmt}/b{i}/{k}"] = np.array(json.dumps(b[k]))
            out[f"dm/{fmt}/b{i}/keys"] = np.array(sorted(b))
    np.savez_compressed(os.path.join(HERE, "multivec_index_small.npz"), **out)
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
