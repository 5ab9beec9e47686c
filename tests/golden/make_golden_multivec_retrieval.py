#!/usr/bin/env python3
"""Golden vectors for COIL / CITADEL retrieval from an expert index, produced by the UNMODIFIED reference.

  python tests/golden/make_golden_multivec_retrieval.py     # writes tests/golden/multivec_retrieval_small.npz

The reference is imported as make_golden_colbert.install sets it up.  No reference source is edited.  Its
CITADELRetrievalTask imports ``dpr_scale.index.inverted_vector_index``, which is not in its tree; a recording stub of
that module is put into ``sys.modules`` first.  For every case of RETRIEVAL below the reference task loads a checkpoint
holding two seeded tiny encoders (multivec_cases.task_state_dict), sets up over the passage table of PASSAGE_IDS and
runs ``_eval_step`` on the case's two query batches.  Recorded:
  * per query, what ``_eval_step`` passes to ``index.search``: the experts of its embeddings / weights dicts in key
    order with their stacked payloads and weights, and the CLS rows;
  * the query and passage encoder outputs (the passages: the case's two passage batches, corpus ids PASSAGE_IDS) and,
    in float64, ``expert_sim_score`` (query_pool sum) plus, with add_cls, ``sim_score`` of the CLS vectors, per (query
    batch, passage batch);
  * the files ``test_epoch_end`` writes from fixed results: TREC with and without index2docid_path, and QA json.
"""
import collections
import json
import os
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
from tests import multivec_cases, multivec_index_cases as cases  # noqa: E402

# name -> (encoder, topk, add_cls)
RETRIEVAL = {"coil_bert": ("coil_bert", 1, False), "coil_bert_cls": ("coil_bert", 1, True),
             "citadel_bert_k1_cls": ("citadel_bert", 1, True), "citadel_bert_k2": ("citadel_bert", 2, False)}
PASSAGE_IDS = list(range(100, 107))                 # the corpus ids of multivec_index_cases.batches(seed=5)
KEYS = ("expert_repr", "expert_ids", "expert_weights", "attention_mask", "cls_repr")
# fixed results for test_epoch_end: (scores, corpus ids) per query
RESULTS = ([[2.5, 1.0000004, -0.125], [0.0, 3.25, 1e-7]], [[103, 100, 106], [101, 105, 102]])


def passage_table(path):
    with open(path, "w") as f:
        f.write("id\ttext\ttitle\n")
        for i in PASSAGE_IDS:
            f.write(f"{i}\tpassage text {i}\ttitle {i}\n")
    return path


def install_index_stub(calls):
    class IVFGPUIndex:
        def __init__(self, *args, **kwargs):
            self.latency = collections.defaultdict(float)

        def search(self, batch_cls, batch_embeddings, batch_weights, topk):
            calls.append((batch_cls, batch_embeddings, batch_weights, topk))
            n = len(batch_embeddings)
            return torch.zeros(n, topk), torch.zeros(n, topk, dtype=torch.long)

    mod = types.ModuleType("dpr_scale.index.inverted_vector_index")
    mod.IVFGPUIndex = mod.IVFCPUIndex = mod.IVFPQGPUIndex = mod.IVFPQCPUIndex = IVFGPUIndex
    pkg = types.ModuleType("dpr_scale.index")
    pkg.inverted_vector_index = mod
    sys.modules["dpr_scale.index"] = pkg
    sys.modules["dpr_scale.index.inverted_vector_index"] = mod


def main():
    install()
    calls = []
    install_index_stub(calls)
    from dpr_scale.task.citadel_retrieval_task import CITADELRetrievalTask
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29566")
    dist.init_process_group("gloo", rank=0, world_size=1)    # test_epoch_end calls barrier() unconditionally
    out = {}
    tmp = tempfile.mkdtemp()
    table = passage_table(os.path.join(tmp, "passages.tsv"))
    for case, (enc, topk, add_cls) in RETRIEVAL.items():
        mdir = multivec_cases.model_dir(os.path.join(tmp, case), enc)
        ckpt = os.path.join(tmp, case + ".ckpt")
        torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)
        kw = cases.task_kwargs(enc, mdir, topk, add_cls)
        kw["model"]["_target_"] = "dpr_scale.models.citadel_models." + multivec_cases.TARGETS[multivec_cases.TINY[enc][0]]
        task = CITADELRetrievalTask(ctx_embeddings_dir=os.path.join(tmp, "idx"), checkpoint_path=ckpt,
                                    output_path=os.path.join(tmp, "run"), passages=table, topk=3, **kw)
        task.setup("test")
        task.eval()
        q_outs, c_outs, seen = [], [], []
        with torch.no_grad():
            for i, (toks, ids) in enumerate(cases.batches(enc, seed=6)):
                del calls[:]
                task._eval_step({"query_ids": toks, "topic_ids": ids}, i)
                batch_cls, emb, wts, _ = calls[0]
                out[f"{case}/q{i}/topic_ids"] = np.array(ids)
                if add_cls:
                    out[f"{case}/q{i}/batch_cls"] = batch_cls.numpy()
                for j, (e, w) in enumerate(zip(emb, wts)):
                    assert list(e) == list(w)
                    out[f"{case}/q{i}/{j}/experts"] = np.array(list(e), dtype=np.int64)
                    for x in e:
                        out[f"{case}/q{i}/{j}/x{x}/repr"] = torch.stack(e[x]).float().numpy()
                        out[f"{case}/q{i}/{j}/x{x}/dtype"] = np.array(str(e[x][0].dtype))
                        out[f"{case}/q{i}/{j}/x{x}/weight"] = torch.stack(w[x]).float().numpy()
                r = task.encode_queries(toks)
                q_outs.append(r)
                for k in KEYS:
                    if k in r:
                        out[f"{case}/q{i}/{k}"] = r[k].numpy()
            for i, (toks, ids) in enumerate(cases.batches(enc, seed=5)):
                seen.extend(int(c) for c in ids)
                r = task.encode_contexts(toks)
                c_outs.append(r)
                for k in KEYS:
                    if k in r:
                        out[f"{case}/c{i}/{k}"] = r[k].numpy()
            assert seen == PASSAGE_IDS
            for qi, q in enumerate(q_outs):
                q64 = {k: (v.double() if v.is_floating_point() else v) for k, v in q.items()}
                for ci, c in enumerate(c_outs):
                    c64 = {k: (v.double() if v.is_floating_point() else v) for k, v in c.items()}
                    s = task.expert_sim_score(q64, c64)
                    if add_cls:
                        s = s + task.sim_score(q64["cls_repr"], c64["cls_repr"])
                    out[f"{case}/score/q{qi}/c{ci}"] = s.numpy()
        print(case, "queries", sum(len(b[1]) for b in cases.batches(enc, seed=6)))

    # the files test_epoch_end writes from fixed results
    i2d = os.path.join(tmp, "i2d.txt")
    with open(i2d, "w") as f:
        f.write("".join(f"doc{i}\n" for i in range(110)))
    enc = "coil_bert"
    mdir = multivec_cases.model_dir(os.path.join(tmp, "files"), enc)
    ckpt = os.path.join(tmp, "files.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)
    kw = cases.task_kwargs(enc, mdir, 1, False)
    kw["model"]["_target_"] = "dpr_scale.models.citadel_models." + multivec_cases.TARGETS["coil"]
    scores, ids = RESULTS
    for name, i2d_path, qa in (("trec", None, False), ("trec_i2d", i2d, False), ("qa", None, True)):
        odir = os.path.join(tmp, "out_" + name)
        task = CITADELRetrievalTask(ctx_embeddings_dir=os.path.join(tmp, "idx"), checkpoint_path=ckpt,
                                    output_path=odir, passages=table, topk=3, index2docid_path=i2d_path, **kw)
        task.setup("test")
        res = [(scores, ids, [], ["who is q1?", "what is q2?"], [["a1"], ["a2", "b2"]])] if qa else \
            [(scores, ids, ["q1", "q2"], [], [])]
        task.index.latency["encode_time"] = 0.0
        task.test_epoch_end(res)
        fname = "retrieval_0000.json" if qa else "retrieval_0000.trec"
        with open(os.path.join(odir, fname), "rb") as f:
            out[f"files/{name}"] = np.frombuffer(f.read(), dtype=np.uint8)
    out["files/results"] = np.array(json.dumps(RESULTS))
    np.savez_compressed(os.path.join(HERE, "multivec_retrieval_small.npz"), **out)
    shutil.rmtree(tmp, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
