"""SPAR on the H100 kernels:
  * SalientPhraseAwareDenseRetrieverTask's query and passage embeddings against [dense, w * lex] / [dense, lex] from the
    float64 oracle encoder, and the widths the generation tasks write;
  * spar_retrieval against the reference's goldens for concat, mean and sum pooling (one and two segments, saved
    embeddings), and against a float64 exact search over a 100 000 x 1536 concatenated store;
  * tune_spar_weights with GPU pool scoring against the reference's goldens;
  * end to end: generate_*_embeddings task=spar -> run_retrieval -> eval_dpr gives the accuracies, and the passages,
    that per-model embeddings -> spar_retrieval --pooling concat -> eval_dpr gives.
"""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import distill_cases, spar_cases as C
from tests.test_spar_cpu import _spar_argv
from tests.util import rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "tests", "golden", "data")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "spar_small.npz"))


# ------------------------------------------------------------------ the task
def _conf(projection_dim=None):
    return {"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "config": distill_cases.WEAK_CFG,
            "dropout": 0.0, "projection_dim": projection_dim}


def _checkpoints(tmp_path):
    """dense: separate encoders, width 128; lexical: shared encoder with a 16-wide projection."""
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    paths, states = [], []
    for name, shared, pd, seeds in (("dense", False, None, (600, 601)), ("lex", True, 16, (602, 603))):
        t = DenseRetrieverTask(transform={}, model=_conf(pd), datamodule=None, optim={}, shared_model=shared)
        t.setup("fit")
        sq = distill_cases.encoder_state(distill_cases.WEAK_CFG, seeds[0], pd)
        t.query_encoder.load_state_dict(sq)
        sc = sq
        if not shared:
            sc = distill_cases.encoder_state(distill_cases.WEAK_CFG, seeds[1], pd)
            t.context_encoder.load_state_dict(sc)
        paths.append(str(tmp_path / f"{name}.ckpt"))
        torch.save(ModelCheckpoint._payload(t, 0, 0), paths[-1])
        states.append((sq, sc))
    return paths, states


def _tokens(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, 64, (n, S), generator=g)
    am = torch.ones(n, S, dtype=torch.long)
    am[1::2, S // 2:] = 0
    return {"input_ids": ids * am, "token_type_ids": torch.zeros_like(ids), "attention_mask": am}


def test_spar_embeddings_against_float64_oracle(tmp_path):
    from dpr_scale_b200.task.spar_task import (SalientPhraseAwareDenseRetrieverTask, SparGenerateEmbeddingsTask,
                                               SparGenerateQueryEmbeddingsTask)
    from oracle import encoder as oenc
    (dense, lex), ((dq, dc), (lq, lc)) = _checkpoints(tmp_path)
    w = 0.7
    kw = dict(pretrained_checkpoint_path=dense, lexical_model_checkpoint_path=lex, lexical_weight=w, transform={},
              model={}, datamodule=None, optim={})
    task = SalientPhraseAwareDenseRetrieverTask(in_batch_eval=False, **kw)
    task.setup("test")
    task = task.cuda().eval()
    q_ids, c_ids = _tokens(6, 24, 1), _tokens(9, 32, 2)
    with torch.no_grad():
        q, c = task(q_ids, c_ids)
    ocfg = {"layers": 1, "heads": 2, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}

    def enc(sd, toks):
        return oenc.encode({k: v.double() for k, v in sd.items()}, ocfg, toks)
    want_q = torch.cat([enc(dq, q_ids), w * enc(lq, q_ids)], 1)
    want_c = torch.cat([enc(dc, c_ids), enc(lc, c_ids)], 1)
    assert q.dtype == torch.float32 and q.shape == (6, 128 + 16) and c.shape == (9, 128 + 16)
    assert rel_l2(q.cpu().double(), want_q) <= 1e-2 and rel_l2(c.cpu().double(), want_c) <= 1e-2
    assert rel_l2(q[:, 128:].cpu().double(), want_q[:, 128:]) <= 1e-2     # the weighted lexical block on its own
    for cls, key, want, name in ((SparGenerateEmbeddingsTask, "contexts_ids", c, "reps_0000.pkl"),
                                 (SparGenerateQueryEmbeddingsTask, "query_ids", q, "query_reps.pkl")):
        dump = cls(ctx_embeddings_dir=str(tmp_path / "emb"), checkpoint_path=None, **kw)
        dump.setup("test")
        dump = dump.cuda().eval()
        dump.test_step({key: c_ids if key == "contexts_ids" else q_ids}, 0)
        out = dump.test_epoch_end([len(want)])
        assert os.path.basename(out) == name
        with open(out, "rb") as f:
            reps = pickle.load(f)
        assert reps.shape == want.shape and rel_l2(reps, want.cpu()) <= 1e-5


# ------------------------------------------------------------------ spar_retrieval
@pytest.mark.parametrize("shard", [1, 2])
@pytest.mark.parametrize("pooling,weights", C.RETRIEVAL_CASES)
def test_spar_retrieval_matches_reference(gold, tmp_path, pooling, weights, shard):
    from dpr_scale_b200 import spar_retrieval as S
    dirs = [C.write_model_dir(tmp_path / f"m{m}", m) for m in (1, 2)]
    out = tmp_path / "out"
    save = pooling == "concat" and shard == 2
    argv = _spar_argv(tmp_path, dirs, pooling, weights, out, ["--shard", str(shard)] + ["--save_embeddings"] * save)
    S.main([a if a != "cpu" else "cuda" for a in argv])
    for tag, name, w in zip("ab", C.QUERY_FILES, weights):
        key = f"retrieval/{pooling}_{tag}.json"
        run = json.load(open(out / f"{pooling}_{tag}.json"))
        rows = np.asarray([[int(c["id"]) - 1 for c in q["ctxs"]] for q in run])
        scores = np.asarray([[c["score"] for c in q["ctxs"]] for q in run])
        q64, p64 = C.pooled_float64(pooling, w, name)
        C.check_ranking(rows, scores, q64, p64, gold[key + "/ids"] - 1)
    if save:
        for name in [f"reps_000{i}.pkl" for i in range(8)] + list(C.QUERY_FILES):
            C.check_saved(gold, out / name, name)


def test_spar_retrieval_large_store_against_float64(tmp_path):
    """100 000 passages x (768 + 768) concatenated, model 2 weighted 0.5, in two segments; each query has 40 planted
    passages along its model-1 vector so the top of its list is well separated."""
    from dpr_scale_b200 import spar_retrieval as S
    N, D, Q, w = 100_000, 768, 64, 0.5
    g = torch.Generator(device="cuda").manual_seed(11)
    q1, q2 = torch.randn(Q, D, device="cuda", generator=g), torch.randn(Q, D, device="cuda", generator=g)
    p1, p2 = torch.randn(N, D, device="cuda", generator=g), torch.randn(N, D, device="cuda", generator=g)
    planted = torch.randperm(N, device="cuda", generator=g)[:Q * 40].view(Q, 40)
    p1[planted] = q1[:, None, :] * (1.0 + 0.05 * torch.arange(40, device="cuda"))[None, :, None]
    for m, (p, q), split in ((1, (p1, q1), [37_000, 63_000]), (2, (p2, q2), [50_000, 25_000, 25_000])):
        d = tmp_path / f"m{m}"
        d.mkdir()
        start = 0
        for i, n in enumerate(split):
            with open(d / f"reps_{i:04}.pkl", "wb") as f:
                pickle.dump(p[start:start + n].cpu(), f, protocol=4)
            start += n
        with open(d / "query_reps.pkl", "wb") as f:
            pickle.dump(q.cpu(), f, protocol=4)
    with open(tmp_path / "psgs.tsv", "w") as f:
        f.write("id\ttext\ttitle\n" + "".join(f"{i + 1}\tpassage {i}\tt{i}\n" for i in range(N)))
    with open(tmp_path / "q.jsonl", "w") as f:
        f.write("".join(json.dumps({"question": f"q{i}", "answers": ["x"]}) + "\n" for i in range(Q)))
    S.main(["--model_1_emb_dir", str(tmp_path / "m1"), "--model_2_emb_dir", str(tmp_path / "m2"),
            "--tsv_passages_path", str(tmp_path / "psgs.tsv"), "--jsonl_dataset_paths", str(tmp_path / "q.jsonl"),
            "--output_dir", str(tmp_path / "out"), "--pred_filenames", "run.json", "--query_reps_filenames",
            "query_reps.pkl", "--weights", str(w), "--topk", "100", "--shard", "2"])
    run = json.load(open(tmp_path / "out" / "run.json"))
    rows = np.asarray([[int(c["id"]) - 1 for c in q["ctxs"]] for q in run])
    scores = np.asarray([[c["score"] for c in q["ctxs"]] for q in run])
    qc = torch.cat([q1, w * q2], 1).double().cpu()
    pc = torch.cat([p1, p2], 1).double().cpu()
    C.check_ranking(rows, scores, qc, pc, min_separated=0.3)
    assert (np.sort(rows[:, :40], 1) == np.sort(planted.cpu().numpy(), 1)).all()


# ------------------------------------------------------------------ tune_spar_weights
def test_tuning_on_gpu_equals_reference(gold, tmp_path):
    from dpr_scale_b200 import tune_spar_weights as T
    regex, ks, valid_k = C.TUNE_CASES[1]
    dirs = [C.write_model_dir(tmp_path / f"m{m}", m) for m in (1, 2)]
    C.write_golden_preds(gold, dirs)
    best, _, _ = T.grid_search_weights(dirs[0], dirs[1], C.PRED_FILE, "query_reps_a.pkl", output_dir=str(tmp_path / "o"),
                                       eval_on_ks=ks, valid_on_k=valid_k, regex=regex, device="cuda")
    assert best == float(gold["tune/1/best_weight"])
    C.check_tuned_runs(gold, str(tmp_path / "o"), T.DEFAULT_WEIGHTS)


# ------------------------------------------------------------------ end to end
def _run(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return res.stdout


def test_end_to_end_spar_generation_retrieval_eval(tmp_path):
    from dpr_scale_b200 import eval_dpr
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    from tests.test_distill_gpu import _tiny_model_dir
    mdir = _tiny_model_dir(tmp_path / "model")
    paths = []
    for i, (shared, pd) in enumerate(((False, None), (True, 16))):
        t = DenseRetrieverTask(transform={}, model={"_target_": "dpr_scale_b200.models.hf_model.HFEncoder",
                                                    "model_path": mdir, "dropout": 0.0, "projection_dim": pd},
                               datamodule=None, optim={}, shared_model=shared)
        t.setup("fit")
        with torch.no_grad():
            gen = torch.Generator().manual_seed(70 + i)
            for p in t.parameters():
                p.add_(0.02 * torch.randn(p.shape, generator=gen))
        paths.append(str(tmp_path / f"m{i}.ckpt"))
        torch.save(ModelCheckpoint._payload(t, 0, 0), paths[-1])
    passages = os.path.join(DATA, "passages.tsv")
    texts = [ln.split("\t") for ln in open(passages).read().splitlines()[1:]]
    qs = [ln.split("\t")[1] for ln in open(os.path.join(DATA, "questions.tsv")).read().splitlines()]
    answers = [[texts[(3 * i) % len(texts)][1].split()[2]] for i in range(len(qs))]
    with open(tmp_path / "q.csv", "w") as f:
        f.write("".join(f"{q}\t{a!r}\n" for q, a in zip(qs, answers)))
    with open(tmp_path / "q.jsonl", "w") as f:
        f.write("".join(json.dumps({"question": q, "answers": a}) + "\n" for q, a in zip(qs, answers)))
    w = 0.6
    common = [f"task.model.model_path={mdir}", "task.transform.max_seq_len=32"]
    gen_p = ["datamodule=generate", f"datamodule.test_path={passages}", "datamodule.test_batch_size=4"]
    gen_q = ["datamodule=generate_query_emb", f"datamodule.test_path={tmp_path / 'q.csv'}",
             "datamodule.test_batch_size=3"]
    spar = ["task=spar", f"task.pretrained_checkpoint_path={paths[0]}", f"task.lexical_model_checkpoint_path={paths[1]}",
            f"task.lexical_weight={w}", f"+task.ctx_embeddings_dir={tmp_path / 'spar'}"] + common
    _run(["dpr_scale_b200.generate_embeddings"] + gen_p + spar)
    _run(["dpr_scale_b200.generate_query_embeddings"] + gen_q + spar)
    with open(tmp_path / "spar" / "query_reps.pkl", "rb") as f:
        assert pickle.load(f).shape == (len(qs), 128 + 16)
    for i, p in enumerate(paths):
        one = [f"+task.checkpoint_path={p}", f"+task.ctx_embeddings_dir={tmp_path / f'm{i}'}"] + common
        if i == 1:
            one += ["task.shared_model=true", "task.model.projection_dim=16"]
        _run(["dpr_scale_b200.generate_embeddings"] + gen_p + one)
        _run(["dpr_scale_b200.generate_query_embeddings"] + gen_q + one)
    _run(["dpr_scale_b200.run_retrieval", f"--ctx_embeddings_dir={tmp_path / 'spar'}",
          f"--questions_tsv_path={tmp_path / 'q.csv'}", f"--passages_tsv_path={passages}",
          f"--output_runfile_path={tmp_path / 'run_spar.json'}", "--topk=5"])
    _run(["dpr_scale_b200.spar_retrieval", f"--model_1_emb_dir={tmp_path / 'm0'}", f"--model_2_emb_dir={tmp_path / 'm1'}",
          f"--tsv_passages_path={passages}", f"--jsonl_dataset_paths={tmp_path / 'q.jsonl'}",
          f"--output_dir={tmp_path / 'out'}", "--pred_filenames=run.json", "--query_reps_filenames=query_reps.pkl",
          f"--weights={w}", "--topk=5"])
    ks = [1, 2, 5]
    a = eval_dpr.evaluate_retrieval(str(tmp_path / "run_spar.json"), ks)
    b = eval_dpr.evaluate_retrieval(str(tmp_path / "out" / "run.json"), ks)
    assert a == b and 0 < sum(a[5])
    ra, rb = json.load(open(tmp_path / "run_spar.json")), json.load(open(tmp_path / "out" / "run.json"))
    assert [[c["id"] for c in q["ctxs"]] for q in ra] == [[c["id"] for c in q["ctxs"]] for q in rb]
