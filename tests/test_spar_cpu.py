"""SPAR and answer-accuracy host logic against goldens of the UNMODIFIED reference (tests/golden/make_golden_spar.py ->
spar_small.npz): eval_dpr accuracy lists and augmented runs in both matching modes, tune_spar_weights with the host's
fp32 scoring in place of the GPU's, spar_retrieval's host flow with the search kernels replaced by torch emulations,
command-line refusals, and the ``task=spar`` config and checkpoint key names."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from tests import spar_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "spar_small.npz"))


def _text(gold, key):
    return str(gold[key])


# ------------------------------------------------------------------ eval_dpr
@pytest.mark.parametrize("regex", [False, True])
def test_eval_dpr_equals_reference(gold, tmp_path, regex, capsys):
    from dpr_scale_b200 import eval_dpr
    tag = "regex" if regex else "tokens"
    run = tmp_path / "run.json"
    run.write_text(C.golden_run_text(gold, f"retrieval/{C.EVAL_RUN}"))
    aug = tmp_path / "aug.json"
    argv = ["--retrieval", str(run), "--topk"] + [str(k) for k in C.EVAL_KS] + ["--output_eval_results", str(aug)]
    acc = eval_dpr.main(argv + (["--regex"] if regex else []))
    for k in C.EVAL_KS:
        assert acc[k] == gold[f"eval/{tag}/top{k}"].tolist(), k
    assert C.sha256(aug.read_text()) == _text(gold, f"eval/{tag}/augmented_sha256")
    assert eval_dpr.evaluate_retrieval(str(run), C.EVAL_KS, regex) == acc
    out = capsys.readouterr().out
    assert f"Top{C.EVAL_KS[-1]}\taccuracy: {np.mean(acc[C.EVAL_KS[-1]])}" in out


def test_has_answers_rules():
    from dpr_scale_b200.eval_dpr import has_answers
    assert has_answers("Lake Zürich, 1969.", ["zürich"])               # NFD text, NFC answer, uncased
    assert not has_answers("Zürichsee", ["Zürich"])                            # whole tokens only
    assert has_answers("the U.S. army", ["u.s."]) and has_answers("at & t", ["AT&T"])
    assert not has_answers("colour", ["colou?r"]) and has_answers("COLOR", ["colou?r"], regex=True)
    assert not has_answers("(unclosed", ["(unclosed"], regex=True)             # a pattern that does not compile
    assert has_answers("anything", ["  "]) and not has_answers("a b", ["  "], regex=True)


# ------------------------------------------------------------------ tune_spar_weights
@pytest.mark.parametrize("case", range(len(C.TUNE_CASES)))
def test_tuning_equals_reference(gold, tmp_path, case, capsys):
    from dpr_scale_b200 import tune_spar_weights as T
    regex, ks, valid_k = C.TUNE_CASES[case]
    dirs = [C.write_model_dir(tmp_path / f"m{m}", m) for m in (1, 2)]
    C.write_golden_preds(gold, dirs)
    out = tmp_path / "out"
    timings = {}
    best, best_acc, accs = T.grid_search_weights(dirs[0], dirs[1], C.PRED_FILE, "query_reps_a.pkl", output_dir=str(out),
                                                 eval_on_ks=ks, valid_on_k=valid_k, regex=regex, device="cpu",
                                                 workers=2, timings=timings)
    log = [ln for ln in capsys.readouterr().out.splitlines()
           if ln.startswith(("Accuracy for weight", "Top", "The best weight"))]
    assert "\n".join(log) == _text(gold, f"tune/{case}/log")
    assert best == float(gold[f"tune/{case}/best_weight"])
    assert sorted(os.listdir(out)) == gold[f"tune/{case}/files"].tolist()
    assert set(timings) >= {"load", "answer_matching", "pool_scoring_and_accuracy", "write"}
    C.check_tuned_runs(gold, out, T.DEFAULT_WEIGHTS)
    assert set(accs) == set(T.DEFAULT_WEIGHTS)


def test_tuning_refusals(tmp_path):
    from dpr_scale_b200 import tune_spar_weights as T
    with pytest.raises(ValueError, match="valid_on_k"):
        T.grid_search_weights("a", "b", "p.json", "q.pkl", eval_on_ks=[1, 5], valid_on_k=100, device="cpu")
    with pytest.raises(FileNotFoundError, match="p.json"):
        T.grid_search_weights(str(tmp_path), str(tmp_path), "p.json", "q.pkl", device="cpu")


# ------------------------------------------------------------------ spar_retrieval
def _emulate_search(monkeypatch):
    from dpr_scale_b200 import ops

    def fake_search(q, c, k, index_offset=0, reference_ranking=False):
        s = q.float() @ c.float().T
        v, i = torch.sort(s, dim=1, descending=True, stable=True)
        return v[:, :k].contiguous(), i[:, :k] + index_offset

    def fake_merge(s, idx, k):
        v, o = torch.sort(s, dim=1, descending=True, stable=True)
        return v[:, :k].contiguous(), torch.gather(idx, 1, o[:, :k])
    monkeypatch.setattr(ops, "search_topk", fake_search)
    monkeypatch.setattr(ops, "topk_merge", fake_merge)


def _spar_argv(tmp_path, dirs, pooling, weights, out, extra=()):
    return ["--model_1_emb_dir", dirs[0], "--model_2_emb_dir", dirs[1], "--tsv_passages_path", C.PASSAGES,
            "--jsonl_dataset_paths", C.QUESTIONS, C.QUESTIONS, "--output_dir", str(out),
            "--pred_filenames", f"{pooling}_a.json", f"{pooling}_b.json",
            "--query_reps_filenames", *C.QUERY_FILES, "--weights", *[str(w) for w in weights],
            "--topk", str(C.TOPK), "--pooling", pooling, "--device", "cpu", *extra]


@pytest.mark.parametrize("shard", [1, 2])
@pytest.mark.parametrize("pooling,weights", C.RETRIEVAL_CASES)
def test_spar_retrieval_host_flow(gold, tmp_path, monkeypatch, pooling, weights, shard):
    from dpr_scale_b200 import spar_retrieval as S
    _emulate_search(monkeypatch)
    monkeypatch.setattr(S, "CHUNK_ROWS", 64)                   # chunks that straddle both models' file boundaries
    dirs = [C.write_model_dir(tmp_path / f"m{m}", m) for m in (1, 2)]
    out = tmp_path / "out"
    save = pooling == "concat" and shard == 2
    S.main(_spar_argv(tmp_path, dirs, pooling, weights, out, ["--shard", str(shard)] + (["--save_embeddings"] * save)))
    for tag, name, w in zip("ab", C.QUERY_FILES, weights):
        key = f"retrieval/{pooling}_{tag}.json"
        run = json.load(open(out / f"{pooling}_{tag}.json"))
        questions = [json.loads(ln) for ln in open(C.QUESTIONS)]
        assert [q["question"] for q in run] == [q["question"] for q in questions]
        assert [q["id"] for q in run] == [q.get("id", str(i)) for i, q in enumerate(questions)]
        assert all(list(q) == ["question", "answers", "ctxs", "id"] for q in run)
        rows = np.asarray([[int(c["id"]) - 1 for c in q["ctxs"]] for q in run])
        scores = np.asarray([[c["score"] for c in q["ctxs"]] for q in run])
        q64, p64 = C.pooled_float64(pooling, w, name)
        C.check_ranking(rows, scores, q64, p64, gold[key + "/ids"] - 1)
        kept = gold[key + "/scores"]
        np.testing.assert_allclose(scores[:, :kept.shape[1]], kept, atol=float(C.fp16_bound(q64, p64).max()))
    if save:
        for name in [f"reps_000{i}.pkl" for i in range(8)] + list(C.QUERY_FILES):
            C.check_saved(gold, out / name, name)


def test_spar_retrieval_refusals(tmp_path, monkeypatch):
    from dpr_scale_b200 import spar_retrieval as S
    _emulate_search(monkeypatch)
    dirs = [C.write_model_dir(tmp_path / f"m{m}", m) for m in (1, 2)]
    out = tmp_path / "out"
    argv = _spar_argv(tmp_path, dirs, "concat", [0.5, 1.0], out)
    with pytest.raises(ValueError, match="--weights has 1"):
        S.main(argv[:argv.index("--weights") + 2] + argv[argv.index("--weights") + 3:])
    with pytest.raises(ValueError, match="--pred_filenames has 1"):
        S.main(argv[:argv.index("--pred_filenames") + 2] + argv[argv.index("--pred_filenames") + 3:])
    with pytest.raises(ValueError, match="unknown pooling 'max'"):
        S.main(_spar_argv(tmp_path, dirs, "max", [0.5, 1.0], out))
    with pytest.raises(FileNotFoundError, match="query_reps_x.pkl"):
        S.main([a if a != "query_reps_b.pkl" else "query_reps_x.pkl" for a in argv])
    with pytest.raises(FileNotFoundError, match="reps_"):
        S.main([a if a != dirs[1] else str(tmp_path) for a in argv])
    with pytest.raises(FileNotFoundError, match="nope.tsv"):
        S.main([a if a != C.PASSAGES else str(tmp_path / "nope.tsv") for a in argv])
    os.remove(os.path.join(dirs[1], "reps_0001.pkl"))
    with pytest.raises(ValueError, match="fewer passage vectors"):
        S.main(argv)
    assert not (out / "concat_a.json").exists()
    big = torch.full((C.N_PASSAGES, C.DIM), 7e4)
    with open(os.path.join(dirs[1], "reps_0000.pkl"), "wb") as f:
        pickle.dump(big, f, protocol=4)
    with pytest.raises(ValueError, match="does not fit fp16"):
        S.main(argv)


def test_mean_pooling_needs_equal_widths(tmp_path):
    from dpr_scale_b200 import spar_retrieval as S
    assert S.pooled_width(32, 24, "concat") == 56
    with pytest.raises(ValueError, match="widths"):
        S.pooled_width(32, 24, "mean")


# ------------------------------------------------------------------ task=spar
def _checkpoint(tmp_path, name, seed, shared_model=False, projection_dim=None):
    from dpr_scale_b200.task.dpr_task import DenseRetrieverTask
    from dpr_scale_b200.utils.checkpoint import ModelCheckpoint
    torch.manual_seed(seed)
    model = {"_target_": "dpr_scale_b200.models.hf_model.HFEncoder.from_config", "dropout": 0.0,
             "projection_dim": projection_dim,
             "config": dict(vocab_size=64, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                            intermediate_size=256, max_position_embeddings=40)}
    t = DenseRetrieverTask(transform={}, model=model, datamodule=None, optim={}, shared_model=shared_model)
    t.setup("fit")
    path = str(tmp_path / name)
    torch.save(ModelCheckpoint._payload(t, 0, 0), path)
    return path, t


def test_spar_config_and_state_dict_keys(tmp_path):
    from dpr_scale_b200 import generate_embeddings as G
    from dpr_scale_b200.utils.config import compose, instantiate
    dense, td = _checkpoint(tmp_path, "dense.ckpt", 1)
    lex, tl = _checkpoint(tmp_path, "lex.ckpt", 2, shared_model=True, projection_dim=16)
    cfg = compose("config", ["task=spar", f"task.pretrained_checkpoint_path={dense}",
                             f"task.lexical_model_checkpoint_path={lex}", "task.lexical_weight=0.7"])
    cfg.task.datamodule = None
    task = instantiate(cfg.task, _recursive_=False)
    assert type(task).__name__ == "SalientPhraseAwareDenseRetrieverTask" and task.lexical_weight == 0.7
    task.setup("test")
    sd = task.state_dict()
    assert {k for k in sd} == {"dense_model." + k for k in td.state_dict()} | {"lexical_model." + k for k in tl.state_dict()}
    for k, v in td.state_dict().items():
        assert torch.equal(sd["dense_model." + k], v)
    assert task.query_encoder is task.dense_model.query_encoder
    assert task.lexical_model.query_encoder is task.lexical_model.context_encoder
    assert task.configure_optimizers() is None
    spar = "dpr_scale_b200.task.spar_task.SalientPhraseAwareDenseRetrieverTask"
    assert G.ENSEMBLE_DUMPS[spar] == {G.TASK: "dpr_scale_b200.task.spar_task.SparGenerateEmbeddingsTask",
                                      G.QUERY_TASK: "dpr_scale_b200.task.spar_task.SparGenerateQueryEmbeddingsTask"}


def test_spar_missing_or_corrupt_checkpoint(tmp_path):
    from dpr_scale_b200.task.spar_task import SalientPhraseAwareDenseRetrieverTask as Spar
    dense, _ = _checkpoint(tmp_path, "dense.ckpt", 1)
    kw = dict(transform={}, model={}, datamodule=None, optim={})
    with pytest.raises(FileNotFoundError, match="nope.ckpt"):
        Spar(pretrained_checkpoint_path=dense, lexical_model_checkpoint_path=str(tmp_path / "nope.ckpt"), **kw).setup("test")
    bad = tmp_path / "bad.ckpt"
    bad.write_bytes(b"not a checkpoint")
    with pytest.raises(RuntimeError, match="bad.ckpt"):
        Spar(pretrained_checkpoint_path=str(bad), lexical_model_checkpoint_path=dense, **kw).setup("test")
    with pytest.raises(ValueError, match="lexical_model_checkpoint_path"):
        Spar(pretrained_checkpoint_path=dense, **kw).setup("test")
