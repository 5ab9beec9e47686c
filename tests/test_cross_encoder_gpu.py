"""Cross-encoder reranking on the GPU:

  * dprb_seqcls_head_fwd against float64 for N in {1, 7, 1000}, H in {128, 768, 1024}, L in {1, 2, 3}; bad shapes are
    rejected before any launch;
  * tiny BERT (1 label) and RoBERTa (2 labels) CrossEncoders against the float64 oracle at S in {24, 300, 512}, with
    padding and segment-B token types (gates of tests/test_long_seq_gpu.py's tiny models: rel-L2 <= 1e-2);
  * BERT-base dims (seeded weights, checked by checksum) against the reference's logits in the golden, with a gate of
    twice the reference's own bf16-autocast deviation on the same pairs;
  * python -m dpr_scale_b200.rerank end to end on the fixture run: qids / ctx ids equal to the reference's pickles,
    scores within tolerance, [n, 1] with one label and [n] with two, and a sorted rerank.trec;
  * 2-rank shards concatenate to the 1-rank output (needs 2 GPUs);
  * an unsupported config or sequence raises before any launch.
"""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import rerank_cases
from tests.util import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _npz(name):
    raw = np.load(os.path.join(GOLDEN, name))
    return raw, {k: torch.from_numpy(raw[k]) for k in raw.files if raw[k].dtype.kind != "U"}


# ------------------------------------------------------------------ head kernel
@pytest.mark.parametrize("N", [1, 7, 1000])
@pytest.mark.parametrize("H", [128, 768, 1024])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_head_kernel_matches_float64(N, H, L):
    from dpr_scale_b200 import ops
    g = torch.Generator().manual_seed(N * 7 + H + L)
    pre = 2.0 * torch.randn(N, H, generator=g)          # tanh both linear and saturated
    W = 0.05 * torch.randn(L, H, generator=g)
    b = torch.randn(L, generator=g)
    logits, score = ops.seqcls_head_fwd(pre.cuda(), W.cuda(), b.cuda())
    torch.cuda.synchronize()
    t = torch.tanh(pre.double())
    ref = t @ W.double().T + b.double()
    bound = (t.abs() @ W.double().abs().T) + b.double().abs()      # sum of |terms|
    err = (logits.cpu().double() - ref).abs()
    assert bool((err <= 1e-6 + 2e-6 * bound).all()), float((err / (1e-6 + bound)).max())
    assert torch.equal(score.cpu(), logits.cpu().max(1).values)


def test_head_kernel_rejects_bad_shapes_before_launching():
    from dpr_scale_b200 import ops
    from dpr_scale_b200._lib import DprbError
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for H, L in ((100, 1), (1032, 1), (128, 0), (128, ops.SEQCLS_MAX_LABELS + 1)):
        pre = torch.zeros(4, H, device="cuda")
        W = torch.zeros(max(L, 1), H, device="cuda")[:L] if L else torch.zeros(0, H, device="cuda")
        with pytest.raises(DprbError):
            ops.seqcls_head_fwd(pre, W, torch.zeros(max(L, 1), device="cuda"))
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ tiny models vs the oracle
def _tiny(kind):
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    m = CrossEncoder.from_config(rerank_cases.tiny_config(kind), seed=3)
    with torch.no_grad():                     # non-zero biases / LayerNorm parameters; logits of order 1
        gen = torch.Generator().manual_seed(4)
        for p in m.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=gen))
        dense, out = m._head_linears()
        out.weight.mul_(20.0)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    return m.cuda(), sd


@pytest.mark.parametrize("kind", ["bert", "roberta"])
@pytest.mark.parametrize("S", [24, 300, 512])
def test_tiny_cross_encoder_matches_oracle(kind, S):
    from oracle import cross_encoder as oce
    m, sd = _tiny(kind)
    cfg = rerank_cases.tiny_config(kind)
    toks = rerank_cases.pair_tokens(torch.Generator().manual_seed(S), 6, S, cfg["vocab_size"], cfg["pad_token_id"])
    logits, score = m.logits_and_scores(toks)
    torch.cuda.synchronize()
    ref = oce.logits(sd, rerank_cases.ORACLE_CFG[kind], toks)
    assert logits.shape == (6, cfg["num_labels"]) and logits.dtype == torch.float32
    err = rel_l2(logits.cpu(), ref)
    print(kind, S, "logits rel-L2", f"{err:.3g}", "max|ref|", float(ref.abs().max()))
    assert err <= 1e-2, err
    assert torch.equal(score, logits.max(1).values)
    assert torch.equal(m(toks), logits)                     # deterministic, forward == logits_and_scores()[0]


# ------------------------------------------------------------------ BERT-base dims vs the reference
def test_bert_base_matches_reference_golden():
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    raw, g = _npz("rerank_bert_base.npz")
    model, cfg = rerank_cases.bert_base_seqcls()
    assert torch.equal(rerank_cases.checksums(model), g["checksum"]), "seeded weights differ from the golden's"
    ce = CrossEncoder.from_config(cfg)
    ce.load_state_dict({"transformer." + k: v for k, v in model.state_dict().items()
                        if not k.endswith(("position_ids", "token_type_ids"))}, strict=True)
    del model
    ce = ce.cuda()
    toks = {k.split("/")[-1]: g[k] for k in g if k.startswith("tokens/")}
    logits = ce(toks).cpu()
    want = g["logits"]
    d = float((logits - want).abs().max())
    amp = float(g["amp_max_abs"])
    print(f"bert-base S={rerank_cases.BASE_S}: max|dlogit| {d:.3g}, reference bf16 autocast {amp:.3g}, "
          f"max|logit| {float(want.abs().max()):.3g}, rel-L2 {rel_l2(logits, want):.3g}")
    assert d <= max(2.0 * amp, 2e-3), (d, amp)
    assert rel_l2(logits, want) <= 1e-2


# ------------------------------------------------------------------ the CLI
def _cli_args(model_dir, out_dir, kw):
    return ["task=cross_encoder_rerank", "task/model=cross_encoder", "datamodule=cross_encoder_rerank",
            f"task.model.model_path={model_dir}", f"task.transform.max_seq_len={rerank_cases.MAX_LEN}",
            f"datamodule.test_path={kw['test_path']}", f"datamodule.test_question_path={kw['test_question_path']}",
            f"datamodule.test_passage_path={kw['test_passage_path']}",
            f"datamodule.test_batch_size={kw['test_batch_size']}", "datamodule.use_title=true",
            f"+task.output_dir={out_dir}"]


def _model_dir(tmp_path, kind):
    """The seeded tiny model the reference's pickles came from (checked by checksum), as a checkpoint directory."""
    raw, g = _npz("rerank_small.npz")
    cfg = json.loads(str(raw[f"{kind}/config"]))
    sd = rerank_cases.reference_state_dict(kind)
    assert torch.equal(rerank_cases.sd_checksum(sd), g[f"{kind}/sd_checksum"]), "seeded weights differ from the golden's"
    mdir = rerank_cases.hf_model_dir(str(tmp_path / f"{kind}_model"), cfg, rerank_cases.TINY[kind]["seed"])
    return mdir, raw, g, sd


def _pickles(d, rank=0):
    out = {}
    for what in ("scores", "qids", "ctx_ids"):
        with open(os.path.join(d, f"{what}_{rank:04}.pkl"), "rb") as f:
            out[what] = pickle.load(f)
    return out


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_rerank_cli_matches_reference_pickles(tmp_path, kind):
    from dpr_scale_b200 import rerank
    mdir, raw, g, sd = _model_dir(tmp_path, kind)
    out_dir = str(tmp_path / f"{kind}_out")
    run = rerank.main(_cli_args(mdir, out_dir, rerank_cases.datamodule_kwargs()))
    got = _pickles(out_dir)
    assert got["qids"] == raw[f"{kind}/pkl/qids"].tolist()
    assert got["ctx_ids"] == raw[f"{kind}/pkl/ctx_ids"].tolist()
    want = g[f"{kind}/pkl/scores"]
    s = got["scores"]
    assert torch.is_tensor(s) and s.dtype == torch.float32 and tuple(s.shape) == tuple(want.shape)
    assert tuple(s.shape) == ((24, 1) if kind == "bert" else (24,))
    # A logit is tanh(features) . w + b with |tanh| <= 1, so a feature error of relative size r moves it by at most
    # r * sqrt(H) * |w|.  These tiny heads have |w| ~ 0.23 and logits of only ~0.03, so the gate is stated on that
    # scale: r = 2e-3 (the oracle tests above measure 1e-3 .. 3e-3 rel-L2 on logits of order 1).
    w = sd["transformer.classifier." + ("weight" if kind == "bert" else "out_proj.weight")]
    gate = 2e-3 * w.shape[1] ** 0.5 * float(w.norm(dim=1).max())
    d = float((s - want).abs().max())
    print(kind, "max|dscore|", d, "gate", gate, "max|score|", float(want.abs().max()))
    assert d <= gate, (d, gate)
    lines = [ln.split() for ln in open(run).read().splitlines()]
    run_rows = [ln.split() for ln in open(rerank_cases.datamodule_kwargs()["test_path"]).read().splitlines()]
    assert len(lines) == len(run_rows)
    flat = s.reshape(-1).tolist()
    score_of = {(q, c): v for q, c, v in zip(got["qids"], got["ctx_ids"], flat)}
    for q in dict.fromkeys(r[0] for r in run_rows):
        mine = [ln for ln in lines if ln[0] == q]
        assert sorted(ln[2] for ln in mine) == sorted(r[2] for r in run_rows if r[0] == q)
        assert [int(ln[3]) for ln in mine] == list(range(1, len(mine) + 1))
        vals = [score_of[(q, ln[2])] for ln in mine]
        assert vals == sorted(vals, reverse=True)
        assert [float(ln[4]) for ln in mine] == vals


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_shards_concatenate_to_the_one_rank_output(tmp_path):
    mdir, raw, g, _ = _model_dir(tmp_path, "roberta")
    kw = rerank_cases.datamodule_kwargs()
    one, two = str(tmp_path / "one"), str(tmp_path / "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    for nproc, out in ((1, one), (2, two)):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m",
               "dpr_scale_b200.rerank"] + _cli_args(mdir, out, kw)
        subprocess.run(cmd, check=True, cwd=ROOT, env=env, timeout=600)
    a = _pickles(one)
    parts = [_pickles(two, r) for r in range(2)]
    assert a["qids"] == parts[0]["qids"] + parts[1]["qids"]
    assert a["ctx_ids"] == parts[0]["ctx_ids"] + parts[1]["ctx_ids"]
    assert len(parts[0]["qids"]) == len(raw["shard2/rank0"])
    assert torch.allclose(a["scores"], torch.cat([parts[0]["scores"], parts[1]["scores"]]), rtol=0, atol=1e-6)
    assert open(os.path.join(one, "rerank.trec")).read() == open(os.path.join(two, "rerank.trec")).read()


# ------------------------------------------------------------------ refusals
def test_unsupported_config_or_sequence_raises_before_any_launch():
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    base = rerank_cases.tiny_config("bert")
    with pytest.raises(ValueError):           # head dim 32 (MiniLM)
        CrossEncoder.from_config(dict(base, hidden_size=384, num_attention_heads=12, intermediate_size=1536))
    m, _ = _tiny("bert")
    n1 = ops.launch_count()
    toks = rerank_cases.pair_tokens(torch.Generator().manual_seed(1), 2, 513, base["vocab_size"], 0)
    with pytest.raises(ValueError):           # beyond the 512 positions
        m(toks)
    assert ops.launch_count() == n1 == n0
