"""ColBERT reranking on the GPU:

  * dprb_maxsim_fwd against float64 on the same bf16 inputs over B x LQ x LD x P x pool, with no mask, suffix padding,
    holes, an all-masked passage and an all-masked query; token 0 of both sides is large, so scoring it shows.  Gate per
    pair: 2^-12 of the sum over its query rows of max_j sum_k |q_ik d_jk| (fp32 accumulation of exact bf16 products);
    the worst error is printed as a share of it.  Exact cases: a padded passage whose real scores are all negative
    scores exactly 0 per row; scores are bitwise repeatable; NaN-sentinel outputs with guard elements show every score
    written and nothing else; more than 65 535 pairs, every one compared; bad shapes are rejected before any launch;
  * the token forward against the float64 oracle (tiny BERT / RoBERTa at S in {24, 128, 257, 512}, BERT-base dims at
    S = 256; gate 2^-7 of max|ref|), padded rows exactly zero, and token row 0 equal to bf16(pooled) of
    dprb_encoder_fwd with DPRB_NO_CLS_PRUNE=1 bit for bit (child process);
  * one encoding per distinct query equals encoding every row, bit for bit;
  * python -m dpr_scale_b200.rerank end to end against the reference's pickles for both pools; BERT-base against the
    golden within twice the reference's own bf16-autocast deviation; the 2-rank split (needs 2 GPUs).
"""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import colbert_cases, rerank_cases
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_CFG = {"bert": rerank_cases.ORACLE_CFG["bert"], "roberta": rerank_cases.ORACLE_CFG["roberta"]}
MASKS = ("none", "suffix", "holes", "dead_passage", "dead_query")


# ------------------------------------------------------------------ MaxSim kernel
def _reference(q, d, qm, dm, idx, pool):
    """float64 scores and the per-pair gate, on the GPU."""
    qz = q.double() * qm.double().unsqueeze(-1)
    dz = d.double() * dm.double().unsqueeze(-1)
    qq, dd = qz[idx.long(), 1:], dz[:, 1:]
    s = torch.bmm(qq, dd.transpose(1, 2)).max(-1).values
    ref = s.sum(1) if pool == "sum" else s.max(1).values
    absb = torch.bmm(qq.abs(), dd.abs().transpose(1, 2)).max(-1).values.sum(1)
    return ref, 2.0 ** -12 * absb + 1e-30


def _masks(kind, n, S, gen):
    m = torch.ones(n, S, dtype=torch.int32)
    if kind == "suffix":
        lens = torch.randint(1, S + 1, (n,), generator=gen)
        lens[0] = S
        m = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).int()
    elif kind == "holes":
        m = (torch.rand(n, S, generator=gen) > 0.3).int()
    return m


def _case(B, LQ, LD, P, mask, seed):
    gen = torch.Generator().manual_seed(seed)
    nq = max(1, (B + 1) // 2)
    SQ, SD = LQ + 1, LD + 1
    q = torch.randn(nq, SQ, P, generator=gen)
    d = torch.randn(B, SD, P, generator=gen)
    q[:, 0] = 100.0                                      # token 0 would dominate every score if it were read
    d[:, 0] = 100.0
    qm = _masks(mask if mask in ("suffix", "holes") else "none", nq, SQ, gen)
    dm = _masks(mask if mask in ("suffix", "holes") else "none", B, SD, gen)
    if mask == "dead_passage":
        dm[-1, 1:] = 0
    if mask == "dead_query":
        qm[0, 1:] = 0
    idx = torch.randint(0, nq, (B,), generator=gen, dtype=torch.int32)
    idx[0] = 0
    return q.to(torch.bfloat16).cuda(), d.to(torch.bfloat16).cuda(), qm.cuda(), dm.cuda(), idx


@pytest.mark.parametrize("P", [64, 128, 136, 768, 1024])
@pytest.mark.parametrize("pool", ["sum", "max"])
def test_maxsim_matches_float64(P, pool):
    from dpr_scale_b200 import ops
    worst, i = 0.0, 0
    for LQ in (1, 31, 32, 63, 64, 65, 130):
        for LD in (1, 63, 64, 65, 127, 128, 129, 255, 511):
            B = (1, 7, 300)[i % 3]
            mask = MASKS[i % len(MASKS)]
            i += 1
            q, d, qm, dm, idx = _case(B, LQ, LD, P, mask, seed=P * 1000 + i)
            got = ops.maxsim(q, d, qm, dm, idx, pool)
            ref, gate = _reference(q, d, qm, dm, idx.cuda(), pool)
            err = (got.double() - ref).abs() / gate
            worst = max(worst, float(err.max()))
            assert bool((err <= 1.0).all()), (B, LQ, LD, P, mask, pool, float(err.max()))
            if mask == "dead_passage":          # every real column of the last pair is masked: each row scores 0
                assert float(got[-1]) == 0.0
            if mask == "dead_query":
                rows = (idx == 0).nonzero().flatten().cuda()           # every row offers exactly 0 (sum and max)
                assert bool((got[rows] == 0.0).all())
            assert torch.equal(ops.maxsim(q, d, qm, dm, idx, pool), got)        # bitwise repeatable
    print(f"maxsim P={P} pool={pool}: worst error {worst:.3g} of the gate")


@pytest.mark.parametrize("pool", ["sum", "max"])
def test_padded_passage_with_negative_scores_gives_exactly_zero(pool):
    from dpr_scale_b200 import ops
    P, LQ, LD = 128, 40, 150
    q = torch.ones(1, LQ + 1, P, dtype=torch.bfloat16, device="cuda")
    d = -torch.rand(2, LD + 1, P).to(torch.bfloat16).cuda()         # every real score is negative
    dm = torch.ones(2, LD + 1, dtype=torch.int32, device="cuda")
    dm[0, 100:] = 0                                                  # pair 0 is shorter than the batch's width
    s = ops.maxsim(q, d, None, dm, torch.zeros(2, dtype=torch.int32), pool)
    assert float(s[0]) == 0.0                                        # max(0, negative) per row, summed
    assert float(s[1]) < 0.0                                         # no padding: the real maxima


def test_every_score_written_and_nothing_else():
    from dpr_scale_b200 import _lib
    q, d, qm, dm, idx = _case(300, 65, 129, 136, "holes", seed=5)
    G = 64
    buf = torch.full((300 + 2 * G,), float("nan"), device="cuda")
    idx_d = idx.cuda()
    rc = _lib.load().dprb_maxsim_fwd(q.data_ptr(), d.data_ptr(), qm.data_ptr(), dm.data_ptr(), idx_d.data_ptr(),
                                     q.shape[0], q.shape[1], 300, d.shape[1], 136, 0, buf.data_ptr() + 4 * G,
                                     torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:G]).all()) and bool(torch.isnan(buf[-G:]).all())
    assert not bool(torch.isnan(buf[G:-G]).any())


def test_more_than_65535_pairs():
    from dpr_scale_b200 import ops
    B = 70_001
    q, d, qm, dm, idx = _case(B, 5, 9, 64, "suffix", seed=9)
    got = ops.maxsim(q, d, qm, dm, idx, "sum")
    ref, gate = _reference(q, d, qm, dm, idx.cuda(), "sum")
    err = (got.double() - ref).abs() / gate
    print(f"maxsim B={B}: worst error {float(err.max()):.3g} of the gate")
    assert got.shape == (B,) and bool((err <= 1.0).all())


def test_bad_shapes_are_rejected_before_any_launch():
    from dpr_scale_b200 import _lib, ops
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    buf = torch.zeros(1 << 20, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(4, device="cuda")
    idx = torch.zeros(4, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for SQ, SD, P, pool in ((8, 8, 100, 0), (8, 8, 1032, 0), (1, 8, 64, 0), (8, 1, 64, 0), (513, 8, 64, 0),
                            (8, 513, 64, 0), (8, 8, 64, 2)):
        assert lib.dprb_maxsim_fwd(buf.data_ptr(), buf.data_ptr(), None, None, idx.data_ptr(), 2, SQ, 4, SD, P, pool,
                                   out.data_ptr(), st) == 1
    with pytest.raises(ValueError):
        ops.maxsim(buf[:2 * 8 * 64].view(2, 8, 64), buf[:4 * 8 * 64].view(4, 8, 64), None, None,
                   torch.tensor([0, 1, 2, 0]))
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ token forward
def _tiny(name):
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    kind, proj, _ = colbert_cases.TINY[name]
    m = ColBERTEncoder.from_config(colbert_cases.encoder_config(kind), projection_dim=proj)
    sd = colbert_cases.tiny_state_dict(name)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


@pytest.mark.parametrize("name", list(colbert_cases.TINY))
@pytest.mark.parametrize("S", [24, 128, 257, 512])
def test_token_forward_matches_oracle(name, S):
    from oracle import colbert as oc
    m, sd = _tiny(name)
    kind = colbert_cases.TINY[name][0]
    cfg = colbert_cases.encoder_config(kind)
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(S), 4, S, cfg["vocab_size"], cfg["pad_token_id"])
    with torch.no_grad():
        rep = m(toks)["expert_repr"].cpu()
    ref = oc.expert_repr(sd, ORACLE_CFG[kind], toks)
    err = float((rep.double() - ref).abs().max())
    gate = 2.0 ** -7 * float(ref.abs().max())
    print(f"{name} S={S}: max|err| {err:.3g} = {err / gate:.3g} of the gate")
    assert rep.dtype == torch.float32 and rep.shape == ref.shape
    assert err <= gate
    assert bool((rep[toks["attention_mask"][:, 1:] == 0] == 0).all())          # padded rows: exact zeros


def test_bert_base_token_forward_matches_oracle():
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    from oracle import colbert as oc
    sd, cfg = colbert_cases.bert_base_state_dict()
    m = ColBERTEncoder.from_config(cfg, projection_dim=colbert_cases.BASE_P)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    _, d = colbert_cases.bert_base_tokens()
    d = {k: v[:3] for k, v in d.items()}
    with torch.no_grad():
        rep = m(d)["expert_repr"].cpu()
    ref = oc.expert_repr(sd, {"layers": 12, "heads": 12, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}, d)
    err = float((rep.double() - ref).abs().max())
    gate = 2.0 ** -7 * float(ref.abs().max())
    print(f"bert-base S=256: max|err| {err:.3g} = {err / gate:.3g} of the gate")
    assert err <= gate


_CHILD = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from tests import colbert_cases
from dpr_scale_b200.models.hf_model import HFEncoder
from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
cfg = colbert_cases.encoder_config("roberta")
sd = colbert_cases.tiny_state_dict("roberta_none")
m = ColBERTEncoder.from_config(cfg); m.load_state_dict(sd, strict=True); m = m.cuda()
e = HFEncoder.from_config(cfg, dropout=0.0)
e.transformer.load_state_dict({k[len("transformer."):]: v for k, v in sd.items()}, strict=True); e = e.cuda().eval()
toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(3), 5, 77, cfg["vocab_size"], cfg["pad_token_id"])
with torch.no_grad():
    reps, _ = m.token_reps(toks)
    pooled = e(toks)
print("SAME" if torch.equal(reps[:, 0].cpu(), pooled.to(torch.bfloat16).cpu()) else "DIFFERENT")
"""


def test_token_row_zero_is_the_unpruned_pooled_output():
    env = dict(os.environ, DPRB_NO_CLS_PRUNE="1")
    out = subprocess.run([sys.executable, "-c", _CHILD, ROOT], env=env, cwd=ROOT, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1] == "SAME"


# ------------------------------------------------------------------ the task
def _npz(name):
    raw = np.load(os.path.join(GOLDEN, name))
    return raw, {k: torch.from_numpy(raw[k]) for k in raw.files if raw[k].dtype.kind != "U"}


def _task(tmp_path, name, pool):
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    ckpt = str(tmp_path / f"{name}.ckpt")
    torch.save({"state_dict": colbert_cases.task_state_dict(name)}, ckpt)
    mdir = colbert_cases.model_dir(str(tmp_path / f"{name}_model"), name)
    return ckpt, mdir, RerankMultiVecRetrieverTask(
        checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), query_pool=pool, transform={}, datamodule=None,
        optim={}, shared_model=False, model={"_target_": "dpr_scale_b200.models.citadel_models.colbert_model."
                                             "ColBERTEncoder", "model_path": mdir,
                                             "projection_dim": colbert_cases.TINY[name][1]})


@pytest.mark.parametrize("pool", ["sum", "max"])
def test_one_encoding_per_distinct_query_is_bit_identical(tmp_path, pool):
    from tests.test_colbert_cpu import golden_batches
    _, _, task = _task(tmp_path, "bert_p128", pool)
    task.setup("test")
    task.cuda()
    for b in golden_batches():
        b = dict(b, query_ids={k: v.cuda() for k, v in b["query_ids"].items()},
                 contexts_ids={k: v.cuda() for k, v in b["contexts_ids"].items()})
        task.dedupe_queries = True
        a = task._scores(b)
        task.dedupe_queries = False
        c = task._scores(b)
        assert torch.equal(a, c)
    assert any(len(set(b["qid"])) < len(b["qid"]) for b in golden_batches())      # the fixture has repeated queries


def _cli_args(mdir, ckpt, out_dir, pool, name):
    kw = rerank_cases.datamodule_kwargs()
    return ["task=multivec_rerank", "task/model=colbert_model", "datamodule=multivec_rerank",
            f"task.model.model_path={mdir}", f"task.model.projection_dim={colbert_cases.TINY[name][1]}",
            f"task.transform.max_seq_len={rerank_cases.MAX_LEN}", f"datamodule.test_path={kw['test_path']}",
            f"datamodule.test_question_path={kw['test_question_path']}",
            f"datamodule.test_passage_path={kw['test_passage_path']}",
            f"datamodule.test_batch_size={kw['test_batch_size']}", "datamodule.use_title=true",
            f"+task.query_pool={pool}", f"+task.checkpoint_path={ckpt}", f"+task.output_dir={out_dir}"]


def _pickles(d, rank=0):
    out = {}
    for what in ("scores", "qids", "ctx_ids"):
        with open(os.path.join(d, f"{what}_{rank:04}.pkl"), "rb") as f:
            out[what] = pickle.load(f)
    return out


@pytest.mark.parametrize("name", colbert_cases.TASK_KINDS)
@pytest.mark.parametrize("pool", ["sum", "max"])
def test_rerank_cli_matches_reference_pickles(tmp_path, name, pool):
    from dpr_scale_b200 import rerank
    raw, g = _npz("colbert_small.npz")
    ckpt, mdir, _ = _task(tmp_path, name, pool)
    out_dir = str(tmp_path / "cli_out")
    run = rerank.main(_cli_args(mdir, ckpt, out_dir, pool, name))
    got = _pickles(out_dir)
    assert got["qids"] == raw[f"{name}/{pool}/pkl/qids"].tolist()
    assert got["ctx_ids"] == raw[f"{name}/{pool}/pkl/ctx_ids"].tolist()
    want = g[f"{name}/{pool}/pkl/scores"]
    s = got["scores"]
    assert torch.is_tensor(s) and s.dtype == torch.float32 and s.shape == want.shape == (24,)
    d = float((s - want).abs().max())
    gate = 2.0 ** -7 * float(want.abs().max())
    print(f"{name} {pool}: max|dscore| {d:.3g} = {d / gate:.3g} of the gate, max|score| {float(want.abs().max()):.3g}")
    assert d <= gate
    lines = [ln.split() for ln in open(run).read().splitlines()]
    assert len(lines) == 24
    score_of = {(q, c): v for q, c, v in zip(got["qids"], got["ctx_ids"], s.tolist())}
    for q in dict.fromkeys(ln[0] for ln in lines):
        vals = [score_of[(q, ln[2])] for ln in lines if ln[0] == q]
        assert vals == sorted(vals, reverse=True)


@pytest.mark.parametrize("pool", ["sum", "max"])
def test_bert_base_matches_reference_golden(pool):
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.colbert_model import ColBERTEncoder
    raw, g = _npz("colbert_bert_base.npz")
    sd, cfg = colbert_cases.bert_base_state_dict()
    assert torch.equal(colbert_cases.sd_checksum(sd), g["checksum"]), "seeded weights differ from the golden's"
    m = ColBERTEncoder.from_config(cfg, projection_dim=colbert_cases.BASE_P)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    q = {k.split("/")[-1]: g[k] for k in g if k.startswith("query/")}
    d = {k.split("/")[-1]: g[k] for k in g if k.startswith("passage/")}
    with torch.no_grad():
        qr, qm = m.token_reps(q)
        dr, dm = m.token_reps(d)
        s = ops.maxsim(qr, dr, qm, dm, torch.arange(colbert_cases.BASE_PAIRS, dtype=torch.int32), pool).cpu()
    want = g[f"{pool}/scores"]
    diff = float((s - want).abs().max())
    amp = float(g[f"{pool}/amp_max_abs"])
    print(f"bert-base {pool}: max|dscore| {diff:.3g}, reference bf16 autocast {amp:.3g}, max|score| "
          f"{float(want.abs().max()):.4g}")
    assert diff <= 2.0 * amp


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_shards_concatenate_to_the_one_rank_output(tmp_path):
    name = "roberta_p128"
    ckpt, mdir, _ = _task(tmp_path, name, "sum")
    one, two = str(tmp_path / "one"), str(tmp_path / "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    for nproc, out in ((1, one), (2, two)):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m",
               "dpr_scale_b200.rerank"] + _cli_args(mdir, ckpt, out, "sum", name)
        subprocess.run(cmd, check=True, cwd=ROOT, env=env, timeout=600)
    raw, _ = _npz("colbert_small.npz")
    a = _pickles(one)
    parts = [_pickles(two, r) for r in range(2)]
    assert a["qids"] == parts[0]["qids"] + parts[1]["qids"]
    assert len(parts[0]["qids"]) == len(raw["shard2/rank0"])
    assert a["ctx_ids"] == parts[0]["ctx_ids"] + parts[1]["ctx_ids"]
    # scores are not compared: each rank pads its own batches, and the padded width takes part in MaxSim
