"""SPLADE and dense (DPR) reranking on the GPU:

  * dprb_splade_pool_fwd against float64 on the same fp16 operands and fp32 bias, over N in {1, 3, 257}, segment lengths
    0, 1, 63, 64, 65, 127, 128, 129 and 511 mixed within a call, V in {1, 8, 255, 256, 257, 30522, 50265} and K in
    {64, 128, 768, 1024} with ldx = ldw = K and K + 8.  Gate per element: 2^-12 of (max over the segment's rows of
    sum_k |x_rk W_vk|, plus |bias_v|) - the fp32 accumulation of exact fp16 products over K <= 1024 terms errs by at
    most K 2^-24 <= 2^-14 of that sum, and log1p(relu(.)) is 1-Lipschitz - plus 2^-20 of the value for log1pf's own
    rounding.  Poisoned (NaN) rows before off[0] and after off[N] and NaN columns beyond K show they never reach a result;
  * exact checks: empty segments give exact-zero rows, permuting or regrouping sequences permutes the rows bit for bit,
    repeated calls are bitwise equal, NaN-sentinel outputs with ldo > V and guard rows show every [N, V] element written
    and nothing else, a call with more than 65 535 tiles is compared element by element, and bad shapes are refused
    before any launch;
  * SPLADEEncoder against the float64 oracle (tiny BERT / RoBERTa, padding and masked tails) and at BERT-base dims against
    the reference's golden; RerankDenseRetrieverTask with HFEncoder and SPLADEEncoder against the float64 oracle and the
    golden pickles, dedupe on / off bitwise equal, and python -m dpr_scale_b200.rerank end to end.
"""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.util import GOLDEN

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENGTHS = (0, 1, 63, 64, 65, 127, 128, 129, 511)
GUARD = 5                                           # poisoned rows before off[0] and after off[N]


# ------------------------------------------------------------------ pool kernel
def _case(N, V, K, ld, lengths, seed):
    """x fp16 [GUARD + T + GUARD, ld] (guard rows and columns >= K are NaN), W fp16 [V, ld] (columns >= K NaN),
    bias fp32 [V], off int32 [N + 1] starting at GUARD."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor([lengths[(seed + i) % len(lengths)] for i in range(N)], dtype=torch.long)
    T = int(lens.sum())
    x = torch.full((GUARD + T + GUARD, ld), float("nan"))
    x[GUARD:GUARD + T, :K] = torch.randn(T, K, generator=g)
    W = torch.full((V, ld), float("nan"))
    W[:, :K] = torch.randn(V, K, generator=g) / K ** 0.5
    bias = 0.5 * torch.randn(V, generator=g)
    off = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)]) + GUARD
    return x.half().cuda(), W.half().cuda(), bias.cuda(), off.int().cuda()


def _reference(x, W, bias, off, K):
    """float64 out [N, V] and its gate, one sequence at a time."""
    Wd = W[:, :K].double()
    b = bias.double()
    offs = off.tolist()
    N, V = len(offs) - 1, W.shape[0]
    ref = torch.zeros(N, V, dtype=torch.float64, device=W.device)
    gate = torch.zeros(N, V, dtype=torch.float64, device=W.device)
    for n in range(N):
        lo, hi = offs[n], offs[n + 1]
        if hi == lo:
            continue
        xs = x[lo:hi, :K].double()
        ref[n] = torch.log1p(torch.relu((xs @ Wd.T).max(0).values + b))
        gate[n] = 2.0 ** -12 * ((xs.abs() @ Wd.abs().T).max(0).values + b.abs())
    return ref, gate + 2.0 ** -20 * ref + 1e-30


def _pool(x, W, bias, off, K, out=None):
    from dpr_scale_b200 import ops
    return ops.splade_pool(x, W, off, K, bias, out)


@pytest.mark.parametrize("K", [64, 128, 768, 1024])
@pytest.mark.parametrize("pad", [0, 8])
def test_pool_matches_float64(K, pad):
    worst, cases = 0.0, 0
    for vi, V in enumerate((1, 8, 255, 256, 257, 30522, 50265)):
        for N in ((1, 3, 257) if V <= 257 else (1, 3)):
            seed = K * 1000 + pad * 100 + vi * 10 + N
            x, W, bias, off = _case(N, V, K, K + pad, LENGTHS, seed)
            got = _pool(x, W, bias, off, K)
            ref, gate = _reference(x, W, bias, off, K)
            err = (got.double() - ref).abs() / gate
            worst = max(worst, float(err.max()))
            cases += 1
            assert bool(torch.isfinite(got).all()), (N, V, K, pad)
            assert bool((err <= 1.0).all()), (N, V, K, pad, float(err.max()))
            empty = (off[1:] == off[:-1]).cpu()
            assert bool((got[empty.cuda()] == 0).all())                     # an empty segment is an exact-zero row
            assert torch.equal(_pool(x, W, bias, off, K), got)              # bitwise repeatable
    print(f"splade_pool K={K} ld=K+{pad}: worst error {worst:.3g} of the gate over {cases} cases")


def test_pool_without_bias_and_all_negative_logits():
    x, W, bias, off = _case(3, 257, 128, 128, LENGTHS, seed=7)
    ref, gate = _reference(x, W, torch.zeros_like(bias), off, 128)
    got = _pool(x, W, None, off, 128)
    assert bool(((got.double() - ref).abs() <= gate).all())
    got = _pool(x, W, torch.full_like(bias, -1e4), off, 128)
    assert bool((got == 0).all())


def test_permuting_and_regrouping_sequences_is_bitwise():
    N, V, K = 40, 30522, 768
    lengths = (0, 1, 63, 64, 65, 127, 128, 129, 511, 7, 200)
    x, W, bias, off = _case(N, V, K, K, lengths, seed=11)
    base = _pool(x, W, bias, off, K)
    offs = off.tolist()
    segs = [x[offs[n]:offs[n + 1]] for n in range(N)]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(3)).tolist()
    xp = torch.cat([segs[p] for p in perm])
    lens = torch.tensor([offs[p + 1] - offs[p] for p in perm])
    offp = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)]).int().cuda()
    got = _pool(xp, W, bias, offp, K)
    assert torch.equal(got.view(torch.int32), base[perm].view(torch.int32))
    for cut in (1, 17, 39):                                   # two calls over disjoint groups of sequences
        a = _pool(x, W, bias, off[:cut + 1], K)
        b = _pool(x, W, bias, off[cut:], K)
        assert torch.equal(torch.cat([a, b]).view(torch.int32), base.view(torch.int32)), cut


def test_every_element_written_and_nothing_else():
    N, V, K, G, ldo = 257, 30522, 768, 3, 30522 + 37
    x, W, bias, off = _case(N, V, K, K, LENGTHS, seed=13)
    buf = torch.full((N + 2 * G, ldo), float("nan"), device="cuda")
    _pool(x, W, bias, off, K, out=buf[G:G + N])
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:G]).all()) and bool(torch.isnan(buf[G + N:]).all())
    assert bool(torch.isnan(buf[G:G + N, V:]).all())
    assert not bool(torch.isnan(buf[G:G + N, :V]).any())
    ref, gate = _reference(x, W, bias, off, K)
    assert bool(((buf[G:G + N, :V].double() - ref).abs() <= gate).all())


def test_more_than_65535_tiles():
    V, K = 50265, 64
    lengths = (107, 0, 64, 150, 1, 129)
    N = 600
    x, W, bias, off = _case(N, V, K, K, lengths, seed=17)
    T = int(off[-1] - off[0])
    tiles = -(-x.shape[0] // 128) * -(-V // 256)
    assert tiles > 65535
    got = _pool(x, W, bias, off, K)
    worst = 0.0
    offs = off.tolist()
    for s in range(0, N, 50):                       # every element, 50 sequences at a time
        ref, gate = _reference(x, W, bias, off[s:s + 51], K)
        err = (got[s:s + 50].double() - ref).abs() / gate
        worst = max(worst, float(err.max()))
        assert bool((err <= 1.0).all()), s
    print(f"splade_pool {tiles} tiles (T={T}, V={V}): worst error {worst:.3g} of the gate; {len(offs) - 1} sequences")


def test_bad_shapes_are_rejected_before_any_launch():
    from dpr_scale_b200 import _lib, ops
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    buf = torch.zeros(1 << 20, dtype=torch.float16, device="cuda")
    out = torch.zeros(1 << 16, device="cuda")
    off = torch.tensor([0, 4, 8], dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    good = dict(ldx=64, ldw=64, T=8, N=2, V=100, K=64, ldo=100)
    bad = [dict(K=0), dict(K=60), dict(K=1032), dict(ldx=56), dict(ldx=68), dict(ldw=56), dict(ldw=68), dict(V=0),
           dict(N=0), dict(ldo=99), dict(T=-1), dict(T=1 << 31)]
    for change in bad:
        a = dict(good, **change)
        assert lib.dprb_splade_pool_fwd(p, a["ldx"], p, a["ldw"], None, off.data_ptr(), a["T"], a["N"], a["V"], a["K"],
                                        out.data_ptr(), a["ldo"], st) == 1, change
    assert lib.dprb_splade_pool_fwd(p + 2, 64, p, 64, None, off.data_ptr(), 8, 2, 100, 64, out.data_ptr(), 100, st) == 1
    assert lib.dprb_splade_pool_fwd(p, 64, p, 64, None, None, 8, 2, 100, 64, out.data_ptr(), 100, st) == 1
    with pytest.raises(ValueError):
        ops.splade_pool(buf[:8 * 64].view(8, 64), buf[:100 * 64].view(100, 64), off, 72)
    with pytest.raises(ValueError):
        ops.splade_pool(buf[:8 * 64].view(8, 64), buf[:100 * 64].view(100, 64), off, 64,
                        out=out[:2 * 50].view(2, 50))
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ encoders
def _oracle_cfg(kind):
    from tests import rerank_cases
    return rerank_cases.ORACLE_CFG[kind]


@pytest.mark.parametrize("name", ["splade_bert", "splade_roberta"])
@pytest.mark.parametrize("S", [20, 257])
def test_tiny_encoders_match_oracle(name, S):
    from oracle import splade as osp
    from tests import colbert_cases, splade_cases
    kind, _ = splade_cases.TINY[name]
    sd = splade_cases.tiny_state_dict(name)
    m = splade_cases.build(name, sd).cuda()
    cfg = colbert_cases.encoder_config(kind)
    toks = splade_cases.tiny_tokens(cfg, S=S, n=7, seed=S)
    with torch.no_grad():
        got = m(toks).cpu()
    ref = osp.reps(sd, _oracle_cfg(kind), toks)
    err = float((got.double() - ref).abs().max())
    gate = 2.0 ** -7 * float(ref.abs().max())
    print(f"{name} S={S}: max|err| {err:.3g} = {err / gate:.3g} of the gate")
    assert got.dtype == torch.float32 and got.shape == ref.shape and err <= gate
    assert bool((got[-1] == 0).all())


def test_bert_base_matches_reference_golden():
    """Reps (every 16th vocabulary column) and rerank scores within twice the reference's own bf16-autocast deviation."""
    from dpr_scale_b200.models.citadel_models.splade_model import SPLADEEncoder
    from tests import colbert_cases, splade_cases
    raw = np.load(os.path.join(GOLDEN, "splade_bert_base.npz"))
    g = {k: torch.from_numpy(raw[k]) for k in raw.files}
    sd, cfg = splade_cases.bert_base_state_dict()
    assert torch.equal(colbert_cases.sd_checksum(sd), g["checksum"]), "seeded weights differ from the golden's"
    m = SPLADEEncoder.from_config(cfg)
    m.load_state_dict(sd, strict=True)
    m.cuda()
    q = {k.split("/")[-1]: g[k] for k in g if k.startswith("query/") and "reps" not in k}
    d = {k.split("/")[-1]: g[k] for k in g if k.startswith("passage/") and "reps" not in k}
    with torch.no_grad():
        qr, dr = m(q).cpu(), m(d).cpu()
    cs = splade_cases.BASE_COL_STRIDE
    for side, r in (("query", qr), ("passage", dr)):
        diff = float((r[:, ::cs] - g[f"{side}/reps_cols"]).abs().max())
        amp = float(g[f"{side}/amp_reps_max_abs"])
        print(f"bert-base SPLADE {side} reps: max|drep| {diff:.3g}, reference bf16 autocast {amp:.3g}")
        assert diff <= 2.0 * amp
    s = (qr * dr).sum(1)
    diff = float((s - g["scores"]).abs().max())
    amp = float(g["amp_max_abs"])
    print(f"bert-base SPLADE scores: max|dscore| {diff:.3g}, reference bf16 autocast {amp:.3g}, "
          f"max|score| {float(g['scores'].abs().max()):.4g}")
    assert diff <= 2.0 * amp


# ------------------------------------------------------------------ the task and the CLI
def _task(tmp_path, model):
    from dpr_scale_b200.task.dpr_rerank_task import RerankDenseRetrieverTask
    from tests import splade_cases
    _, _, proj, seed = splade_cases.TASK[model]
    ckpt = str(tmp_path / f"{model}.ckpt")
    torch.save({"state_dict": splade_cases.task_state_dict(model)}, ckpt)
    mdir = splade_cases.model_dir(str(tmp_path / f"{model}_model"), model, seed)
    mconf = {"_target_": splade_cases.TARGETS[model].replace("dpr_scale.", "dpr_scale_b200."), "model_path": mdir}
    if proj:
        mconf["projection_dim"] = proj
    task = RerankDenseRetrieverTask(checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), transform={},
                                    datamodule=None, optim={}, shared_model=False, model=mconf)
    return ckpt, mdir, task


def _cli_args(mdir, ckpt, out_dir, model):
    from tests import rerank_cases, splade_cases
    kw = rerank_cases.datamodule_kwargs()
    proj = splade_cases.TASK[model][2]
    extra = [f"task.model.projection_dim={proj}"] if proj else []
    return ["task=dpr_rerank", f"task/model={'hf_model' if model == 'hf' else 'splade_model'}",
            "datamodule=multivec_rerank", f"task.model.model_path={mdir}", *extra,
            f"task.transform.max_seq_len={rerank_cases.MAX_LEN}", f"datamodule.test_path={kw['test_path']}",
            f"datamodule.test_question_path={kw['test_question_path']}",
            f"datamodule.test_passage_path={kw['test_passage_path']}",
            f"datamodule.test_batch_size={kw['test_batch_size']}", "datamodule.use_title=true",
            f"+task.checkpoint_path={ckpt}", f"+task.output_dir={out_dir}"]


def _pickles(out_dir, rank=0):
    got = {}
    for what in ("scores", "qids", "ctx_ids"):
        with open(os.path.join(out_dir, f"{what}_{rank:04}.pkl"), "rb") as f:
            got[what] = pickle.load(f)
    return got


@pytest.mark.parametrize("model", ["hf", "splade"])
def test_rerank_task_and_cli(tmp_path, model):
    """Each batch's scores against the float64 oracle and the reference's pickle.  Gate: 2^-7 of the largest per-pair
    sum |q| . |d| (the scores inherit the bf16 encoder's relative error on every term).  Dedupe on / off are bitwise
    equal.  The CLI's pickles: the reference's qids / ctx ids and scores bitwise those of the batches; rerank.trec in
    descending score order, and in the golden's order wherever its adjacent gaps exceed twice the gate."""
    from dpr_scale_b200 import rerank
    from oracle import splade as osp
    from tests import splade_cases
    from tests.test_colbert_cpu import golden_batches
    raw = np.load(os.path.join(GOLDEN, "splade_small.npz"))
    ckpt, mdir, task = _task(tmp_path, model)
    task.setup("test")
    task.cuda()
    full = splade_cases.task_state_dict(model)
    enc = osp.dense if model == "hf" else osp.reps
    ours, ref, bound = [], [], []
    for b in golden_batches():
        bc = dict(b, query_ids={k: v.cuda() for k, v in b["query_ids"].items()},
                  contexts_ids={k: v.cuda() for k, v in b["contexts_ids"].items()})
        task.dedupe_queries = True
        s = task._scores(bc).cpu()
        task.dedupe_queries = False
        assert torch.equal(task._scores(bc).cpu().view(torch.int32), s.view(torch.int32))
        ours.append(s)
        q = enc(full, _oracle_cfg("bert"), b["query_ids"], "query_encoder.")
        d = enc(full, _oracle_cfg("bert"), b["contexts_ids"], "context_encoder.")
        ref.append(osp.rerank_score(q, d))
        bound.append(osp.rerank_score(q.abs(), d.abs()))
    ours, ref, bound = torch.cat(ours), torch.cat(ref), torch.cat(bound)
    gate = 2.0 ** -7 * float(bound.max())
    err = float((ours.double() - ref).abs().max())
    want = torch.from_numpy(raw[f"{model}/pkl/scores"])
    dev = float((ours - want).abs().max())
    print(f"dense rerank {model}: max|dscore| vs float64 {err:.3g} = {err / gate:.3g} of the gate; vs the reference's "
          f"pickle {dev:.3g} (max|score| {float(want.abs().max()):.3g})")
    assert err <= gate and dev <= gate

    out_dir = str(tmp_path / "cli_out")
    task.dedupe_queries = True
    run = rerank.main(_cli_args(mdir, ckpt, out_dir, model))
    got = _pickles(out_dir)
    assert got["qids"] == raw[f"{model}/pkl/qids"].tolist()
    assert got["ctx_ids"] == raw[f"{model}/pkl/ctx_ids"].tolist()
    s = got["scores"]
    assert torch.is_tensor(s) and s.dtype == torch.float32 and torch.equal(s, ours)
    lines = [ln.split() for ln in open(run).read().splitlines()]
    assert len(lines) == len(got["qids"])
    score_of = {(q, c): v for q, c, v in zip(got["qids"], got["ctx_ids"], s.tolist())}
    gold_of = {(q, c): v for q, c, v in zip(got["qids"], got["ctx_ids"], want.tolist())}
    for q in dict.fromkeys(ln[0] for ln in lines):
        ids = [ln[2] for ln in lines if ln[0] == q]
        vals = [score_of[(q, c)] for c in ids]
        assert vals == sorted(vals, reverse=True)
        gold = sorted(ids, key=lambda c: -gold_of[(q, c)])
        for a, b in zip(gold, gold[1:]):                 # the golden's order holds where its gaps are clear
            if gold_of[(q, a)] - gold_of[(q, b)] > 2 * gate:
                assert ids.index(a) < ids.index(b), (q, a, b)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_shards_concatenate_to_the_one_rank_output(tmp_path):
    ckpt, mdir, _ = _task(tmp_path, "splade")
    one, two = str(tmp_path / "one"), str(tmp_path / "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    for nproc, out in ((1, one), (2, two)):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m",
               "dpr_scale_b200.rerank"] + _cli_args(mdir, ckpt, out, "splade")
        subprocess.run(cmd, check=True, cwd=ROOT, env=env, timeout=600)
    a = _pickles(one)
    parts = [_pickles(two, r) for r in range(2)]
    assert a["qids"] == parts[0]["qids"] + parts[1]["qids"]
    assert a["ctx_ids"] == parts[0]["ctx_ids"] + parts[1]["ctx_ids"]
    # SPLADE vectors do not depend on the padded width, so the shards' scores are the one-rank scores
    b = torch.cat([parts[0]["scores"], parts[1]["scores"]])
    assert float((a["scores"] - b).abs().max()) <= 1e-3 * max(1.0, float(a["scores"].abs().max()))
