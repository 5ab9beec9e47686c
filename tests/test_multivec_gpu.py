"""COIL / CITADEL reranking on the GPU:

  * dprb_maxsim_expert_fwd against float64 (oracle.multivec.expert_score) on the same bf16 inputs, ids and weights, over
    B x LQ x LD x P x KQ x KD x pool x CLS and four id alphabets: dense matches (4 symbols), sparse matches (64 symbols),
    no match at all (the sum is exactly 0 without CLS) and zero weights.  Gate per pair: 2^-12 of the sum over its rows
    (i, a) of max over (j, b) of sum_k |q_ik d_jk| * |wq| * |wd| where the ids agree (fp32 accumulation of exact bf16
    products, two fp32 roundings of the weights), plus 2^-12 of sum |q_cls d_cls|.  Exact cases: with KQ = KD = 1, equal
    ids and the 0/1 masks as weights the scores are dprb_maxsim_fwd's bit for bit; bitwise repeatable; NaN-sentinel
    outputs show every score written and nothing else; 70 001 pairs; bad shapes rejected before any launch;
  * the CITADEL router (the masked-LM head on dprb_search_topk) against float64 logits, the encoders against the float64
    oracle, BERT-base dims against the reference's golden, and python -m dpr_scale_b200.rerank end to end.
"""
import numpy as np
import pytest
import torch

from tests.util import GOLDEN

pytestmark = pytest.mark.gpu

ALPHABETS = ("dense", "sparse", "none", "zero_w")


# ------------------------------------------------------------------ scoring kernel
def _ids(kind, shape, gen, side):
    if kind == "dense":
        return torch.randint(0, 4, shape, generator=gen)
    if kind == "none":                              # disjoint alphabets: nothing ever matches
        return torch.randint(0, 50, shape, generator=gen) + (0 if side == "q" else 1000)
    return torch.randint(0, 64, shape, generator=gen)


def _weights(kind, shape, gen):
    w = torch.rand(shape, generator=gen) * 2.0
    if kind == "zero_w":
        w[torch.rand(shape, generator=gen) < 0.5] = 0.0
    return w


def _case(B, LQ, LD, P, KQ, KD, alphabet, seed, cls=False, Pc=128):
    """Pairs with padded (masked) tokens whose weights are 0; token 0 is large so reading it shows."""
    gen = torch.Generator().manual_seed(seed)
    nq = max(1, (B + 1) // 2)
    SQ, SD = LQ + 1, LD + 1
    q = torch.randn(nq, SQ, P, generator=gen)
    d = torch.randn(B, SD, P, generator=gen)
    q[:, 0] = 100.0
    d[:, 0] = 100.0
    qm = (torch.arange(SQ) < torch.randint(2, SQ + 1, (nq, 1), generator=gen)).float() if SQ > 2 else torch.ones(nq, SQ)
    dm = (torch.arange(SD) < torch.randint(2, SD + 1, (B, 1), generator=gen)).float() if SD > 2 else torch.ones(B, SD)
    qm[0], dm[0] = 1.0, 1.0
    q_ids, d_ids = _ids(alphabet, (nq, SQ, KQ), gen, "q"), _ids(alphabet, (B, SD, KD), gen, "d")
    q_w = _weights(alphabet, (nq, SQ, KQ), gen) * qm.unsqueeze(-1)
    d_w = _weights(alphabet, (B, SD, KD), gen) * dm.unsqueeze(-1)
    q_ids[:, 0], d_ids[:, 0], q_w[:, 0], d_w[:, 0] = 0, 0, 100.0, 100.0      # token 0 is never read
    idx = torch.randint(0, nq, (B,), generator=gen, dtype=torch.int32)
    idx[0] = 0
    qc = dc = None
    if cls:
        qc = torch.randn(nq, Pc, generator=gen).to(torch.bfloat16).cuda()
        dc = torch.randn(B, Pc, generator=gen).to(torch.bfloat16).cuda()
    bf = lambda t: t.to(torch.bfloat16).cuda()
    return (bf(q), bf(d), q_ids.int().cuda(), q_w.cuda(), d_ids.int().cuda(), d_w.cuda(), idx, qc, dc)


def _reference(case, pool, chunk_elems=1 << 27):
    """float64 scores and per-pair gates, on the GPU, a chunk of pairs at a time."""
    from oracle.multivec import expert_score
    q, d, qi, qw, di, dw, idx, qc, dc = case
    idx = idx.cuda().long()
    B, LQ, LD = d.shape[0], q.shape[1] - 1, d.shape[1] - 1
    per = LQ * qi.shape[2] * LD * di.shape[2]
    step = max(1, chunk_elems // per)
    ref, gate = [], []
    for s in range(0, B, step):
        sl = slice(s, min(B, s + step))
        qq, dd = q[idx[sl], 1:].double(), d[sl, 1:].double()
        a = (qi[idx[sl], 1:], qw[idx[sl], 1:], di[sl, 1:], dw[sl, 1:])
        c = (qc[idx[sl]], dc[sl]) if qc is not None else (None, None)
        ref.append(expert_score(qq, dd, *a, pool, *c))
        g = expert_score(qq.abs(), dd.abs(), a[0], a[1].abs(), a[2], a[3].abs(), "sum")
        if qc is not None:
            g = g + (c[0].double() * c[1].double()).abs().sum(1)
        gate.append(2.0 ** -12 * g + 1e-30)
    return torch.cat(ref), torch.cat(gate)


def _run(case, pool):
    from dpr_scale_b200 import ops
    q, d, qi, qw, di, dw, idx, qc, dc = case
    return ops.maxsim_expert(q, d, qi, qw, di, dw, idx, pool, qc, dc)


@pytest.mark.parametrize("P", [32, 64, 128, 136, 1024])
@pytest.mark.parametrize("pool", ["sum", "max"])
def test_maxsim_expert_matches_float64(P, pool):
    worst, i = 0.0, 0
    for LQ in (1, 31, 64, 65, 130):
        for LD in (1, 127, 129, 511):
            for KQ, KD in ((1, 1), (2, 4), (8, 8), (4, 1), (1, 8)):
                B = (1, 7, 300)[i % 3] if KQ * KD <= 8 else (1, 7, 40)[i % 3]
                alphabet = ALPHABETS[i % len(ALPHABETS)]
                cls = i % 2 == 1
                i += 1
                case = _case(B, LQ, LD, P, KQ, KD, alphabet, seed=P * 10000 + i, cls=cls, Pc=(64, 128, 1024)[i % 3])
                got = _run(case, pool)
                ref, gate = _reference(case, pool)
                err = (got.double() - ref).abs() / gate
                worst = max(worst, float(err.max()))
                assert bool((err <= 1.0).all()), (B, LQ, LD, P, KQ, KD, alphabet, cls, pool, float(err.max()))
                if alphabet == "none" and not cls and pool == "sum":
                    assert bool((got == 0.0).all())                  # every entry is an exact 0
                assert torch.equal(_run(case, pool), got)           # bitwise repeatable
    print(f"maxsim_expert P={P} pool={pool}: worst error {worst:.3g} of the gate over {i} cases")


@pytest.mark.parametrize("pool", ["sum", "max"])
def test_one_expert_with_mask_weights_equals_maxsim_bitwise(pool):
    from dpr_scale_b200 import ops
    for B, LQ, LD, P in ((1, 1, 1, 64), (7, 31, 129, 128), (300, 130, 511, 136), (40, 65, 255, 1024)):
        gen = torch.Generator().manual_seed(B + LQ + LD)
        nq = max(1, (B + 1) // 2)
        q = torch.randn(nq, LQ + 1, P, generator=gen).to(torch.bfloat16).cuda()
        d = -torch.rand(B, LD + 1, P, generator=gen).to(torch.bfloat16).cuda() if B == 7 else \
            torch.randn(B, LD + 1, P, generator=gen).to(torch.bfloat16).cuda()
        qm = (torch.rand(nq, LQ + 1, generator=gen) > 0.3).int().cuda()
        dm = (torch.rand(B, LD + 1, generator=gen) > 0.3).int().cuda()
        idx = torch.randint(0, nq, (B,), generator=gen, dtype=torch.int32)
        want = ops.maxsim(q, d, qm, dm, idx, pool)
        ones_q = torch.full((nq, LQ + 1, 1), 7, dtype=torch.int32, device="cuda")
        ones_d = torch.full((B, LD + 1, 1), 7, dtype=torch.int32, device="cuda")
        got = ops.maxsim_expert(q, d, ones_q, qm.float().unsqueeze(-1), ones_d, dm.float().unsqueeze(-1), idx, pool)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (B, LQ, LD, P)


def test_every_score_written_and_nothing_else():
    from dpr_scale_b200 import _lib
    q, d, qi, qw, di, dw, idx, qc, dc = _case(300, 65, 129, 136, 2, 3, "dense", seed=5, cls=True, Pc=64)
    G = 64
    buf = torch.full((300 + 2 * G,), float("nan"), device="cuda")
    idx_d = idx.cuda()
    rc = _lib.load().dprb_maxsim_expert_fwd(q.data_ptr(), d.data_ptr(), qi.data_ptr(), qw.data_ptr(), di.data_ptr(),
                                            dw.data_ptr(), qc.data_ptr(), dc.data_ptr(), idx_d.data_ptr(), q.shape[0],
                                            q.shape[1], 300, d.shape[1], 136, 2, 3, 64, 0, buf.data_ptr() + 4 * G,
                                            torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:G]).all()) and bool(torch.isnan(buf[-G:]).all())
    assert not bool(torch.isnan(buf[G:-G]).any())


def test_more_than_65535_pairs():
    B = 70_001
    case = _case(B, 5, 9, 64, 2, 2, "dense", seed=9, cls=True, Pc=32)
    got = _run(case, "sum")
    ref, gate = _reference(case, "sum")
    err = (got.double() - ref).abs() / gate
    print(f"maxsim_expert B={B}: worst error {float(err.max()):.3g} of the gate")
    assert got.shape == (B,) and bool((err <= 1.0).all())


def test_bad_shapes_are_rejected_before_any_launch():
    from dpr_scale_b200 import _lib, ops
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    buf = torch.zeros(1 << 20, dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    w = torch.zeros(1 << 16, device="cuda")
    out = torch.zeros(4, device="cuda")
    idx = torch.zeros(4, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    good = dict(SQ=8, SD=8, P=64, KQ=1, KD=1, Pc=64, pool=0, cls=True)
    bad = [dict(P=100), dict(P=1032), dict(SQ=1), dict(SD=1), dict(SQ=513), dict(SD=513), dict(KQ=0), dict(KQ=9),
           dict(KD=0), dict(KD=9), dict(Pc=60), dict(Pc=1032), dict(Pc=0), dict(pool=2)]
    assert lib.dprb_maxsim_expert_fwd(p, p, ids.data_ptr(), w.data_ptr(), ids.data_ptr(), w.data_ptr(), p, None,
                                      idx.data_ptr(), 2, 8, 4, 8, 64, 1, 1, 64, 0, out.data_ptr(), st) == 1
    for change in bad:
        a = dict(good, **change)
        assert lib.dprb_maxsim_expert_fwd(p, p, ids.data_ptr(), w.data_ptr(), ids.data_ptr(), w.data_ptr(), p, p,
                                          idx.data_ptr(), 2, a["SQ"], 4, a["SD"], a["P"], a["KQ"], a["KD"], a["Pc"],
                                          a["pool"], out.data_ptr(), st) == 1, change
    qv, dv = buf[:2 * 8 * 64].view(2, 8, 64), buf[:4 * 8 * 64].view(4, 8, 64)
    qi, di = ids[:2 * 8].view(2, 8, 1), ids[:4 * 8].view(4, 8, 1)
    qw, dw = w[:2 * 8].view(2, 8, 1), w[:4 * 8].view(4, 8, 1)
    with pytest.raises(ValueError):                                  # query index out of range
        ops.maxsim_expert(qv, dv, qi, qw, di, dw, torch.tensor([0, 1, 2, 0]))
    with pytest.raises(ValueError):                                  # nine experts
        ops.maxsim_expert(qv, dv, ids[:2 * 8 * 9].view(2, 8, 9), w[:2 * 8 * 9].view(2, 8, 9), di, dw,
                          torch.tensor([0, 1, 1, 0]))
    with pytest.raises(ValueError):                                  # one CLS operand
        ops.maxsim_expert(qv, dv, qi, qw, di, dw, torch.tensor([0, 1, 1, 0]), "sum", buf[:2 * 64].view(2, 64), None)
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ router
def _bert_base(model):
    from tests import multivec_cases
    sd, cfg = multivec_cases.bert_base_state_dict(model)
    from dpr_scale_b200.models.citadel_models.citadel_model import CITADELEncoder
    from dpr_scale_b200.models.citadel_models.coil_model import COILEncoder
    cls = COILEncoder if model == "coil" else CITADELEncoder
    m = cls.from_config(cfg, *multivec_cases.BASE[model])
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def test_router_against_float64_logits():
    """The chosen experts against float64 logits of the same fp16 router tokens.  The operand rounding (the fp16 decoder
    rows and bias: 2^-11 relative) and the fp32 accumulation over H + 1 terms bound each logit's error by
    delta_t = (2^-11 + (H + 1) 2^-24) max_v (sum_k |x_tk W_vk| + |b_v|); so every chosen expert's float64 logit is within
    2 delta_t of the float64 rank-r best, the ids equal float64's wherever consecutive float64 logits of the top k + 1
    are more than 2 delta_t apart, and the weights are log1p(relu(.)) of the chosen float64 logit within delta_t."""
    from dpr_scale_b200.models.citadel_models.colbert_model import encode_tokens
    from tests import multivec_cases
    m, _ = _bert_base("citadel")
    _, d = multivec_cases.bert_base_tokens()
    d = {k: v[:4] for k, v in d.items()}
    k = 2
    with torch.no_grad():
        hidden, am, N, S = encode_tokens(m._body, d)
        x = m.router_tokens(hidden)
        logit, ids = m.route(hidden, k)
        H = m.config["hidden_size"]
        W, b = m.word_embeddings().detach().double(), m.router_bias().detach().double()
        xd = x[:, :H].double()
        assert bool((x[:, H] == 1).all()) and bool((x[:, H + 1:] == 0).all())
        L = xd @ W.T + b
        A = (xd.abs() @ W.abs().T + b.abs()).max(1).values
    live = am.view(-1) != 0
    out = {}
    for name, eps in (("fp16", 2.0 ** -11), ("bf16", 2.0 ** -8)):
        delta = (eps + (H + 1) * 2.0 ** -24) * A
        top = L.topk(k + 1, dim=1).values
        gap = (top[:, :-1] - top[:, 1:]).min(1).values
        out[name] = (delta, gap, float(((gap <= 2 * delta) & live).sum()) / float(live.sum()))
    delta, gap, frac = out["fp16"]
    chosen = L.gather(1, ids)
    assert bool((chosen >= top[:, :k] - 2 * delta[:, None]).all())
    assert bool((logit.double() - chosen).abs().le(delta[:, None] + 1e-6).all())
    clear = gap > 2 * delta
    assert torch.equal(ids[clear], L.topk(k, dim=1).indices[clear])
    with torch.no_grad():
        _, _, w, _ = m.expert_reps(d, topk=k)
    want = torch.log1p(torch.relu(chosen)).view(N, S, k) * am.unsqueeze(-1)
    assert float((w.double() - want).abs().max()) <= float(delta.max()) + 1e-6
    print(f"router at BERT-base dims: delta median {float(delta.median()):.3g}; tokens within 2 delta of a top-{k} tie: "
          f"{100 * frac:.2f}% with fp16 operands, {100 * out['bf16'][2]:.2f}% with bf16 operands")


# ------------------------------------------------------------------ encoders and the task
def _oracle_cfg(kind):
    from tests import rerank_cases
    return rerank_cases.ORACLE_CFG[kind]


def _oracle_on_kernel_ids(sd, kind, toks, ids, prefix=""):
    """The float64 oracle with the kernel's expert ids: weights = log1p(relu(float64 logit of each chosen id))."""
    from oracle import multivec as om
    r = om.citadel(sd, _oracle_cfg(kind), toks, 1, True, prefix)
    am = torch.as_tensor(toks["attention_mask"])[:, 1:].unsqueeze(-1).double()
    ids = ids[:, 1:].long().cpu()
    r["expert_ids"] = ids
    r["expert_weights"] = torch.log1p(torch.relu(r["logits"].gather(2, ids))) * am
    return r


@pytest.mark.parametrize("name", ["coil_bert", "coil_roberta", "citadel_bert", "citadel_roberta"])
@pytest.mark.parametrize("S", [24, 257])
def test_tiny_encoders_match_oracle(name, S):
    from oracle import multivec as om
    from tests import colbert_cases, multivec_cases
    model, kind, _, _, _ = multivec_cases.TINY[name]
    sd = multivec_cases.tiny_state_dict(name)
    m = multivec_cases.build(name, sd).cuda()
    cfg = colbert_cases.encoder_config(kind)
    toks = colbert_cases.seq_tokens(torch.Generator().manual_seed(S), 5, S, cfg["vocab_size"], cfg["pad_token_id"])
    for topk in ((1, 3) if model == "citadel" else (1,)):
        with torch.no_grad():
            r = {k: v.cpu() for k, v in m(toks, topk=topk, add_cls=True).items()}
        if model == "coil":
            ref = om.coil(sd, _oracle_cfg(kind), toks, True)
            assert torch.equal(r["expert_ids"], toks["input_ids"][:, 1:])
            assert torch.equal(r["expert_weights"], toks["attention_mask"][:, 1:])
        else:
            ref = om.citadel(sd, _oracle_cfg(kind), toks, topk, True)
            am = toks["attention_mask"][:, 1:].unsqueeze(-1).double()
            chosen = ref["logits"].gather(2, r["expert_ids"])
            want_w = torch.log1p(torch.relu(chosen)) * am
            amp = float(ref["logits"].abs().max())
            assert float((r["expert_weights"].double() - want_w).abs().max()) <= 2.0 ** -7 * amp
            top = (ref["logits"].topk(topk, dim=2).values * am)
            assert bool((chosen * am >= top - 2.0 ** -7 * amp).all())             # never far from the true top-k
        for key in ("expert_repr", "cls_repr"):
            err = float((r[key].double() - ref[key]).abs().max())
            gate = 2.0 ** -7 * float(ref[key].abs().max())
            print(f"{name} S={S} k={topk} {key}: max|err| {err:.3g} = {err / gate:.3g} of the gate")
            assert r[key].dtype == torch.float32 and r[key].shape == ref[key].shape and err <= gate


def _task(tmp_path, name, pool):
    from dpr_scale_b200.task.citadel_eval_task import RerankMultiVecRetrieverTask
    from tests import multivec_cases
    model, kind, proj, cls_proj, _ = multivec_cases.TINY[name]
    ckpt = str(tmp_path / f"{name}.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(name)}, ckpt)
    mdir = multivec_cases.model_dir(str(tmp_path / f"{name}_model"), name)
    qk, ck = multivec_cases.TASK_TOPK
    task = RerankMultiVecRetrieverTask(
        checkpoint_path=ckpt, output_dir=str(tmp_path / "out"), query_pool=pool, add_cls=True, query_topk=qk,
        context_topk=ck, transform={}, datamodule=None, optim={}, shared_model=False,
        model=dict({"_target_": "dpr_scale_b200.models.citadel_models." + multivec_cases.TARGETS[model],
                    "model_path": mdir}, **multivec_cases.ctor_kwargs(model, proj, cls_proj)))
    return ckpt, mdir, task


def _cli_args(mdir, ckpt, out_dir, pool, name):
    from tests import multivec_cases, rerank_cases
    model, _, proj, cls_proj, _ = multivec_cases.TINY[name]
    kw = rerank_cases.datamodule_kwargs()
    qk, ck = multivec_cases.TASK_TOPK
    dims = [f"task.model.{k}={'null' if v is None else v}" for k, v in
            multivec_cases.ctor_kwargs(model, proj, cls_proj).items()]
    return ["task=multivec_rerank", f"task/model={model}_model", "datamodule=multivec_rerank",
            f"task.model.model_path={mdir}", *dims, f"task.transform.max_seq_len={rerank_cases.MAX_LEN}",
            f"datamodule.test_path={kw['test_path']}", f"datamodule.test_question_path={kw['test_question_path']}",
            f"datamodule.test_passage_path={kw['test_passage_path']}",
            f"datamodule.test_batch_size={kw['test_batch_size']}", "datamodule.use_title=true",
            f"+task.query_pool={pool}", "+task.add_cls=true", f"+task.query_topk={qk}", f"+task.context_topk={ck}",
            f"+task.checkpoint_path={ckpt}", f"+task.output_dir={out_dir}"]


@pytest.mark.parametrize("name", ["coil_bert", "coil_roberta", "citadel_bert", "citadel_roberta"])
@pytest.mark.parametrize("pool", ["sum", "max"])
def test_rerank_task_and_cli(tmp_path, name, pool):
    """Each batch's scores against the float64 oracle scored on the kernel's expert ids.  Gate: 2^-7 of the largest
    per-pair bound (the score of |q|, |d|, |w| with sum pooling, plus sum |q_cls d_cls|): CITADEL scores are sums of
    terms of both signs, so max|score| can be far below the size of the terms whose bf16 rounding it inherits.  The
    CLI's pickles: the reference's qids / ctx ids, scores bitwise those of the batches, and for COIL (no routing) within
    the same gate of the reference's scores; rerank.trec in descending score order."""
    import pickle
    import os
    from dpr_scale_b200 import rerank
    from oracle import multivec as om
    from tests import multivec_cases
    from tests.test_colbert_cpu import golden_batches
    model, kind, _, _, _ = multivec_cases.TINY[name]
    raw = np.load(os.path.join(GOLDEN, "multivec_small.npz"))
    ckpt, mdir, task = _task(tmp_path, name, pool)
    task.setup("test")
    task.cuda()
    full = multivec_cases.task_state_dict(name)
    qk, ck = multivec_cases.TASK_TOPK
    ours, ref, bound = [], [], []
    for b in golden_batches():
        bc = dict(b, query_ids={k: v.cuda() for k, v in b["query_ids"].items()},
                  contexts_ids={k: v.cuda() for k, v in b["contexts_ids"].items()})
        ours.append(task._scores(bc).cpu())
        if model == "coil":
            q = om.coil(full, _oracle_cfg(kind), b["query_ids"], True, "query_encoder.")
            d = om.coil(full, _oracle_cfg(kind), b["contexts_ids"], True, "context_encoder.")
        else:
            with torch.no_grad():
                _, qi, _, _ = task.query_encoder.expert_reps(bc["query_ids"], topk=qk)
                _, di, _, _ = task.context_encoder.expert_reps(bc["contexts_ids"], topk=ck)
            q = _oracle_on_kernel_ids(full, kind, b["query_ids"], qi, "query_encoder.")
            d = _oracle_on_kernel_ids(full, kind, b["contexts_ids"], di, "context_encoder.")
        ref.append(om.expert_score(q["expert_repr"], d["expert_repr"], q["expert_ids"], q["expert_weights"],
                                   d["expert_ids"], d["expert_weights"], pool, q["cls_repr"], d["cls_repr"]))
        bound.append(om.expert_score(q["expert_repr"].abs(), d["expert_repr"].abs(), q["expert_ids"],
                                     q["expert_weights"].abs(), d["expert_ids"], d["expert_weights"].abs(), "sum") +
                     (q["cls_repr"] * d["cls_repr"]).abs().sum(1))
    ours, ref, bound = torch.cat(ours), torch.cat(ref), torch.cat(bound)
    gate = 2.0 ** -7 * float(bound.max())
    err = float((ours.double() - ref).abs().max())
    print(f"{name} {pool}: max|dscore| vs float64 on the kernel's ids {err:.3g} = {err / gate:.3g} of the gate")
    assert err <= gate

    out_dir = str(tmp_path / "cli_out")
    run = rerank.main(_cli_args(mdir, ckpt, out_dir, pool, name))
    got = {}
    for what in ("scores", "qids", "ctx_ids"):
        with open(os.path.join(out_dir, f"{what}_0000.pkl"), "rb") as f:
            got[what] = pickle.load(f)
    assert got["qids"] == raw[f"{name}/{pool}/pkl/qids"].tolist()
    assert got["ctx_ids"] == raw[f"{name}/{pool}/pkl/ctx_ids"].tolist()
    s = got["scores"]
    assert torch.is_tensor(s) and s.dtype == torch.float32 and torch.equal(s, ours)
    want = torch.from_numpy(raw[f"{name}/{pool}/pkl/scores"])
    dev = float((s - want).abs().max())
    print(f"{name} {pool}: max|dscore| vs the reference's pickle {dev:.3g} (max|score| {float(want.abs().max()):.3g})")
    if model == "coil":
        assert dev <= gate
    lines = [ln.split() for ln in open(run).read().splitlines()]
    assert len(lines) == len(got["qids"])
    score_of = {(q, c): v for q, c, v in zip(got["qids"], got["ctx_ids"], s.tolist())}
    for q in dict.fromkeys(ln[0] for ln in lines):
        vals = [score_of[(q, ln[2])] for ln in lines if ln[0] == q]
        assert vals == sorted(vals, reverse=True)


@pytest.mark.parametrize("model", ["coil", "citadel"])
@pytest.mark.parametrize("pool", ["sum", "max"])
def test_bert_base_matches_reference_golden(model, pool):
    """Within twice the reference's own bf16-autocast deviation.  For CITADEL the pairs with no near-tied token (fp32
    top-1 gap at most twice the bf16 run's largest logit deviation) are reported."""
    import os
    from dpr_scale_b200 import ops
    from tests import colbert_cases, multivec_cases
    raw = np.load(os.path.join(GOLDEN, "multivec_bert_base.npz"))
    g = {k: torch.from_numpy(raw[k]) for k in raw.files}
    m, sd = _bert_base(model)
    assert torch.equal(colbert_cases.sd_checksum(sd), g[f"{model}/checksum"]), "seeded weights differ from the golden's"
    q = {k.split("/")[-1]: g[k] for k in g if k.startswith("query/")}
    d = {k.split("/")[-1]: g[k] for k in g if k.startswith("passage/")}
    with torch.no_grad():
        qr, qi, qw, qc = m.expert_reps(q, topk=1, add_cls=True)
        dr, di, dw, dc = m.expert_reps(d, topk=1, add_cls=True)
        s = ops.maxsim_expert(qr, dr, qi, qw, di, dw, torch.arange(multivec_cases.BASE_PAIRS, dtype=torch.int32), pool,
                              qc, dc).cpu()
    want = g[f"{model}/{pool}/scores"]
    amp = float(g[f"{model}/{pool}/amp_max_abs"])
    diff = (s - want).abs()
    msg = ""
    if model == "citadel":
        thr = 2.0 * float(g["citadel/amp_logit_max_abs"])
        near = torch.zeros(multivec_cases.BASE_PAIRS, dtype=torch.bool)
        for side in ("query", "passage"):
            live = g[f"{side}/attention_mask"][:, 1:] != 0
            near |= ((g[f"citadel/{side}/gap"] <= thr) & live).any(1)
        kept = ~near
        msg = f", {int(near.sum())} of {len(near)} pairs have a near-tied token (gap <= {thr:.3g})"
        if bool(kept.any()):
            msg += f", max|dscore| on the others {float(diff[kept].max()):.3g}"
    print(f"bert-base {model} {pool}: max|dscore| {float(diff.max()):.3g}, reference bf16 autocast {amp:.3g}, "
          f"max|score| {float(want.abs().max()):.4g}{msg}")
    assert float(diff.max()) <= 2.0 * amp
