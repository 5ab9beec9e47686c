"""COIL / CITADEL expert-index generation on the H100:

  * dprb_expert_group against a NumPy statement of the contract (keep rule, stable sort by expert or (sequence,
    expert)) over N in {1, 3, 128}, S up to 512, K 1..8, P in {8, 32, 128, 1024}, V up to 50 265, a dominant expert,
    batches where every entry is dropped and context-id mode: keys, order and weights exact, payloads bitwise equal to
    the fp32 product of the same inputs, two runs bitwise equal;
  * the tasks end to end on tiny encoders: every file equals the float64 oracle (oracle/multivec_index.py) run on the
    encoders' own ids and weights, and the payloads of COIL (ids = input ids) and of CITADEL entries routed as the
    reference routed them are within the bf16-rep bound of the reference's files;
  * the CLIs on the fixture corpus, whose files load with plain pickle + torch;
  * a 2-rank run (two GPUs only).
"""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import multivec_cases, multivec_index_cases as cases, rerank_cases
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(GOLDEN, "multivec_index_small.npz"))


def _inputs(N, S, K, P, V, seed, dominant=False, threshold=0.3):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (N, S, K), generator=g, dtype=torch.int32)
    if dominant:                                    # one expert holds most entries
        ids[torch.rand(N, S, K, generator=g) < 0.7] = V // 2
    w = torch.rand(N, S, K, generator=g)
    w[torch.rand(N, S, K, generator=g) < 0.2] = 0.0
    lens = torch.randint(1, S + 1, (N,), generator=g)
    mask = (torch.arange(S)[None] < lens[:, None]).int()
    reps = torch.randn(N, S, max(P, 8), generator=g).bfloat16()
    tokens = torch.randint(0, V, (N, S), generator=g)
    return ids, w, mask, reps, tokens


def _expected(ids, w, mask, threshold, per_seq, ctx):
    N, S, K = ids.shape
    n, s, k = np.meshgrid(np.arange(N), np.arange(S), np.arange(K), indexing="ij")
    keep = (s >= 1) & (mask.numpy()[n, s] != 0)
    if not ctx:
        keep &= w.numpy() > threshold
    n, s, k, x = n[keep], s[keep], k[keep], ids.numpy()[keep]
    order = np.lexsort((x, n)) if per_seq else np.argsort(x, kind="stable")     # entries enter in (n, s, k) order
    return x[order], n[order], s[order], k[order]


CASES = [  # (N, S, K, P, V, per_sequence, context_id, dominant)
    (1, 2, 1, 8, 1, False, False, False), (3, 17, 3, 32, 50265, False, False, False),
    (3, 64, 8, 1024, 30522, True, False, False), (128, 256, 2, 32, 30522, False, False, False),
    (128, 256, 2, 32, 30522, True, False, True), (128, 512, 1, 128, 50265, False, False, False),
    (16, 512, 8, 8, 50265, True, False, False), (128, 64, 4, 0, 30522, False, True, False),
    (7, 33, 5, 128, 300, True, False, False), (3, 40, 2, 32, 30522, True, False, True),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N{}_S{}_K{}_P{}_V{}_{}{}{}".format(
    *c[:5], "q" if c[5] else "p", "_ctx" if c[6] else "", "_dom" if c[7] else ""))
def test_expert_group_matches_contract(case):
    from dpr_scale_b200 import ops
    N, S, K, P, V, per_seq, ctx, dom = case
    ids, w, mask, reps, tokens = _inputs(N, S, K, P, V, seed=N * 1000 + S + K, dominant=dom)
    thr = 0.3
    d = {k: v.cuda() for k, v in dict(ids=ids, w=w, mask=mask, reps=reps[..., :P] if P else reps,
                                      tokens=tokens).items()}
    reps_arg = None if ctx else d["reps"].contiguous()
    with torch.no_grad():
        runs = [ops.expert_group(reps_arg, d["ids"], d["w"], d["mask"], V, thr, d["tokens"] if ctx else None, per_seq)
                for _ in range(2)]
    torch.cuda.synchronize()
    x, n, s, k = _expected(ids, w, mask, thr, per_seq, ctx)
    expert, seq, tok, weight, payload = (t.cpu() for t in runs[0])
    print(f"{case}: {len(x)} kept of {N * (S - 1) * K}")
    assert np.array_equal(expert.numpy(), x) and np.array_equal(seq.numpy(), n) and np.array_equal(tok.numpy(), s)
    assert torch.equal(weight, w[n, s, k])
    if ctx:
        assert torch.equal(payload, tokens[n, s].float())
    else:
        rows = d["reps"][torch.from_numpy(n).cuda(), torch.from_numpy(s).cuda()].float()
        want = d["w"][torch.from_numpy(n).cuda(), torch.from_numpy(s).cuda(), torch.from_numpy(k).cuda()]
        assert torch.equal(payload.cuda(), want[:, None] * rows)                  # fp32 product, bit for bit
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)


def test_every_entry_dropped():
    from dpr_scale_b200 import ops
    ids, w, mask, reps, _ = _inputs(5, 40, 2, 32, 1000, seed=3)
    with torch.no_grad():
        out = ops.expert_group(reps.cuda(), ids.cuda(), w.cuda(), mask.cuda(), 1000, threshold=2.0)
        assert all(t.shape[0] == 0 for t in out)
        out = ops.expert_group(reps.cuda(), ids.cuda(), w.cuda(), torch.zeros_like(mask).cuda(), 1000,
                               tokens=torch.zeros(5, 40, dtype=torch.int32).cuda())
        assert all(t.shape[0] == 0 for t in out)


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def _run_task(tmp_path, case, query):
    from dpr_scale_b200.task.citadel_eval_task import (GenerateMultiVecEmbeddingsTask,
                                                       GenerateMultiVecQueryEmbeddingsTask)
    if query:
        enc, topk, add_cls = cases.QUERY[case]
        ctx_id, thr = False, 0.0
    else:
        enc, topk, add_cls, ctx_id, thr = cases.PASSAGE[case]
    model = multivec_cases.TINY[enc][0]
    mdir = multivec_cases.model_dir(str(tmp_path / "model"), enc)
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)
    kw = cases.task_kwargs(enc, mdir, topk, add_cls)
    kw["model"]["_target_"] = "dpr_scale_b200.models.citadel_models." + multivec_cases.TARGETS[model]
    out = str(tmp_path / "out")
    cls = GenerateMultiVecQueryEmbeddingsTask if query else GenerateMultiVecEmbeddingsTask
    task = cls(ctx_embeddings_dir=out, checkpoint_path=ckpt, add_context_id=ctx_id, weight_threshold=thr, **kw)
    task.setup("test")
    task.cuda()
    outs, mine = [], []
    with torch.no_grad():
        for i, (toks, ids) in enumerate(cases.batches(enc, seed=6 if query else 5)):
            toks = {k: v.cuda() for k, v in toks.items()}
            encoder = task.query_encoder if query else task.context_encoder
            r = encoder(toks, topk=topk, add_cls=add_cls)
            mine.append(({k: v.cpu().numpy() for k, v in r.items()}, toks["input_ids"].cpu().numpy(), ids))
            batch = {"query_ids": toks, "topic_ids": ids} if query else {"contexts_ids": toks, "corpus_ids": ids}
            outs.append(task.test_step(batch, i))
        task.test_epoch_end(outs)
    return out, mine


def _rep_gate(want):
    return 2.0 ** -7 * max(1e-30, float(np.abs(want).max()))


@pytest.mark.parametrize("case", list(cases.PASSAGE))
def test_passage_task_matches_oracle_and_reference(tmp_path, case):
    from oracle import multivec_index as om
    enc, _, add_cls, ctx_id, thr = cases.PASSAGE[case]
    out, mine = _run_task(tmp_path, case, False)
    want = om.passage_index(mine, ctx_id, thr)
    edir = os.path.join(out, "expert_0000")
    assert sorted(int(f[:-4]) for f in os.listdir(edir)) == sorted(want)
    for x, (ids, w, reps) in want.items():
        got = _load(os.path.join(edir, f"{x}.pkl"))
        assert isinstance(got, tuple) and len(got) == 3
        assert got[0].dtype == torch.int64 and got[1].dtype == got[2].dtype == torch.float32
        assert np.array_equal(got[0].numpy(), ids) and np.array_equal(got[1].numpy(), w.astype(np.float32))
        assert np.array_equal(got[2].numpy(), reps.astype(np.float32))
    # against the reference's files: experts the reference routed the same way
    same = 0
    for x in G[f"p/{case}/experts"].tolist():
        if x not in want or not np.array_equal(want[x][0], G[f"p/{case}/x{x}/ids"]):
            assert not enc.startswith("coil"), f"COIL expert {x} differs from the reference's"
            continue
        ref_w, ref_r = G[f"p/{case}/x{x}/weights"], G[f"p/{case}/x{x}/reprs"]
        assert np.abs(want[x][1] - ref_w).max() <= _rep_gate(ref_w) + 1e-6
        assert np.abs(want[x][2] - ref_r).max() <= _rep_gate(ref_r)
        same += 1
    print(f"{case}: {same} of {len(G[f'p/{case}/experts'])} reference experts hold the same entries")
    assert same >= len(G[f"p/{case}/experts"]) // 2
    if add_cls:
        cls = _load(os.path.join(out, "cls_0000.pkl"))
        assert cls.dtype == torch.float32 and cls.shape == G[f"p/{case}/cls"].shape
        assert np.abs(cls.numpy() - G[f"p/{case}/cls"]).max() <= _rep_gate(G[f"p/{case}/cls"])
    else:
        assert not os.path.exists(os.path.join(out, "cls_0000.pkl"))


@pytest.mark.parametrize("case", list(cases.QUERY))
def test_query_task_matches_oracle(tmp_path, case):
    from oracle import multivec_index as om
    enc, _, add_cls = cases.QUERY[case]
    out, mine = _run_task(tmp_path, case, True)
    emb, wts = [], []
    for r, _, _ in mine:
        e, w = om.query_index(r)
        emb.extend(e)
        wts.extend(w)
    assert _load(os.path.join(out, "query_id.pkl")) == [t for _, _, ids in mine for t in ids]
    got_e, got_w = _load(os.path.join(out, "query_repr.pkl")), _load(os.path.join(out, "query_weight.pkl"))
    assert len(got_e) == len(got_w) == len(emb)
    for j in range(len(emb)):
        assert sorted(got_e[j]) == sorted(emb[j]) == sorted(got_w[j])
        for x in emb[j]:
            assert all(t.dtype == torch.float32 and t.shape == (len(emb[j][x][0]),) for t in got_e[j][x])
            assert all(t.dtype == torch.float32 and t.dim() == 0 for t in got_w[j][x])
            assert np.array_equal(torch.stack(got_e[j][x]).numpy(), np.stack(emb[j][x]).astype(np.float32))
            assert np.array_equal(torch.stack(got_w[j][x]).numpy(), np.array(wts[j][x]).astype(np.float32))
    if enc.startswith("coil"):                      # no routing: the reference's dicts, within the bf16-rep bound
        for j in range(len(emb)):
            assert list(G[f"q/{case}/{j}/experts"]) == list(emb[j]) or sorted(G[f"q/{case}/{j}/experts"]) == \
                sorted(emb[j])
            for x in emb[j]:
                ref = G[f"q/{case}/{j}/x{x}/repr"]
                assert np.abs(np.stack(emb[j][x]) - ref).max() <= _rep_gate(ref)
    assert os.path.exists(os.path.join(out, "query_cls.pkl")) == add_cls


def _cli_args(mdir, ckpt, out, enc, query):
    model, _, proj, cls_proj, _ = multivec_cases.TINY[enc]
    dims = [f"task.model.{k}={'null' if v is None else v}" for k, v in
            multivec_cases.ctor_kwargs(model, proj, cls_proj).items()]
    data = rerank_cases.DATA
    common = [f"task/model={model}_model", f"task.model.model_path={mdir}", *dims,
              f"task.transform.max_seq_len={rerank_cases.MAX_LEN}", "datamodule.test_batch_size=4",
              f"+task.checkpoint_path={ckpt}", f"+task.ctx_embeddings_dir={out}", "+task.add_cls=true",
              "+task.query_topk=2", "+task.context_topk=2"]
    if query:
        return ["task=generate_multivec_query_embeddings", "datamodule=generate_multivec_query_emb",
                f"datamodule.test_path={os.path.join(data, 'questions.tsv')}", "datamodule.trec_format=true"] + common
    return ["task=generate_multivec_embeddings", "datamodule=generate",
            f"datamodule.test_path={os.path.join(data, 'passages.tsv')}"] + common


def test_cli_on_fixture_corpus(tmp_path):
    from dpr_scale_b200 import generate_multivec_embeddings, generate_multivec_query_embeddings
    enc = "citadel_bert"
    mdir = multivec_cases.model_dir(str(tmp_path / "model"), enc)
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)
    out = str(tmp_path / "index")
    generate_multivec_embeddings.main(_cli_args(mdir, ckpt, out, enc, False))
    generate_multivec_query_embeddings.main(_cli_args(mdir, ckpt, out, enc, True))
    code = ("import os, pickle, sys, torch\n"
            f"d = {out!r}\n"
            "n = 0\n"
            "for f in os.listdir(os.path.join(d, 'expert_0000')):\n"
            "    ids, w, r = pickle.load(open(os.path.join(d, 'expert_0000', f), 'rb'))\n"
            "    assert ids.dtype == torch.int64 and w.shape == ids.shape and r.shape[0] == ids.shape[0]\n"
            "    n += len(ids)\n"
            "cls = pickle.load(open(os.path.join(d, 'cls_0000.pkl'), 'rb'))\n"
            "q = pickle.load(open(os.path.join(d, 'query_id.pkl'), 'rb'))\n"
            "e = pickle.load(open(os.path.join(d, 'query_repr.pkl'), 'rb'))\n"
            "w = pickle.load(open(os.path.join(d, 'query_weight.pkl'), 'rb'))\n"
            "qc = pickle.load(open(os.path.join(d, 'query_cls.pkl'), 'rb'))\n"
            "assert len(q) == len(e) == len(w) == qc.shape[0] == 7 and cls.shape[0] == 11 and n > 0\n"
            "assert not any(m.startswith('dpr_scale_b200') for m in sys.modules)\n"
            "print('entries', n, 'queries', len(q))\n")
    env = {k: v for k, v in os.environ.items() if k != "PYTHONPATH"}
    res = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=env, capture_output=True, text=True,
                         timeout=300)
    print(res.stdout, res.stderr[-2000:])
    assert res.returncode == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_shards_hold_the_one_rank_entries(tmp_path):
    enc = "citadel_bert"
    mdir = multivec_cases.model_dir(str(tmp_path / "model"), enc)
    ckpt = str(tmp_path / "task.ckpt")
    torch.save({"state_dict": multivec_cases.task_state_dict(enc)}, ckpt)
    one, two = str(tmp_path / "one"), str(tmp_path / "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    for nproc, out in ((1, one), (2, two)):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={nproc}", "-m",
               "dpr_scale_b200.generate_multivec_embeddings"] + _cli_args(mdir, ckpt, out, enc, False)
        subprocess.run(cmd, check=True, cwd=ROOT, env=env, timeout=600)

    def entries(d, ranks):
        acc = {}
        for r in ranks:
            ed = os.path.join(d, f"expert_{r:04}")
            assert os.path.isdir(ed)
            for f in sorted(os.listdir(ed)):
                ids, w, reps = _load(os.path.join(ed, f))
                acc.setdefault(int(f[:-4]), []).extend(zip(ids.tolist(), w.tolist()))
        return {x: sorted(v) for x, v in acc.items()}

    assert entries(one, [0]) == entries(two, [0, 1])
    cls = torch.cat([_load(os.path.join(two, f"cls_{r:04}.pkl")) for r in (0, 1)])
    assert cls.shape == _load(os.path.join(one, "cls_0000.pkl")).shape
