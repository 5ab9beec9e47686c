"""Cross-encoder training on the GPU:

  * dprb_seqcls_group_ce against float64 (loss, logits, dpre, dweight, dbias) for B in {1, 37} groups, H in {128, 768,
    1024}, G in {2, 8, 64 = the maximum}, with and without the head's dropout (masks replayed through
    dprb_dropout_mask); two runs are bitwise equal; bad shapes are rejected before any launch;
  * tiny BERT and RoBERTa cross-encoders: the group_ce loss and every parameter gradient against the float64 oracle
    (oracle/cross_encoder_train.py) fed the masks the CUDA path drew, dropout off and at p = 0.1, S in {24, 300, 512}:
    logits rel-L2 <= 2e-2, loss within 1 %, every parameter gradient cosine >= 0.997 and rel-L2 <= 7e-2.  Over two runs
    the worst tensors sat at cosine 0.9988 / rel-L2 0.050 without dropout (embedding-side tensors, bf16 operands through
    the whole body; the body's atomics make the numbers vary run to run) and 0.9999 / 0.016 with it;
  * a few fused AdamW steps reduce the loss on a fixed batch;
  * python -m dpr_scale_b200.main on the fixture JSONL writes a checkpoint that python -m dpr_scale_b200.rerank loads
    strictly and scores with.
"""
import glob
import os
import pickle
import subprocess
import sys

import pytest
import torch

from tests import rerank_cases
from tests.test_dropout_gpu import P, _masks
from tests.util import cosine, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "tests", "golden", "data")


# ------------------------------------------------------------------ the kernel
def _kernel_inputs(B, G, H, seed):
    g = torch.Generator().manual_seed(seed)
    pre = 2.0 * torch.randn(B * G, H, generator=g)
    W = 0.05 * torch.randn(1, H, generator=g)
    b = torch.randn(1, generator=g)
    labels = torch.randint(0, G, (B,), generator=g)
    return pre, W, b, labels


@pytest.mark.parametrize("B", [1, 37])
@pytest.mark.parametrize("H", [128, 768, 1024])
@pytest.mark.parametrize("G", [2, 8, 64])
@pytest.mark.parametrize("p", [0.0, P])
def test_group_ce_kernel_matches_float64(B, H, G, p):
    from dpr_scale_b200 import ops
    assert G <= ops.SEQCLS_GROUP_MAX
    pre, W, b, labels = _kernel_inputs(B, G, H, B * 1000 + H + G)
    seed = 1234 + G
    loss, logits, dpre, dW, db = ops.seqcls_group_ce(pre.cuda(), W.cuda(), b.cuda(), labels.cuda(), G, p, seed)
    N = B * G
    mult = ops.dropout_mask(N, H, p, seed, 0, ops.DROP_SITE_HEAD).double().cpu()
    if p > 0:
        mult = mult / (1.0 - round(p * 65536) / 65536.0)
        assert abs(float((mult > 0).double().mean()) - (1 - p)) < 0.02
    x = pre.double().requires_grad_(True)
    Wd, bd = W.double().requires_grad_(True), b.double().requires_grad_(True)
    t = torch.tanh(x) * mult
    ref_logits = (t @ Wd.T + bd).view(-1)
    ref_logits.retain_grad()
    ref_loss = torch.nn.functional.cross_entropy(ref_logits.view(B, G), labels)
    ref_loss.backward()
    torch.cuda.synchronize()
    bound = (t.detach().abs() @ Wd.detach().abs().T).view(-1) + bd.detach().abs()
    err = (logits.cpu().double() - ref_logits.detach()).abs()
    assert bool((err <= 1e-6 + 2e-6 * bound).all()), float((err / (1e-6 + bound)).max())
    assert abs(float(loss) - float(ref_loss.detach())) <= 1e-5 * (1.0 + float(ref_loss.detach()))
    dx = x.grad
    # one bf16 rounding, plus fp32's 1 - t^2 where tanh saturates
    amp = ref_logits.grad.abs().view(-1, 1) * Wd.detach().abs() * mult
    assert bool(((dpre.cpu().double() - dx).abs() <= 2 ** -8 * dx.abs() + 1e-6 * amp + 1e-12).all())
    scale = (t.detach().abs().sum(0) / B + 1e-30)
    assert bool(((dW.cpu().double().view(-1) - Wd.grad.view(-1)).abs() <= 1e-5 * scale + 1e-9).all())
    assert abs(float(db) - float(bd.grad)) <= 1e-6 * N / B + 1e-7


def test_group_ce_kernel_is_bitwise_repeatable():
    from dpr_scale_b200 import ops
    pre, W, b, labels = _kernel_inputs(300, 8, 768, 9)
    args = (pre.cuda(), W.cuda(), b.cuda(), labels.cuda(), 8, P, 77)
    first = ops.seqcls_group_ce(*args)
    for _ in range(2):
        again = ops.seqcls_group_ce(*args)
        for a, c in zip(first, again):
            assert torch.equal(a, c)


def test_group_ce_kernel_rejects_bad_shapes_before_launching():
    from dpr_scale_b200 import _lib, ops
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for rows, H, G in ((8, 128, 1), (130, 128, 65), (8, 100, 4), (8, 1032, 4), (9, 128, 4)):
        with pytest.raises(ValueError):
            ops.seqcls_group_ce(torch.zeros(rows, H, device="cuda"), torch.zeros(1, H, device="cuda"), None,
                                torch.zeros(max(rows // max(G, 1), 1), dtype=torch.int64, device="cuda"), G)
    with pytest.raises(ValueError):                                   # two labels
        ops.seqcls_group_ce(torch.zeros(8, 128, device="cuda"), torch.zeros(2, 128, device="cuda"), None,
                            torch.zeros(2, dtype=torch.int64, device="cuda"), 4)
    # the C entry point checks the same limits itself
    lib = _lib.load()
    buf = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    x = torch.zeros(130, 128, device="cuda")
    lab = torch.zeros(2, dtype=torch.int64, device="cuda")
    outs = [torch.empty(130 * 128, device="cuda") for _ in range(5)]
    for B, G, H, p in ((2, 65, 128, 0.0), (2, 1, 128, 0.0), (2, 4, 100, 0.0), (2, 4, 128, 1.0), (0, 4, 128, 0.0)):
        rc = lib.dprb_seqcls_group_ce(x.data_ptr(), x.data_ptr(), None, lab.data_ptr(), B, G, H, p, 0,
                                      *[o.data_ptr() for o in outs], buf.data_ptr(), buf.numel(),
                                      torch.cuda.current_stream().cuda_stream)
        assert rc != 0
    assert ops.launch_count() == n0


# ------------------------------------------------------------------ tiny models against the oracle
def _tiny(kind, p, seed=3):
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    cfg = dict(rerank_cases.tiny_config(kind), num_labels=1, hidden_dropout_prob=p, attention_probs_dropout_prob=p)
    m = CrossEncoder.from_config(cfg, seed=seed)
    with torch.no_grad():
        gen = torch.Generator().manual_seed(4)
        for q in m.parameters():
            q.add_(0.02 * torch.randn(q.shape, generator=gen))
        m._head_linears()[1].weight.mul_(20.0)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    return m.cuda(), sd


def _tokens(kind, N, S, seed):
    g = torch.Generator().manual_seed(seed)
    pad = 1 if kind == "roberta" else 0
    ids = torch.randint(5, rerank_cases.VOCAB, (N, S), generator=g)
    lens = torch.randint(max(2, S // 3), S + 1, (N,), generator=g)
    lens[0] = S
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).to(torch.int64)
    ids = torch.where(am.bool(), ids, torch.full_like(ids, pad))
    tt = ((torch.arange(S).unsqueeze(0) >= (lens // 2).unsqueeze(1)) & am.bool()).to(torch.int64)
    return {"input_ids": ids, "token_type_ids": tt, "attention_mask": am}


@pytest.mark.parametrize("kind", ["bert", "roberta"])
@pytest.mark.parametrize("S", [24, 300, 512])
@pytest.mark.parametrize("p", [0.0, P])
def test_tiny_training_loss_and_grads_match_float64_oracle(kind, S, p):
    from dpr_scale_b200 import ops
    from oracle.cross_encoder_train import group_ce
    B, G = 2, 4
    N = B * G
    m, sd = _tiny(kind, p)
    m.train()
    tok = _tokens(kind, N, S, 7 + S)
    labels = torch.tensor([0, 2])
    loss, logits = m.group_ce({k: v.cuda() for k, v in tok.items()}, labels, G)
    loss.backward()
    torch.cuda.synchronize()
    H, heads, L = m.config["hidden_size"], m.config["num_attention_heads"], m.config["num_hidden_layers"]
    body = head_in = head = None
    if p > 0:
        drop_p, seed = m._body.last_dropout
        body = _masks(drop_p, seed, N, S, H, heads, L)
        sc = 1.0 / (1.0 - round(p * 65536) / 65536.0)
        head = ops.dropout_mask(N, H, p, seed, 0, ops.DROP_SITE_HEAD).double().cpu() * sc
        if kind == "roberta":
            head_in = ops.dropout_mask(N, H, p, seed, 0, ops.DROP_SITE_HEAD_IN).double().cpu() * sc
        body = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else v.double())
                for k, v in body.items()}
    ref_sd = {k: v.double().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ocfg = rerank_cases.ORACLE_CFG[kind]
    ref_loss, ref_logits = group_ce(ref_sd, ocfg, tok, labels, G, body, head_in, head)
    ref_loss.backward()
    assert rel_l2(logits.cpu().double(), ref_logits.detach()) <= 2e-2
    assert abs(float(loss) - float(ref_loss)) <= 1e-2 * max(1.0, float(ref_loss))
    if p > 0:                                     # the masks took effect
        plain, _ = group_ce({k: v.detach() for k, v in ref_sd.items()}, ocfg, tok, labels, G)
        assert abs(float(plain) - float(ref_loss)) > 1e-3
    top = max(float(v.grad.norm()) for v in ref_sd.values() if v.grad is not None)
    worst, checked = (1.0, 0.0), 0
    for k, q in m.named_parameters():
        r = ref_sd[k].grad
        if r is None or float(r.norm()) < 1e-5 * top:
            continue
        got = q.grad.detach().double().cpu()
        cs, rl = cosine(got, r), rel_l2(got, r)
        worst = (min(worst[0], cs), max(worst[1], rl))
        assert cs >= 0.997 and rl <= 7e-2, (k, cs, rl)
        checked += 1
    assert checked >= 20
    print(f"{kind} S={S} p={p}: loss {float(loss):.5f} vs {float(ref_loss):.5f}, worst grad cos / rel {worst}")


def test_optimizer_steps_reduce_the_loss():
    from dpr_scale_b200.optim import FusedAdamW
    m, _ = _tiny("bert", 0.0)
    m.train()
    opt = FusedAdamW(m.parameters(), lr=1e-3)
    opt.attach_encoders([m._body])
    tok = {k: v.cuda() for k, v in _tokens("bert", 16, 24, 3).items()}
    labels = torch.zeros(4, dtype=torch.int64)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss, _ = m.group_ce(tok, labels, 4)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.5 * losses[0], losses
    assert losses == sorted(losses, reverse=True), losses


# ------------------------------------------------------------------ end to end
def _train_args(mdir, ckpt_dir, data):
    return ["task=cross_encoder_train", "task/model=cross_encoder", "datamodule=cross_encoder_train",
            f"task.model.model_path={mdir}", f"task.transform.max_seq_len={rerank_cases.MAX_LEN}",
            "task.optim.lr=1.0e-04", "task.warmup_steps=1", f"datamodule.train_path={data}",
            f"datamodule.val_path={data}", f"datamodule.test_path={data}", "datamodule.batch_size=4",
            "datamodule.val_batch_size=4", "datamodule.test_batch_size=4", "datamodule.num_negative=3",
            "datamodule.num_val_negative=3", "trainer.max_epochs=1", f"checkpoint_callback.dirpath={ckpt_dir}"]


def test_main_trains_a_checkpoint_that_rerank_loads(tmp_path):
    cfg = dict(rerank_cases.tiny_config("bert"), hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    mdir = rerank_cases.hf_model_dir(str(tmp_path / "model"), cfg, rerank_cases.TINY["bert"]["seed"])
    ckpt_dir, out = str(tmp_path / "ckpt"), str(tmp_path / "out")
    env = dict(os.environ, PYTHONPATH=ROOT)
    data = os.path.join(DATA, "synth.jsonl")
    run = subprocess.run([sys.executable, "-m", "dpr_scale_b200.main"] + _train_args(mdir, ckpt_dir, data), cwd=ROOT,
                         env=env, timeout=900, capture_output=True, text=True)
    assert run.returncode == 0, run.stdout[-3000:] + run.stderr[-3000:]
    best = os.path.join(ckpt_dir, "checkpoint_best.ckpt")
    assert os.path.exists(best), sorted(glob.glob(ckpt_dir + "/*"))
    kw = rerank_cases.datamodule_kwargs()
    cmd = [sys.executable, "-m", "dpr_scale_b200.rerank", "task=cross_encoder_rerank", "task/model=cross_encoder",
           "datamodule=cross_encoder_rerank", f"task.model.model_path={mdir}",
           f"task.transform.max_seq_len={rerank_cases.MAX_LEN}", f"task.pretrained_checkpoint_path={best}",
           f"datamodule.test_path={kw['test_path']}", f"datamodule.test_question_path={kw['test_question_path']}",
           f"datamodule.test_passage_path={kw['test_passage_path']}", "datamodule.use_title=true",
           f"+task.output_dir={out}"]
    run = subprocess.run(cmd, cwd=ROOT, env=env, timeout=900, capture_output=True, text=True)
    assert run.returncode == 0, run.stdout[-3000:] + run.stderr[-3000:]
    assert f"Loaded state dict from {best}" in run.stdout
    # the rerank scores are the trained model's, not the starting checkpoint's
    from dpr_scale_b200.models.citadel_models.cross_encoder import CrossEncoder
    sd = torch.load(best, map_location="cpu", weights_only=False)["state_dict"]
    start = CrossEncoder(mdir)
    changed = [k for k, v in start.state_dict().items() if not torch.equal(v, sd["cross_encoder." + k])]
    assert changed
    with open(os.path.join(out, "scores_0000.pkl"), "rb") as f:
        scores = torch.as_tensor(pickle.load(f)).reshape(-1)
    assert scores.numel() > 0 and bool(torch.isfinite(scores).all())
    assert os.path.getsize(os.path.join(out, "rerank.trec")) > 0
