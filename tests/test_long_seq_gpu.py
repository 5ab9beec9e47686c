"""Sequences of 256 < S <= 512 tokens on the GPU: the key-blocked attention kernels (csrc/attention_long.cu), the
16-keys-per-lane pruned last layer (csrc/cls_last.cu) and the assembled encoder.

  * kernel parity against float64 (tests/gpu_checks.check_attention: ctx 2^-7, lse 1e-4, dQ / dK / dV 2^-6 of each
    (sequence, head) problem's max|ref| + atol, fused QKV bias gradient), with and without a padding mask, many
    problems, and attention-probability dropout with the mask replayed from dprb_dropout_mask;
  * the two-kernel backward is deterministic; S = 513 is rejected before any launch;
  * BERT-base at S = 512 (sequence 0 uses position 511) against the reference-generated golden, with the gates of
    tests/test_realdims_gpu.py;
  * a tiny BERT (max_position_embeddings 512) and RoBERTa (514: pad-derived positions up to 513) at S = 512 against the
    oracle in lean-activation, forward-only and dropout mode, with the gates of the existing tiny-model tests.
"""
import pytest
import torch

from tests import realdims_long
from tests.gpu_checks import check_attention
from tests.util import cosine, load_golden, rel_l2

pytestmark = pytest.mark.gpu

PARITY = [(S, 1 + i % 4, masked) for i, S in enumerate((257, 300, 384, 449, 512)) for masked in (True, False)]


@pytest.mark.parametrize("S,heads,masked", PARITY)
def test_long_attention_matches_oracle(S, heads, masked):
    res = check_attention(nseq=2, S=S, heads=heads, masked=masked, seed=100 + S)
    print(S, heads, masked, {k: f"{v:.3g}" for k, v in res.items()})


def test_long_attention_many_problems():
    res = check_attention(nseq=16, S=512, heads=12, masked=True, seed=61)
    print({k: f"{v:.3g}" for k, v in res.items()})


@pytest.mark.parametrize("S", [320, 512])
def test_long_attention_dropout_matches_oracle_with_replayed_mask(S):
    res = check_attention(nseq=3, S=S, heads=2, masked=True, seed=70 + S, dropout=0.1)
    print(S, {k: f"{v:.3g}" for k, v in res.items()})


def test_long_attention_backward_is_deterministic():
    from dpr_scale_b200 import ops
    nseq, S, heads = 6, 512, 4
    g = torch.Generator().manual_seed(8)
    qkv = torch.randn(nseq * S, 3 * heads * 64, generator=g).to(torch.bfloat16).cuda()
    am = torch.ones(nseq, S, dtype=torch.int32)
    am[1, 300:] = 0
    am[4, 400:] = 0
    am = am.cuda()
    site = ops.dropout_site_seed(99, 0, 1)
    ctx, lse = ops.attn_fwd(qkv, am, nseq, S, heads, True, 0.1, site)
    dctx = torch.randn(nseq * S, heads * 64, generator=g).to(torch.bfloat16).cuda()
    outs = []
    for _ in range(2):
        dbias = torch.zeros(3 * heads * 64, device="cuda")
        outs.append((ops.attn_bwd(qkv, am, ctx, lse, dctx, nseq, S, heads, dbias, 0.1, site), dbias))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.isfinite(outs[0][0].float()).all()


def test_attention_rejects_513_before_launching():
    from dpr_scale_b200 import ops
    from dpr_scale_b200._lib import DprbError
    nseq, S, heads = 2, 513, 2
    qkv = torch.zeros(nseq * S, 3 * heads * 64, dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(DprbError, match="513"):
        ops.attn_fwd(qkv, None, nseq, S, heads)
    ctx = torch.zeros(nseq * S, heads * 64, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(nseq, heads, S, device="cuda")
    n1 = ops.launch_count()
    with pytest.raises(DprbError, match="513"):
        ops.attn_bwd(qkv, None, ctx, lse, ctx, nseq, S, heads)
    assert ops.launch_count() == n1
    assert n1 == n0


def test_bert_base_s512_training_step_matches_reference():
    from tests.test_realdims_gpu import _check_probe, _check_step
    name = realdims_long.NAME
    g = load_golden(f"realdims_{name}.npz")
    # the reference's own bf16 autocast is off by 0.64 on this batch (|logit| ~ 410): 5e-2 + a quarter of that
    gate = 5e-2 + 0.25 * abs(float(g["amp_loss"]) - float(g["loss"]))
    task, g = _check_step(name, gate)
    _check_probe(task, g, name)


# ------------------------------------------------------------------ tiny model at S = 512
TINY = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256)
KINDS = {
    "bert": (dict(TINY, model_type="bert", max_position_embeddings=512),
             {"layers": 2, "heads": 2, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}),
    "roberta": (dict(TINY, model_type="roberta", max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                     layer_norm_eps=1e-5),
                {"layers": 2, "heads": 2, "ln_eps": 1e-5, "pad_id": 1, "roberta": True}),
}
N, S = 4, 512


def _tiny(kind, dropout=0.0):
    from dpr_scale_b200.models.hf_model import HFEncoder
    cfg, ocfg = KINDS[kind]
    enc = HFEncoder.from_config(cfg, dropout=dropout, seed=3)
    with torch.no_grad():                 # non-zero biases / LayerNorm parameters
        gen = torch.Generator().manual_seed(4)
        for p in enc.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=gen))
    sd = {k: v.detach().clone() for k, v in enc.state_dict().items()}
    pad = cfg.get("pad_token_id", 0)
    gen = torch.Generator().manual_seed(5)
    lens = torch.randint(S // 4, S + 1, (N,), generator=gen)
    lens[0] = S                           # the last position is used
    ids = torch.randint(3, 64, (N, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    ids = ids * am + pad * (1 - am)
    tokens = {"input_ids": ids, "attention_mask": am}
    if kind == "bert":
        tokens["token_type_ids"] = torch.zeros_like(ids)
    return enc.cuda(), sd, tokens, ocfg


def _check_grads(enc, sd, tol_rel=3e-2):
    """Every parameter gradient of `enc` against the oracle's `sd[k].grad`: cosine >= 0.999 and rel-L2 <= tol_rel.
    Returns (worst cosine, worst rel-L2)."""
    top = max(float(v.grad.norm()) for v in sd.values() if v.grad is not None)
    worst, worst_rel, checked = 1.0, 0.0, 0
    for k, p in enc.named_parameters():
        r = sd[k].grad
        if r is None or float(r.norm()) < 1e-5 * top:
            continue
        got = p.grad.detach().float().cpu()
        cs, rl = cosine(got, r), rel_l2(got, r)
        worst, worst_rel = min(worst, cs), max(worst_rel, rl)
        assert cs >= 0.999 and rl <= tol_rel, (k, cs, rl)
        checked += 1
    assert checked >= 20
    return worst, worst_rel


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_tiny_s512_lean_activations_match_oracle(kind):
    from oracle import encoder as oenc
    enc, sd, tokens, ocfg = _tiny(kind)
    enc.lean_activations = True
    enc.train()                           # dropout 0: train mode only selects the save-for-backward path
    probe = torch.randn(N, 128, generator=torch.Generator().manual_seed(6))
    enc.zero_grad()
    rep = enc(tokens)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = oenc.encode(ref_sd, ocfg, tokens)
    (ref * probe).sum().backward()
    assert rel_l2(rep.detach().cpu(), ref.detach()) <= 1e-2, rel_l2(rep.detach().cpu(), ref.detach())
    print(kind, "lean: worst gradient cosine / rel-L2", _check_grads(enc, ref_sd))


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_tiny_s512_forward_only_matches_oracle(kind):
    from oracle import encoder as oenc
    enc, sd, tokens, ocfg = _tiny(kind, dropout=0.1)
    enc.eval()
    with torch.no_grad():
        rep = enc(tokens)
        rep2 = enc(tokens)
    assert enc.last_dropout[0] == 0.0 and torch.equal(rep, rep2)
    ref = oenc.encode(sd, ocfg, tokens)
    assert rel_l2(rep.cpu(), ref) <= 1e-2, rel_l2(rep.cpu(), ref)


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_tiny_s512_dropout_matches_oracle_with_replayed_masks(kind):
    from oracle import encoder as oenc
    from tests.test_dropout_gpu import P, _masks
    enc, sd, tokens, ocfg = _tiny(kind, dropout=P)
    enc.train()
    probe = torch.randn(N, 128, generator=torch.Generator().manual_seed(7))
    enc.zero_grad()
    rep = enc(tokens)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    masks = _masks(*enc.last_dropout, N, S, 128, 2, 2)
    keep_rate = float((masks[0]["attn"] > 0).float().mean())
    assert abs(keep_rate - (1 - P)) < 0.02, keep_rate
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = oenc.encode(ref_sd, ocfg, tokens, dropout=masks)
    (ref * probe).sum().backward()
    assert rel_l2(rep.detach().cpu(), ref.detach()) <= 1e-2, rel_l2(rep.detach().cpu(), ref.detach())
    assert rel_l2(rep.detach().cpu(), oenc.encode(sd, ocfg, tokens)) > 5e-2     # the masks really were applied
    print(kind, "dropout: worst gradient cosine / rel-L2", _check_grads(enc, ref_sd))
