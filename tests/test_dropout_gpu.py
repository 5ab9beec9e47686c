"""Dropout parity: in train mode the CUDA path applies HF's four dropout sites (embeddings, attention probabilities,
attention-output dense, FFN-output dense) with counter-based masks that are never stored.  The test exports the masks
(dprb_dropout_mask), replays them in the CPU oracle and compares embeddings and parameter gradients (linear probe)."""
import pytest
import torch

from tests.util import BERT_TINY_CFG, cosine, load_golden, rel_l2, sub

pytestmark = pytest.mark.gpu
P = 0.1


def _masks(p, seed, N, S, H, heads, layers):
    """The multipliers keep / (1 - p) of all four dropout sites of one forward's seed (`enc.last_dropout`), as the
    oracle's `dropout=` argument takes them."""
    from dpr_scale_b200 import ops
    assert abs(p - P) < 1e-7
    sc = 1.0 / (1.0 - round(p * 65536) / 65536.0)  # the kernels quantise p to 16 bits
    T = N * S
    out = {"emb": ops.dropout_mask(T, H, p, seed, 0, 0).view(N, S, H).float().cpu() * sc}
    for l in range(layers):
        out[l] = {
            "attn": ops.dropout_mask(N * heads * S, S, p, seed, l, 1).view(N, heads, S, S).float().cpu() * sc,
            "attn_out": ops.dropout_mask(T, H, p, seed, l, 2).view(N, S, H).float().cpu() * sc,
            "ffn_out": ops.dropout_mask(T, H, p, seed, l, 3).view(N, S, H).float().cpu() * sc,
        }
    return out


def test_dropout_matches_oracle_with_replayed_masks():
    from dpr_scale_b200.models.hf_model import HFEncoder
    from oracle import encoder as oenc
    from tests.test_task_gpu import CFG, _batch
    g = load_golden("golden_1rank.npz")
    enc = HFEncoder.from_config(CFG, dropout=P)
    enc.load_state_dict(sub(g, "sd_c/"))
    enc = enc.cuda().train()
    tokens = _batch(g)["contexts_ids"]
    N, S = tokens["input_ids"].shape
    probe = torch.randn(N, 128, generator=torch.Generator().manual_seed(5))
    enc.zero_grad()
    rep = enc(tokens)
    (rep * probe.cuda()).sum().backward()
    torch.cuda.synchronize()
    masks = _masks(*enc.last_dropout, N, S, 128, 2, 2)
    keep_rate = float((masks[0]["attn"] > 0).float().mean())
    assert abs(keep_rate - (1 - P)) < 0.02, keep_rate
    sd = {k: v.clone().requires_grad_(True) for k, v in sub(g, "sd_c/").items()}
    ref = oenc.encode(sd, BERT_TINY_CFG, tokens, dropout=masks)
    (ref * probe).sum().backward()
    assert rel_l2(rep.detach().cpu(), ref.detach()) <= 1e-2, rel_l2(rep.detach().cpu(), ref.detach())
    # and it differs from the no-dropout output (the masks really were applied)
    assert rel_l2(rep.detach().cpu(), oenc.encode(sub(g, "sd_c/"), BERT_TINY_CFG, tokens)) > 5e-2
    top = max(float(v.grad.norm()) for k, v in sd.items() if v.grad is not None)
    worst = 1.0
    for k, p in enc.named_parameters():
        r = sd[k].grad
        if r is None or float(r.norm()) < 1e-5 * top:
            continue
        cs = cosine(p.grad.detach().cpu(), r)
        worst = min(worst, cs)
        assert cs >= 0.999, (k, cs)
        assert rel_l2(p.grad.detach().cpu(), r) <= 3e-2, (k, rel_l2(p.grad.detach().cpu(), r))
    print("dropout probe: worst gradient cosine", worst)


def test_dropout_is_off_in_eval_and_reseeds_each_forward():
    from dpr_scale_b200.models.hf_model import HFEncoder
    from tests.test_task_gpu import CFG, _batch
    g = load_golden("golden_1rank.npz")
    enc = HFEncoder.from_config(CFG, dropout=P)
    enc.load_state_dict(sub(g, "sd_c/"))
    enc = enc.cuda()
    tokens = _batch(g)["contexts_ids"]
    enc.eval()
    with torch.no_grad():
        a, b = enc(tokens), enc(tokens)
    assert torch.equal(a, b) and enc.last_dropout[0] == 0.0
    enc.train()
    c, d = enc(tokens).detach(), enc(tokens).detach()
    assert not torch.equal(c, d)  # fresh masks per forward
    assert rel_l2(c, a) > 1e-2


def test_mask_statistics():
    """The counter-based masks (one hash chain per 8 columns, a finaliser per column pair: csrc/common.cuh Drop) behave
    like independent Bernoulli(1 - p) draws: keep rate, and no correlation between neighbouring columns (same pair, same
    group, next group), neighbouring rows, or two sites / layers of the same seed."""
    from dpr_scale_b200 import ops
    rows, cols, p = 4096, 768, 0.1
    m = ops.dropout_mask(rows, cols, p, 5, 3, 2).float()
    assert abs(float(m.mean()) - (1 - p)) < 2e-3, float(m.mean())
    per_col = m.mean(0)
    assert float((per_col - (1 - p)).abs().max()) < 0.03          # 4096 draws per column: sigma = 0.0047

    def corr(a, b):
        a, b = a - a.mean(), b - b.mean()
        return float((a * b).mean() / (a.std() * b.std()))

    other_site = ops.dropout_mask(rows, cols, p, 5, 3, 3).float()
    other_layer = ops.dropout_mask(rows, cols, p, 5, 4, 2).float()
    pairs = {"same pair": (m[:, 0::2], m[:, 1::2]), "next pair": (m[:, :-2], m[:, 2:]), "next group": (m[:, :-8], m[:, 8:]),
             "next row": (m[:-1], m[1:]), "other site": (m, other_site), "other layer": (m, other_layer)}
    for name, (a, b) in pairs.items():
        assert abs(corr(a, b)) < 5e-3, (name, corr(a, b))          # sigma of the estimate: 6e-4
    assert not torch.equal(m, other_site) and not torch.equal(m, other_layer)


def test_masks_equal_host_restatement():
    """dprb_dropout_mask (the same `Drop` every kernel uses) against oracle/dropout.py, bit for bit: several shapes
    (incl. widths that are not multiples of 8), probabilities, 64-bit seeds, layers and sites."""
    from dpr_scale_b200 import ops
    from oracle import dropout as od
    cases = [(64, 768, 0.1, 7, 0, 0), (300, 128, 0.1, 7, 11, 1), (33, 1024, 0.5, 2 ** 63 + 12345, 23, 2),
             (257, 100, 0.25, 0xDEADBEEFCAFE, 5, 3), (5, 6, 0.9, 1, 0, 1), (1000, 3072, 0.1, 99, 2, 3)]
    for rows, cols, p, seed, layer, site in cases:
        got = ops.dropout_mask(rows, cols, p, seed, layer, site).cpu().numpy()
        want = od.keep_mask(rows, cols, p, seed, layer, site)
        assert (got == want).all(), (rows, cols, p, seed, layer, site, int((got != want).sum()))
    assert ops.dropout_site_seed(2 ** 63 + 12345, 23, 2) == od.site_seed32(2 ** 63 + 12345, 23, 2)
