"""The S <= 128 attention backward (attn_bwd_short_kernel in csrc/attention_wgmma.cu): a persistent kernel that loops
each CTA over the sequences of one head, writes dQ once without atomics and sums the QKV bias gradient itself.

  * attention-probability dropout against float64 (tests/gpu_checks.check_attention) at lengths on both key paddings,
    with holes and prefix masks, 12 and 16 heads; the backward must also be bitwise repeatable there;
  * bitwise repeatability at the training step's shape and at S = 1, 64, 100;
  * schedule invariance: a sequence's dQ / dK / dV are the same bits whether it is computed alone, in a batch that
    fills the grid unevenly, or in a batch larger than the grid;
  * the fused bias gradient: accumulated into dbias (ones here) as the float64 column sums of the returned bf16 dqkv,
    and dbias = None leaves dqkv unchanged.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

P_DROP = 0.1
DEV = "cuda"


def _bits(t):
    return t.view(torch.int16)


def _problem(nseq, S, heads, seed, mask="holes"):
    from dpr_scale_b200 import ops
    from tests.gpu_checks import attn_mask
    g = torch.Generator(device=DEV).manual_seed(seed)
    H = heads * 64
    qkv = (2 * torch.randn(nseq * S, 3 * H, device=DEV, generator=g)).to(torch.bfloat16)
    dctx = torch.randn(nseq * S, H, device=DEV, generator=g).to(torch.bfloat16)
    am = attn_mask(mask, nseq, S, torch.Generator().manual_seed(seed))
    am = am.to(DEV) if am is not None else None
    site = ops.dropout_site_seed(0x5EED + seed, 3, 1)
    ctx, lse = ops.attn_fwd(qkv, am, nseq, S, heads, True, P_DROP, site)
    return dict(qkv=qkv, am=am, ctx=ctx, lse=lse, dctx=dctx, nseq=nseq, S=S, heads=heads, site=site)


def _bwd(p, dbias=None, nseq=None):
    """dqkv of the first nseq sequences of problem p (all of them by default)."""
    from dpr_scale_b200 import ops
    n = p["nseq"] if nseq is None else nseq
    S, heads = p["S"], p["heads"]
    T = n * S
    am = None if p["am"] is None else p["am"][:n]
    return ops.attn_bwd(p["qkv"][:T], am, p["ctx"][:T], p["lse"][:n], p["dctx"][:T], n, S, heads, dbias, P_DROP,
                        p["site"])


DROP_CASES = [(S, heads, mask) for S in (17, 64, 65, 100, 128) for heads in (12, 16) for mask in ("holes", "prefix")]


@pytest.mark.parametrize("S,heads,mask", DROP_CASES, ids=[f"S{c[0]}-h{c[1]}-{c[2]}" for c in DROP_CASES])
def test_dropout_matches_float64(S, heads, mask):
    from tests.gpu_checks import check_attention
    nseq = 5 if mask == "prefix" else 3
    res = check_attention(nseq, S, heads, seed=4000 + 7 * S + heads, dropout=P_DROP, mask=mask, qscale=4.0)
    print({k: f"{v:.3g}" for k, v in res.items()})
    assert res["bwd_repeatable"] == 1.0, "the S <= 128 attn_bwd is not bitwise repeatable"


@pytest.mark.parametrize("nseq,S,heads", [(1024, 128, 12), (300, 1, 12), (200, 64, 12), (150, 100, 16)],
                         ids=["bench-1024x128-h12", "S1", "S64", "S100"])
def test_bitwise_repeatable(nseq, S, heads):
    p = _problem(nseq, S, heads, seed=S)
    a = _bwd(p, torch.zeros(3 * heads * 64, device=DEV))
    b = _bwd(p, torch.zeros(3 * heads * 64, device=DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(a.float()).all()
    assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("nseq,heads", [(1, 1), (131, 1), (19, 7), (12289, 1)],
                         ids=["probs1", "probs131", "probs133", "probs12289"])
def test_schedule_invariant(nseq, heads):
    """The first sequence alone, the first nseq - 1 and all nseq: every CTA computes whole problems, so the rows of a
    sequence do not depend on which CTA ran it or how many problems it ran before."""
    S = 100
    p = _problem(nseq, S, heads, seed=nseq)
    whole = _bwd(p, torch.zeros(3 * heads * 64, device=DEV))
    alone = _bwd(p, torch.zeros(3 * heads * 64, device=DEV), nseq=1)
    assert torch.equal(_bits(alone), _bits(whole[:S]))
    if nseq > 1:
        part = _bwd(p, None, nseq=nseq - 1)
        assert torch.equal(_bits(part), _bits(whole[:(nseq - 1) * S]))


@pytest.mark.parametrize("T", [131072, 16384], ids=["ctx-encoder", "query-encoder"])
def test_fused_dbias(T):
    S, heads = 128, 12
    p = _problem(T // S, S, heads, seed=T, mask="random_prefix")
    dbias = torch.ones(3 * heads * 64, device=DEV)
    with_bias = _bwd(p, dbias)
    without = _bwd(p, None)
    torch.cuda.synchronize()
    assert torch.equal(_bits(with_bias), _bits(without)), "dbias = None changed dqkv"
    want = 1 + with_bias.double().sum(0)
    err = float((dbias.double() - want).abs().max())
    assert err <= 1e-5 * float(want.abs().max()), (err, float(want.abs().max()))
