"""The full self-attention kernels (csrc/attention_wgmma.cu for S <= 256, csrc/attention_long.cu above) against float64,
through tests/gpu_checks.check_attention (its docstring states the gates and the exact checks):

  * every length where the kernels change shape: 1, 2, 16, 17; 63 / 64 / 65 and 127 / 128 / 129 around the switches of
    the short kernels' key padding (64 -> 128 -> 256 keys); 192, 255, 256; 257, 320, 383 / 384 / 385, 449, 511, 512
    around the long kernels' 128-key blocks; 1, 2, 12 and 16 heads in turn;
  * masks: none, prefixes (1, S - 1, S, one key into the last 64- and 128-key block), ~70 % holes with an interior hole
    across a block boundary, left padding (fully masked leading key blocks: the long forward's "no unmasked key yet"
    branch), a single valid key at S - 1;
  * logit scales 1, 4, 10 (|logit| up to ~30), and a late maximum per kernel family (every row's running maximum
    grows at every key block, so the long forward rescales O and l each time);
  * attention-probability dropout replayed from dprb_dropout_mask (site 1), short and long, with holes;
  * more than 65 535 (sequence, head) problems on the short kernels, every problem compared;
  * a 2-head encoder forward over 32 800 sequences (65 600 problems in layer 0) equal to the same sequences encoded
    in batches of 1 024.

Sequences whose mask is all zero are not covered (see check_attention).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

S_SHORT = (1, 2, 16, 17, 63, 64, 65, 127, 128, 129, 192, 255, 256)
S_LONG = (257, 320, 383, 384, 385, 449, 511, 512)
HEADS = (1, 2, 12, 16)
MASKS = ("none", "prefix", "holes", "left", "last")
QSCALES = (1.0, 4.0, 10.0)
P_DROP = 0.1


def _cases():
    cases = []
    for i, S in enumerate(S_SHORT + S_LONG):
        for j, mask in enumerate(MASKS):
            # prefix / left: 5 sequences, one of each length or padding in turn
            nseq = 5 if mask in ("prefix", "left") else 3
            cases.append((nseq, S, HEADS[(i + j) % 4], mask, QSCALES[(i + j) % 3], False, 0.0))
    cases.append((3, 256, 2, "none", 1.0, True, 0.0))
    cases.append((3, 512, 2, "none", 1.0, True, 0.0))
    cases.append((4, 129, 12, "holes", 4.0, False, P_DROP))
    cases.append((3, 385, 2, "holes", 4.0, False, P_DROP))
    return cases


CASES = _cases()


@pytest.mark.parametrize("nseq,S,heads,mask,qscale,late_max,dropout", CASES,
                         ids=[f"n{c[0]}-S{c[1]}-h{c[2]}-{c[3]}-q{c[4]:g}{'-late' if c[5] else ''}-p{c[6]:g}"
                              for c in CASES])
def test_attention_matches_float64(nseq, S, heads, mask, qscale, late_max, dropout):
    from tests.gpu_checks import check_attention
    res = check_attention(nseq, S, heads, seed=2000 + 7 * S + heads, dropout=dropout, mask=mask, qscale=qscale,
                          late_max=late_max)
    print({k: f"{v:.3g}" for k, v in res.items()})


@pytest.mark.parametrize("nseq,S,heads,mask", [(5462, 32, 12, "prefix"), (4097, 100, 16, "holes")],
                         ids=["S32-h12-65544probs", "S100-h16-65552probs"])
def test_attention_more_than_65535_problems(nseq, S, heads, mask):
    """The S <= 256 forward once put the problems on gridDim.y, which stops at 65 535."""
    from tests.gpu_checks import check_attention
    assert nseq * heads > 65535
    res = check_attention(nseq, S, heads, seed=3000 + S, mask=mask, qscale=4.0)
    print({k: f"{v:.3g}" for k, v in res.items()})


def test_encoder_forward_over_65535_problems_is_batch_invariant():
    """A 2-head encoder (layer 0 runs the full attention, layer 1 the pruned CLS attention) over 32 800 sequences of
    16 tokens in one call and in batches of 1 024: every kernel of the forward works row by row or problem by problem
    with the same tiles whatever the batch, so the pooled outputs are bitwise equal."""
    from dpr_scale_b200.models.hf_model import HFEncoder
    cfg = dict(vocab_size=64, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
               max_position_embeddings=16)
    enc = HFEncoder.from_config(cfg, dropout=0.1, seed=7)
    with torch.no_grad():
        gen = torch.Generator().manual_seed(8)
        for p in enc.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=gen))
    enc = enc.cuda().eval()
    N, S = 32800, 16
    gen = torch.Generator().manual_seed(9)
    lens = torch.randint(1, S + 1, (N,), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    tokens = {"input_ids": torch.randint(3, 64, (N, S), generator=gen) * am, "token_type_ids": torch.zeros(N, S).long(),
              "attention_mask": am}
    with torch.no_grad():
        whole = enc(tokens)
        parts = torch.cat([enc({k: v[i:i + 1024] for k, v in tokens.items()}) for i in range(0, N, 1024)])
    torch.cuda.synchronize()
    assert whole.shape == (N, 128) and torch.isfinite(whole).all()
    assert torch.equal(whole, parts), float((whole - parts).abs().max())
