"""The pruned last layer: only the CLS query attends and only the CLS rows go through the output GEMMs and LayerNorms
(csrc/cls_last.cu and the prune_last_layer() branches of csrc/encoder.cu).  Every forward of the library ends there.

  (a) the single-query attention kernels (dprb_attn_cls_fwd / _bwd, MAXK 8 for S <= 256 and 16 above) against a
      float64 softmax over the same bf16 qkv, at lengths around the 32-key lane chunks, 1..16 heads, partial last CTAs,
      no / prefix / holed masks, logits up to ~30 and attention-probability dropout; and against the full attention
      kernels with the same dropout site (the two are the same function of query 0);
  (b) the CLS-row dropout keys (site seed | S << 32: row r is keyed as token r * S): the pruned mask is the full mask
      restricted to the CLS rows, through the GEMM residual-dropout epilogue and both forms of dprb_ln_bwd; and the
      unpruned layer's LN2 backward (dy_cls on every S-th row, dropout) writes zero dz / dzm on the other rows;
  (c) a one-layer encoder (so its only layer is the pruned one) against the same encoder with DPRB_NO_CLS_PRUNE=1 and
      a float64 oracle.

Gates (bf16 outputs are rounded once: 2^-9 relative to the element; the gates are stated against max|ref| of each
compared block and the measured errors are printed):
  probs 1e-5 absolute; ctx_cls 2^-7 * max|ref| + 1e-4; dQ row 0, dK and dV each 2^-7 of their own max + 1e-5;
  full-kernel differentials: ctx 2^-7, dqkv 2^-6 + 4e-3 (the full kernels round P and dS to bf16 before the second
  matmuls, as check_attention states); GEMM fp16 output 2^-10 + 2e-3; LayerNorm dz / dzm 2^-7 + 1e-3 (check_ln's
  gates), and the fp32 column sums dgamma / dbeta / dbias 2e-6 of max|ref| + 1e-6 (measured 3e-7: fp32 accumulation
  order only; check_ln's 1e-4 would sit ~400x above it).
  Encoder: pooled outputs of the pruned and unpruned runs within 2^-7 of max|ref|; for every parameter tensor the
  pruned max-abs error against float64 is at most K_PRUNED = 2 times the unpruned one (measured worst ratio 1.59).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
P_DROP = 0.1


def _scale(p):
    return 1.0 / (1.0 - round(p * 65536) / 65536.0)   # the kernels quantise p to 16 bits


def _maxerr(got, ref):
    return float((got.double() - ref.double()).abs().max()) if got.numel() else 0.0


def _record(name, got, ref, out):
    """Merge max|got - ref| and max|ref| of one block (or one chunk of it) into out[name]."""
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{name}: non-finite values"
    err, scale = _maxerr(got, ref), float(ref.abs().max()) if ref.numel() else 0.0
    e0, s0 = out.get(name, (0.0, 0.0))
    out[name] = (max(e0, err), max(s0, scale))


def _check(name, rtol, atol, out):
    err, scale = out[name]
    assert err <= rtol * scale + atol, f"{name}: max err {err:.4e} > {rtol}*{scale:.4e}+{atol}"


def _gate(name, got, ref, rtol, atol, out):
    _record(name, got, ref, out)
    _check(name, rtol, atol, out)


# ================================================================== (a) single-query attention
def _lengths(S, n):
    """Prefix lengths: CLS only, S - 1, S, and lengths that end inside the last 32-key lane chunk."""
    last0 = 32 * ((S - 1) // 32)                   # first key of the last lane chunk
    cands = [1, max(1, S - 1), S, min(S, last0 + 1), min(S, last0 + 17), max(1, (S + 1) // 2)]
    return [cands[i % len(cands)] for i in range(n)]


def _mask(kind, nseq, S, g):
    if kind == "none":
        return None
    am = torch.ones(nseq, S, dtype=torch.int32)
    if kind == "prefix":
        for i, ln in enumerate(_lengths(S, nseq)):
            am[i, ln:] = 0
    else:                                          # holes: a random non-prefix mask; CLS is always a real token
        am = (torch.rand(nseq, S, generator=g) < 0.7).to(torch.int32)
        am[:, 0] = 1
        if S > 40:
            am[:, S // 3: S // 3 + 20] = 0         # one contiguous interior hole across a chunk boundary
    return am


def _qkv(nseq, S, heads, qscale, g):
    H = heads * 64
    x = torch.randn(nseq * S, 3 * H, generator=g)
    x[:, :H] *= qscale                              # |q.k| / 8 ~ qscale * N(0, 1): up to ~30 at qscale 10, S = 512
    return x.to(torch.bfloat16)


def _cls_reference(qkv, am, dctx, nseq, S, heads, mult):
    """float64: probs [nseq, heads, S], ctx [nseq, H], dq0 [nseq, H], dk / dv [nseq*S, H] of query 0."""
    H = heads * 64
    x = qkv.double().view(nseq, S, 3, heads, 64)
    q = x[:, 0, 0]                                  # nseq, heads, 64
    k = x[:, :, 1].transpose(1, 2)                  # nseq, heads, S, 64
    v = x[:, :, 2].transpose(1, 2)
    s = torch.einsum("nhd,nhsd->nhs", q, k) / 8.0
    if am is not None:
        s = s.masked_fill(am.view(nseq, 1, S) == 0, float("-inf"))
    p = torch.softmax(s, -1)
    pm = p * mult
    ctx = torch.einsum("nhs,nhsd->nhd", pm, v).reshape(nseq, H)
    dO = dctx.double().view(nseq, heads, 64)
    dpm = torch.einsum("nhd,nhsd->nhs", dO, v) * mult
    D = (p * dpm).sum(-1, keepdim=True)
    ds = p * (dpm - D) / 8.0
    dq0 = torch.einsum("nhs,nhsd->nhd", ds, k).reshape(nseq, H)
    dk = (ds[..., None] * q[:, :, None, :]).transpose(1, 2).reshape(nseq * S, H)
    dv = (pm[..., None] * dO[:, :, None, :]).transpose(1, 2).reshape(nseq * S, H)
    return p, ctx, dq0, dk, dv


def _sentinel(shape):
    """bf16 buffer filled with 0xFFFF (a NaN): an element the kernel does not write stays non-finite."""
    return torch.full(shape, -1, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def check_cls_attention(nseq, S, heads, mask, qscale, seed, dropout=0.0):
    from dpr_scale_b200 import ops
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = _qkv(nseq, S, heads, qscale, g).to(DEV)
    am = _mask(mask, nseq, S, g)
    amd = am.to(DEV) if am is not None else None
    dctx = torch.randn(nseq, H, generator=g).to(torch.bfloat16).to(DEV)
    dseed, layer = 0x5EED + seed, 5
    site = ops.dropout_site_seed(dseed, layer, 1) if dropout else 0
    mult = torch.ones(nseq, heads, S, dtype=torch.float64, device=DEV)
    if dropout:   # query 0 of problem (seq, h) is row (seq*heads + h)*S of the attention-probability site
        keep = ops.dropout_mask(nseq * heads * S, S, dropout, dseed, layer, 1).view(nseq * heads, S, S)[:, 0]
        mult = keep.view(nseq, heads, S).double() * _scale(dropout)
    ctx, probs = ops.attn_cls_fwd(qkv, amd, nseq, S, heads, dropout, site)
    dqkv = ops.attn_cls_bwd(qkv, probs, dctx, nseq, S, heads, dropout, site, dqkv=_sentinel((nseq * S, 3 * H)))
    dqkv2 = ops.attn_cls_bwd(qkv, probs, dctx, nseq, S, heads, dropout, site, dqkv=_sentinel((nseq * S, 3 * H)))
    torch.cuda.synchronize()
    assert torch.equal(dqkv.view(torch.int16), dqkv2.view(torch.int16)), "attn_cls_bwd is not deterministic"
    del dqkv2
    res = {}
    d = dqkv.view(nseq, S, 3 * H)
    # the float64 reference one chunk of sequences at a time: at most 2^25 qkv elements (256 MB in float64)
    step = max(1, (1 << 25) // (S * 3 * H))
    for s0 in range(0, nseq, step):
        s1 = min(nseq, s0 + step)
        n = s1 - s0
        amc = amd[s0:s1] if amd is not None else None
        p, c, dq0, dk, dv = _cls_reference(qkv[s0 * S:s1 * S], amc, dctx[s0:s1], n, S, heads, mult[s0:s1])
        _record("probs", probs[s0:s1], p, res)
        _record("ctx_cls", ctx[s0:s1], c, res)
        dc = d[s0:s1]
        # dqkv started as a NaN sentinel: _record also requires every element it compares to be written and finite
        _record("dq_row0", dc[:, 0, :H], dq0, res)
        _record("dk", dc[:, :, H:2 * H].reshape(-1, H), dk, res)
        _record("dv", dc[:, :, 2 * H:].reshape(-1, H), dv, res)
        if S > 1:
            assert float(dc[:, 1:, :H].float().abs().max()) == 0.0, "dQ rows j > 0 must be exactly zero"
        if amc is not None:
            assert not probs[s0:s1].masked_select(amc.view(n, 1, S) == 0).any(), "masked keys must get probability 0"
            if bool((amc == 0).any()):
                assert float(dc[:, :, H:][amc == 0].float().abs().max()) == 0.0, \
                    "dK / dV of masked keys must be exactly zero"
        del p, c, dq0, dk, dv
    _check("probs", 0.0, 1e-5, res)
    _check("ctx_cls", 2 ** -7, 1e-4, res)
    for name in ("dq_row0", "dk", "dv"):
        _check(name, 2 ** -7, 1e-5, res)
    return res, (qkv, amd, ctx, probs, dctx, dqkv, site)


S_SHORT = (1, 2, 31, 32, 33, 100, 128, 255, 256)     # MAXK 8
S_LONG = (257, 288, 300, 449, 480, 511, 512)         # MAXK 16
HEADS = (1, 2, 12, 16)


def _cls_cases():
    cases = []
    for i, S in enumerate(S_SHORT + S_LONG):
        # nseq 5: 5 / 10 / 60 / 80 problems (1, 2 and 12 heads leave a partial last CTA of 8 warps)
        cases.append((5, S, HEADS[i % 4], "prefix", 10.0 if i % 2 else 3.0, 0.0))
        cases.append((3, S, HEADS[(i + 1) % 4], "holes" if i % 2 else "none", 3.0 if i % 2 else 10.0, 0.0))
    for S, heads in ((33, 12), (100, 2), (256, 16), (300, 1), (480, 12), (512, 16)):
        cases.append((5, S, heads, "prefix", 4.0, P_DROP))
    cases.append((3, 511, 2, "holes", 4.0, P_DROP))
    cases.append((256, 512, 16, "prefix", 10.0, 0.0))   # 4096 problems
    cases.append((300, 256, 12, "holes", 4.0, P_DROP))  # 3600 problems, MAXK 8
    return cases


CLS_CASES = _cls_cases()


@pytest.mark.parametrize("nseq,S,heads,mask,qscale,dropout", CLS_CASES,
                         ids=[f"n{c[0]}-S{c[1]}-h{c[2]}-{c[3]}-q{c[4]:g}-p{c[5]:g}" for c in CLS_CASES])
def test_cls_attention_matches_float64(nseq, S, heads, mask, qscale, dropout):
    res, _ = check_cls_attention(nseq, S, heads, mask, qscale, seed=1000 + S * 7 + heads, dropout=dropout)
    print({k: f"{e:.3g}/{s:.3g}" for k, (e, s) in res.items()})


@pytest.mark.parametrize("S,heads", [(100, 12), (256, 16), (300, 2), (512, 16)])
def test_cls_attention_matches_full_kernels_with_dropout(S, heads):
    """The single-query kernels against row 0 of the full attention kernels on the same dropout site: forward ctx, and the
    full backward fed a dctx that is zero outside the CLS rows (mathematically the same dqkv)."""
    from dpr_scale_b200 import ops
    nseq = 3
    _, (qkv, amd, ctx, probs, dctx, dqkv, site) = check_cls_attention(nseq, S, heads, "prefix", 4.0, seed=77 + S,
                                                                      dropout=P_DROP)
    H = heads * 64
    full_ctx, lse = ops.attn_fwd(qkv, amd, nseq, S, heads, True, P_DROP, site)
    res = {}
    _gate("ctx_vs_full", ctx, full_ctx.view(nseq, S, H)[:, 0], 2 ** -7, 1e-4, res)
    dctx_full = torch.zeros(nseq, S, H, dtype=torch.bfloat16, device=DEV)
    dctx_full[:, 0] = dctx
    full_dqkv = ops.attn_bwd(qkv, amd, full_ctx, lse, dctx_full.view(nseq * S, H), nseq, S, heads, None, P_DROP, site)
    torch.cuda.synchronize()
    _gate("dqkv_vs_full", dqkv, full_dqkv, 2 ** -6, 4e-3, res)
    print({k: f"{e:.3g}/{s:.3g}" for k, (e, s) in res.items()})


# ================================================================== (b) CLS-row dropout keys
def _cls_site(seed, layer, site, S):
    from oracle import dropout as od
    return od.site_seed32(seed, layer, site) | (S << 32)     # encoder.cu site_seed_cls


@pytest.mark.parametrize("R,S,H", [(7, 40, 768), (1000, 77, 1024), (33, 512, 256)])
def test_cls_row_mask_is_the_full_mask_on_cls_rows(R, S, H):
    from dpr_scale_b200 import ops
    from oracle import dropout as od
    seed, layer, site = 0xC1A55 + R, 11, 2
    full = ops.dropout_mask(R * S, H, P_DROP, seed, layer, site)[::S].cpu().numpy()
    want = od.keep_mask(R, H, P_DROP, seed, layer, site, row_mul=S)
    assert np.array_equal(full, want), int((full != want).sum())
    assert not np.array_equal(want, od.keep_mask(R, H, P_DROP, seed, layer, site))   # the row key matters


@pytest.mark.parametrize("R,S,H", [(7, 40, 768), (7, 300, 1024), (1000, 77, 768), (1000, 40, 1024)])
def test_gemm_residual_dropout_on_cls_rows(R, S, H):
    """The pruned layer's output GEMMs: D(fp16) = dropout(A W^T + bias) + stream[r * S] with ld_aux = S * H from the
    full fp16 residual stream, the mask keyed by row r * S."""
    from dpr_scale_b200 import ops
    from oracle import dropout as od
    from tests.gpu_checks import _bf
    from tests.test_gemm_epilogue_gpu import _guarded, _untouched
    g = torch.Generator().manual_seed(R + S + H)
    A = _bf(torch.randn(R, H, generator=g))
    W = _bf(torch.randn(H, H, generator=g) * 0.05)
    bias = torch.randn(H, generator=g)
    stream = (torch.randn(R * S, H, generator=g) * 3).half()
    seed, layer = 0xBEEF + R, 4
    out_buf, out = _guarded(R, H, H, torch.float16, g)
    before = out_buf.clone()
    ops.gemm(A.cuda(), W.cuda(), out, R, H, H, H, H, H, False, False,
             ops.EPI_BIAS_RESIDUAL | ops.GEMM_AUX_F16 | ops.GEMM_OUT_F16, bias.cuda(), stream.cuda(), S * H,
             dropout_p=P_DROP, drop_seed=_cls_site(seed, layer, 2, S))
    torch.cuda.synchronize()
    keep = torch.from_numpy(od.keep_mask(R, H, P_DROP, seed, layer, 2, row_mul=S)).double()
    want = (A.double() @ W.double().T + bias.double()) * keep * od.scale(P_DROP) + stream[::S].double()
    res = {}
    _gate("gemm_cls_drop", out.cpu(), want, 2 ** -10, 2e-3, res)
    _untouched("gemm_cls_drop", before, out_buf, R, H)
    print({k: f"{e:.3g}/{s:.3g}" for k, (e, s) in res.items()})


def _ln_ref(z, gamma, beta, dy, eps):
    zr = z.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    mu = zr.mean(-1, keepdim=True)
    var = ((zr - mu) ** 2).mean(-1, keepdim=True)
    y = (zr - mu) / torch.sqrt(var + eps) * gr + br
    y.backward(dy.double())
    return zr.grad, gr.grad, br.grad


@pytest.mark.parametrize("form", ["sparse", "dense"])
@pytest.mark.parametrize("H", [256, 320, 512, 768, 1024])
def test_ln_bwd_dropout_on_cls_rows(form, H):
    """LN backward of the pruned layer (fp16 z, hidden dropout keyed by row * S): sparse = the LN2 form (fp32 dy_cls,
    cls_stride 1), dense = the LN1 form (bf16 dy).  dz, dzm = dz * mask / (1-p), dgamma, dbeta, dbias = colsum(dzm)."""
    from dpr_scale_b200 import ops
    from oracle import dropout as od
    R, S, eps = 333, 96, 1e-12
    g = torch.Generator().manual_seed(H + (1 if form == "dense" else 0))
    z = (torch.randn(R, H, generator=g) * 2 + 0.3).half()
    gamma = 1 + 0.1 * torch.randn(H, generator=g)
    beta = 0.1 * torch.randn(H, generator=g)
    _, stats, _ = ops.ln_fwd(z.cuda(), gamma.cuda(), beta.cuda(), eps)
    seed, layer = 0xD0D0 + H, 3
    dgamma, dbeta, dbias = (torch.zeros(H, device=DEV) for _ in range(3))
    site = _cls_site(seed, layer, 3, S)
    if form == "sparse":
        dy = torch.randn(R, H, generator=g)
        dz, dzm = ops.ln_bwd(None, z.cuda(), stats, gamma.cuda(), dgamma, dbeta, dbias, dy.cuda(), 1, P_DROP, site)
    else:
        dy = torch.randn(R, H, generator=g).to(torch.bfloat16)
        dz, dzm = ops.ln_bwd(dy.cuda(), z.cuda(), stats, gamma.cuda(), dgamma, dbeta, dbias, None, 1, P_DROP, site)
    torch.cuda.synchronize()
    rdz, rdg, rdb = _ln_ref(z, gamma, beta, dy, eps)
    keep = torch.from_numpy(od.keep_mask(R, H, P_DROP, seed, layer, 3, row_mul=S)).double()
    res = {}
    _gate("ln_dz", dz.cpu(), rdz, 2 ** -7, 1e-3, res)
    _gate("ln_dzm", dzm.cpu(), rdz * keep * od.scale(P_DROP), 2 ** -7, 1e-3, res)
    _gate("ln_dgamma", dgamma.cpu(), rdg, 2e-6, 1e-6, res)
    _gate("ln_dbeta", dbeta.cpu(), rdb, 2e-6, 1e-6, res)
    _gate("ln_dbias", dbias.cpu(), dzm.double().cpu().sum(0), 2e-6, 1e-6, res)
    print({k: f"{e:.3g}/{s:.3g}" for k, (e, s) in res.items()})


@pytest.mark.parametrize("H", [256, 768])
def test_ln_bwd_sparse_strided_dropout_zeroes_non_cls_rows(H):
    """The unpruned last layer's LN2 backward (DPRB_NO_CLS_PRUNE=1): fp32 dy_cls on rows t % S == 0 only, hidden
    dropout.  dz AND dzm must be written as exact zeros on every other row - the wgrad / dgrad GEMMs that follow read
    all T rows of dzm.  Both outputs start as a NaN sentinel."""
    from dpr_scale_b200 import ops
    from oracle import dropout as od
    nseq, S, eps = 9, 40, 1e-12
    T = nseq * S
    g = torch.Generator().manual_seed(H + 5)
    z = (torch.randn(T, H, generator=g) * 2 + 0.3).half()
    gamma = 1 + 0.1 * torch.randn(H, generator=g)
    beta = 0.1 * torch.randn(H, generator=g)
    _, stats, _ = ops.ln_fwd(z.cuda(), gamma.cuda(), beta.cuda(), eps)
    dy_cls = torch.randn(nseq, H, generator=g)
    seed, layer = 0xFACE + H, 0
    dgamma, dbeta, dbias = (torch.zeros(H, device=DEV) for _ in range(3))
    dz, dzm = ops.ln_bwd(None, z.cuda(), stats, gamma.cuda(), dgamma, dbeta, dbias, dy_cls.cuda(), S, P_DROP,
                         od.site_seed32(seed, layer, 3), dz=_sentinel((T, H)), dzm=_sentinel((T, H)))
    torch.cuda.synchronize()
    dy = torch.zeros(T, H)
    dy[::S] = dy_cls
    rdz, rdg, rdb = _ln_ref(z, gamma, beta, dy, eps)
    keep = torch.from_numpy(od.keep_mask(T, H, P_DROP, seed, layer, 3)).double()
    res = {}
    _gate("ln_dz", dz.cpu(), rdz, 2 ** -7, 1e-3, res)
    _gate("ln_dzm", dzm.cpu(), rdz * keep * od.scale(P_DROP), 2 ** -7, 1e-3, res)
    rest = torch.arange(T) % S != 0
    assert float(dz.cpu()[rest].float().abs().max()) == 0.0 and float(dzm.cpu()[rest].float().abs().max()) == 0.0
    _gate("ln_dgamma", dgamma.cpu(), rdg, 2e-6, 1e-6, res)
    _gate("ln_dbeta", dbeta.cpu(), rdb, 2e-6, 1e-6, res)
    _gate("ln_dbias", dbias.cpu(), dzm.double().cpu().sum(0), 2e-6, 1e-6, res)
    print({k: f"{e:.3g}/{s:.3g}" for k, (e, s) in res.items()})


# ================================================================== (c) the assembled pruned layer
ENC_CASES = [(H, S, p) for H in (256, 768) for S in (40, 300) for p in (0.0, P_DROP)]
ENC_IDS = [f"H{H}-S{S}-p{p:g}" for H, S, p in ENC_CASES]
N_SEQ, DROP_SEED = 5, 0x123456789ABCDEF
K_PRUNED = 2.0     # pruned error <= K_PRUNED * unpruned error + atol: per parameter tensor, per 32-row block of positions


def _enc_cfg(H):
    return dict(vocab_size=96, hidden_size=H, num_hidden_layers=1, num_attention_heads=H // 64, intermediate_size=4 * H,
                max_position_embeddings=320)


def _enc_case(H, S, p):
    """Encoder (one layer), tokens with mixed lengths (one of length 1) and the probe loss of one case."""
    from dpr_scale_b200.models.hf_model import HFEncoder
    enc = HFEncoder.from_config(_enc_cfg(H), dropout=p, seed=H + S)
    with torch.no_grad():                 # non-zero biases / LayerNorm parameters
        gen = torch.Generator().manual_seed(H * 3 + S)
        for prm in enc.parameters():
            prm.add_(0.05 * torch.randn(prm.shape, generator=gen))
    gen = torch.Generator().manual_seed(S)
    lens = torch.tensor([S, 1, S - 1, S // 2 + 3, S // 3])
    ids = torch.randint(3, 96, (N_SEQ, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    tokens = {"input_ids": ids * am, "token_type_ids": (torch.arange(S) >= S // 2).long().expand(N_SEQ, S) * am,
              "attention_mask": am}
    probe = torch.randn(N_SEQ, H, generator=gen)
    return enc, tokens, probe


def _enc_run(H, S, p):
    """pooled and every parameter gradient of the dprb encoder on one case (fixed dropout seed)."""
    enc, tokens, probe = _enc_case(H, S, p)
    enc = enc.cuda().train()
    enc.zero_grad()
    pooled, state = enc._run_forward(tokens, True, train_dropout=True, force_seed=DROP_SEED)
    enc._run_backward(state, probe.cuda().float())
    state.release()
    torch.cuda.synchronize()
    return {"pooled": pooled.cpu(), "last_dropout": enc.last_dropout,
            "grads": {k: v.grad.detach().cpu().clone() for k, v in enc.named_parameters() if v.grad is not None}}


def _unpruned_child(path):
    """Runs in a child process with DPRB_NO_CLS_PRUNE=1 (read once per process): every case, saved to `path`."""
    torch.save({ENC_IDS[i]: _enc_run(*c) for i, c in enumerate(ENC_CASES)}, path)


@pytest.fixture(scope="module")
def unpruned(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("unpruned") / "runs.pt")
    env = dict(os.environ, DPRB_NO_CLS_PRUNE="1")
    code = f"from tests.test_pruned_layer_gpu import _unpruned_child; _unpruned_child({path!r})"
    r = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return torch.load(path)


@pytest.mark.skipif(os.environ.get("DPRB_NO_CLS_PRUNE") is not None,
                    reason="DPRB_NO_CLS_PRUNE is set: this process cannot run the pruned layer to compare")
@pytest.mark.parametrize("H,S,p", ENC_CASES, ids=ENC_IDS)
def test_pruned_layer_matches_unpruned_and_float64(unpruned, H, S, p):
    from oracle import encoder as oenc
    from tests.test_dropout_gpu import _masks
    cid = f"H{H}-S{S}-p{p:g}"
    got = _enc_run(H, S, p)
    un = unpruned[cid]
    assert un["last_dropout"] == got["last_dropout"]
    enc, tokens, probe = _enc_case(H, S, p)
    masks = None
    if p:   # the masks of the run's dropout seed, replayed in the oracle
        masks = _masks(*got["last_dropout"], N_SEQ, S, H, H // 64, 1)
        masks = {"emb": masks["emb"].double(), 0: {k: v.double() for k, v in masks[0].items()}}
    sd = {k: v.detach().double().clone().requires_grad_(True) for k, v in enc.state_dict().items()}
    ocfg = {"layers": 1, "heads": H // 64, "ln_eps": 1e-12, "pad_id": 0, "roberta": False}
    ref = oenc.encode(sd, ocfg, tokens, dropout=masks)
    (ref * probe.double()).sum().backward()
    ref = ref.detach()
    scale = float(ref.abs().max())
    d_pool = _maxerr(got["pooled"], un["pooled"])
    print(cid, f"pooled pruned-vs-unpruned {d_pool:.3g} (scale {scale:.3g}); "
               f"vs float64: pruned {_maxerr(got['pooled'], ref):.3g} unpruned {_maxerr(un['pooled'], ref):.3g}")
    assert d_pool <= 2 ** -7 * scale + 1e-5, (d_pool, scale)
    worst = 0.0
    for name, g_pr in got["grads"].items():
        r = sd[name].grad
        if r is None:
            continue
        e_pr, e_un = _maxerr(g_pr, r), _maxerr(un["grads"][name], r)
        atol = 1e-5 * float(r.abs().max()) + 1e-9
        worst = max(worst, e_pr / max(e_un, 1e-30))
        print(cid, f"  {name}: pruned {e_pr:.3g} unpruned {e_un:.3g} scale {float(r.abs().max()):.3g}")
        assert e_pr <= K_PRUNED * e_un + atol, (name, e_pr, e_un, float(r.abs().max()))
        if name.endswith("position_embeddings.weight"):
            # Row j collects key j's dK / dV, so a per-key error shows here and not in a whole-tensor figure.  The rule
            # is applied per block of 32 rows (one lane chunk of the attention kernels: keys 32c .. 32c + 31) on the RMS
            # error: the error of a single row is one rounding error of dS_j times a fixed row vector, so per-row
            # pruned / unpruned ratios are ratios of two scalar rounding errors (measured up to 2.5 max-abs and 1.96
            # RMS over 300 rows), while a wrong or missing dK / dV of any key is of the size of the row itself.
            ep, eu = (g_pr.double() - r)[:S], (un["grads"][name].double() - r)[:S]
            worst_c = 0.0
            for c0 in range(0, S, 32):
                rp, ru = float(ep[c0:c0 + 32].pow(2).mean().sqrt()), float(eu[c0:c0 + 32].pow(2).mean().sqrt())
                tol = 1e-5 * float(r[c0:c0 + 32].abs().max()) + 1e-9
                worst_c = max(worst_c, rp / max(ru, 1e-30))
                assert rp <= K_PRUNED * ru + tol, ("position rows", c0, c0 + 32, rp, ru)
            print(cid, f"  position rows: worst pruned/unpruned RMS ratio of a 32-row block {worst_c:.3g}")
    print(cid, f"parameters: worst pruned/unpruned max-abs error ratio {worst:.3g}")
