"""The assembled encoder (csrc/encoder.cu) against float64, stage by stage: every activation the forward saves and every
stage of each layer's backward, each fed the GPU's own rounded inputs to that stage.

The forward and backward run as in training: ``HFEncoder._run_forward`` with save_for_backward, then ``_run_backward``
with ``bwd_chunk_layers = 1`` and a ``grad_sync`` hook, so dprb_encoder_bwd runs one layer per call ([L-1, L), ...,
[0, 1)) and the hook snapshots the backward scratch (gA = dx, gB = dz1, gB2 = dz1 * keep / (1 - p), gH = dhpre, gQKV),
the rebuilt lean tensors and that layer's gradients after each call.  The saved activations are read as typed views of
the caller's workspace at the offsets plan() carves (test_encoder_layout_cpu restates it and
holds the restatement to dprb_encoder_workspace_bytes).  Dropout multipliers come from dprb_dropout_mask (the pruned
layer: the full masks restricted to rows r * S).

u = 2^-24 (fp32), b = 2^-8 (bf16), h = 2^-11 (fp16); every gate is per element, |GPU - float64| <= bound:
  * GEMM stages (qkv, z1, hact / hpre, z2, gH, dx, dW*, the dropped / residual epilogues): an fp32 accumulation of K
    terms (K + 2) u sum|terms|, the dropout multiply and residual add one u each, then the 16-bit store:
    b |ref| + (1 + b) E (bf16) or h |ref| + (1 + h) E (fp16, the residual stream z1 / z2);
  * column sums (db1, dbo, dbqkv, dbeta, dgamma, the embedding tables) of N rows: (N + 4) u sum|terms|;
  * LayerNorm forward / backward: the bounds of test_train_heads_gpu (_ln_fwd_bounds, _ln_bwd_fp32) on the GPU's z and
    statistics; the fp16 residual copies rA / rB (never saved) are rebuilt as fp16 of the float64 LayerNorm of the
    GPU's z and statistics, allowed one fp16 ulp plus the fp32 LayerNorm error;
  * GELU: the epilogue's fitted CDF (common.cuh: |x Phi_fit - gelu| <= 3.0e-5, |gelu_fit' - gelu'| <= 1.25e-4, confirmed
    on a float64 restatement of gelu_and_grad2 in test_encoder_layout_cpu) plus |gelu'| <= 1.13 (|gelu''| <= 0.8)
    times the pre-activation's bound and 128 u (1 + |x|) for the MUFU approximations;
  * attention (ctx, lse, dqkv): the per-problem gates of gpu_checks.check_attention (ctx 2^-7 max + 1e-4, lse 1e-4,
    dq / dk / dv 2^-6 max + 1e-5 beyond the first-order bound of dS); the pruned layer's probabilities 1e-5 absolute;
  * dz2 and dctx are overwritten within a layer's backward: they are rebuilt in float64 from observed tensors and their
    bound (the bf16 store included) is carried to first order through each consumer (|e| |W|, the LayerNorm backward
    Jacobian r (|g e| + mean|g e| + |xhat| mean|g e xhat|), the softmax backward).
Exact: the lean re-run attention output equals full mode's saved ctx bit for bit; every saved forward activation except
hpre is bitwise the same in full and lean mode.  Negative controls feed the same checker a plausibly wrong reference and
require a ratio above 1.

Each test prints its worst error / gate per stage.  Worst ratios over every case, both modes and the unpruned child,
measured on an H100 80GB HBM3 (700 W limit):
  forward   embeddings out 0.99, mean 0.004, rstd 0.017; qkv 0.99; ctx 0.62, lse 0.010, pruned probs 0.001; z1 0.92;
            LayerNorm out 0.99 (bf16 stores: half an ulp approaches the gate by construction), mean 0.002, rstd 0.017;
            hact 0.98, hpre gelu' 0.98 / pre 0.99; z2 0.61; pooled 0.42; fwd_tokens' last layer within the same figures
  backward  dgamma2 0.29, dbeta2 0.007, db2 0.82, dW2 0.96, gH 0.55, db1 0.097, dW1 0.49, gB 0.65, gB2 0.60,
            dgamma1 0.62, dbeta1 0.49, dbo 0.007, dWo 0.47, dq / dk 0 beyond their first-order bound, dv 0.30,
            dbqkv 0.006, dWqkv 0.071, dx 0.99, rebuilt hact 0.96; embeddings dgamma 0.012, dbeta 0.010, word 0.058,
            position 0.043, token type 0.012
  controls  bf16 residual 3.7, FFN mask at the attention output 4e6, gB for dWo 7e4, CLS residual at stride H 1e6,
            another layer's x1 in dW1 2e5
"""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U, BF, HF = 2.0 ** -24, 2.0 ** -8, 2.0 ** -11
from tests.test_encoder_layout_cpu import DGELU_FIT, GELU_FIT, gelu64 as _gelu64, layout as _layout, views as _views
DROP_SEED = 0x0DDBA11C0FFEE123
P_DROP = 0.1

# id: (kind, H, heads, I, L, nseq, S, p)
CASES = {
    "tiny-S37": ("bert", 128, 2, 1288, 3, 6, 37, P_DROP),
    "tiny-S200-p0": ("bert", 128, 2, 1288, 2, 5, 200, 0.0),
    "h320-S200": ("bert", 320, 5, 1288, 3, 5, 200, P_DROP),
    "base-S128": ("bert", 768, 12, 3072, 3, 6, 128, P_DROP),
    "large-S256": ("roberta", 1024, 16, 4096, 2, 3, 256, P_DROP),
    "large-S512": ("roberta", 1024, 16, 4096, 2, 2, 512, P_DROP),
}


# ------------------------------------------------------------------ checker
class Ratios:
    """Worst |GPU - ref| / bound per stage; failures are collected so one run reports every stage."""

    def __init__(self):
        self.worst, self.bad = {}, []

    def add(self, name, ratio, detail=""):
        self.worst[name] = max(ratio, self.worst.get(name, 0.0))
        if not ratio <= 1.0:
            self.bad.append(f"{name}: {ratio:.3g}x gate {detail}")

    def check(self, name, got, ref, bound):
        got = got.detach().to("cuda", torch.float64)
        if not bool(torch.isfinite(got).all()):
            self.add(name, float("inf"), "(non-finite)")
            return
        err = (got - ref).abs()
        bound = torch.broadcast_to(bound, err.shape)
        ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
        self.add(name, ratio, f"({int((err > bound).sum())} of {err.numel()} elements)")

    def problems(self, name, got, ref, rtol, atol, bound=None):
        """check_attention's per-(sequence, head) gate: max|err| - bound of each problem within rtol max|ref| + atol."""
        got = got.double()
        if not bool(torch.isfinite(got).all()):
            self.add(name, float("inf"), "(non-finite)")
            return
        err = (got - ref).abs()
        if bound is not None:
            err = (err - bound).clamp_min(0)
        e, sc = err.amax(dim=(-2, -1)), ref.abs().amax(dim=(-2, -1))
        self.add(name, float((e / (rtol * sc + atol)).max()))

    def exact(self, name, got, want):
        same = torch.equal(got.contiguous().view(torch.uint8), want.contiguous().view(torch.uint8))
        self.add(name, 0.0 if same else float("inf"), "(not bitwise equal)")

    def report(self, tag):
        print(f"{tag}: " + ", ".join(f"{k} {v:.3f}" for k, v in self.worst.items()))

    def assert_ok(self):
        assert not self.bad, "; ".join(self.bad[:20])


def _f64(t):
    return t.detach().to("cuda", torch.float64)


def _mean(t):
    return t.mean(1, keepdim=True)


def _store(ref, e, fmt):
    return (BF if fmt == "bf16" else HF) * ref.abs() + (1 + (BF if fmt == "bf16" else HF)) * e


def _rowsum_bound(terms_abs, extra=4):
    return (terms_abs.shape[0] + extra) * U * terms_abs.sum(0)


def _ln_fwd(r, tag, Z, stats, g, be, eps, out16=None, mult=None):
    """LayerNorm forward on the GPU's z: stats and the 16-bit output; returns (out64 * mult, its fp32 bound) of the
    GPU's statistics' LayerNorm for rebuilding the residual copies."""
    from tests.test_train_heads_gpu import _ln_fwd_bounds
    P = Z.shape[1]
    mu = _mean(Z)
    rs = (_mean((Z - mu) ** 2) + eps).rsqrt()
    xh = (Z - mu) * rs
    e_mu, rel_r, e_out = _ln_fwd_bounds(Z.abs().sum(1, keepdim=True), mu, rs, xh, g, be, P)
    r.check(f"{tag}.mean", stats[:, :1], mu, e_mu)
    r.check(f"{tag}.rstd", stats[:, 1:], rs, rel_r * rs)
    m = 1.0 if mult is None else mult
    ref = (xh * g + be) * m
    e = e_out * m + U * ref.abs()
    if out16 is not None:
        r.check(f"{tag}.out", out16, ref, _store(ref, e, "bf16"))
    # the GPU's statistics' LayerNorm: what the fp16 residual copy rounds (5 fp32 roundings of the element)
    mg, rg = _f64(stats[:, :1]), _f64(stats[:, 1:])
    xg = (Z - mg) * rg
    refg = (xg * g + be) * m
    return refg, 5 * U * ((xg * g).abs() + be.abs()) * (m if mult is not None else 1.0) + U * refg.abs()


def _residual(refg, e, fmt="fp16"):
    """fp16 copy rebuilt from the float64 LayerNorm output; its bound allows one fp16 ulp plus the fp32 error."""
    dt = torch.float16 if fmt == "fp16" else torch.bfloat16
    q = refg.to(dt).double()
    ulp = (2.0 ** -10) * (refg.abs() + e) + 2.0 ** -24
    return q, ulp + e


def _ln_bwd(Z, stats, g, dy, e_dy=None):
    """float64 LayerNorm backward on the GPU's z and statistics: (xg, dz, fp32 bound of dz incl. the carried e_dy)."""
    from tests.test_train_heads_gpu import _ln_bwd_fp32
    P = Z.shape[1]
    mg, rg = _f64(stats[:, :1]), _f64(stats[:, 1:])
    xg = (Z - mg) * rg
    gd = g * dy
    s1, s2 = _mean(gd), _mean(gd * xg)
    dz = rg * (gd - s1 - xg * s2)
    e = _ln_bwd_fp32(rg, xg, gd, s1, s2, P)
    if e_dy is not None:
        ge = g.abs() * e_dy
        e = e + rg * (ge + _mean(ge) + xg.abs() * _mean(ge * xg.abs()))
    return xg, dz, e


# ------------------------------------------------------------------ attention references
def _attn_chunks(nseq, heads, S):
    step = max(1, (1 << 22) // (heads * S * S))
    return [(s0, min(nseq, s0 + step)) for s0 in range(0, nseq, step)]


def _split_qkv(qkv, n, S, heads):
    x = _f64(qkv).view(n, S, 3, heads, 64)
    return [x[:, :, i].transpose(1, 2) for i in range(3)]        # n, heads, S, 64


def _attn_fwd_check(r, tag, qkv, am, mult, ctx, lse, nseq, S, heads):
    for s0, s1 in _attn_chunks(nseq, heads, S):
        n = s1 - s0
        q, k, v = _split_qkv(qkv[s0 * S:s1 * S], n, S, heads)
        sc = q @ k.transpose(-1, -2) / 8.0
        sc = sc.masked_fill(am[s0:s1].view(n, 1, 1, S) == 0, float("-inf"))
        lse_r = torch.logsumexp(sc, -1)
        pm = torch.exp(sc - lse_r[..., None]) * mult[s0:s1]
        o = pm @ v
        c = _f64(ctx[s0 * S:s1 * S]).view(n, S, heads, 64).transpose(1, 2)
        r.problems(f"{tag}.ctx", c, o, 2 ** -7, 1e-4)
        r.problems(f"{tag}.lse", _f64(lse.view(nseq, heads, S)[s0:s1])[..., None], lse_r[..., None], 0.0, 1e-4)


def _attn_bwd_check(r, tag, qkv, am, mult, ctx, dctx, e_dctx, dqkv, nseq, S, heads):
    """gQKV of the full attention backward against float64 from the GPU's qkv and the float64 dctx (bound e_dctx)."""
    for s0, s1 in _attn_chunks(nseq, heads, S):
        n, r0, r1 = s1 - s0, s0 * S, s1 * S
        q, k, v = _split_qkv(qkv[r0:r1], n, S, heads)
        sc = q @ k.transpose(-1, -2) / 8.0
        sc = sc.masked_fill(am[s0:s1].view(n, 1, 1, S) == 0, float("-inf"))
        p = torch.softmax(sc, -1)
        m = mult[s0:s1]
        pm = p * m
        dO = dctx[r0:r1].view(n, S, heads, 64).transpose(1, 2)
        eO = e_dctx[r0:r1].view(n, S, heads, 64).transpose(1, 2)
        dp = (dO @ v.transpose(-1, -2)) * m
        edp = (eO @ v.abs().transpose(-1, -2)) * m
        ds = p * (dp - (p * dp).sum(-1, keepdim=True)) / 8.0
        c_got = _f64(ctx[r0:r1]).view(n, S, heads, 64).transpose(1, 2)
        dD = (dO.abs() * (c_got - pm @ v).abs()).sum(-1, keepdim=True) if S > 256 else 0.0
        A = p * (2 ** -12 * (dp.abs() + (p * dp.abs()).sum(-1, keepdim=True)) + dD
                 + edp + (p * edp).sum(-1, keepdim=True)) / 8.0
        got = _f64(dqkv[r0:r1]).view(n, S, 3, heads, 64)
        r.problems(f"{tag}.dq", got[:, :, 0].transpose(1, 2), ds @ k, 2 ** -6, 1e-5, A @ k.abs())
        r.problems(f"{tag}.dk", got[:, :, 1].transpose(1, 2), ds.transpose(-1, -2) @ q, 2 ** -6, 1e-5,
                   A.transpose(-1, -2) @ q.abs())
        r.problems(f"{tag}.dv", got[:, :, 2].transpose(1, 2), pm.transpose(-1, -2) @ dO, 2 ** -6, 1e-5,
                   pm.transpose(-1, -2) @ eO)


def _cls_attn(qkv, am, mult0, nseq, S, heads, dctx=None, e_dctx=None):
    """Query 0 of every sequence (the pruned layer): probs [n, heads, S], ctx [n, H]; with dctx also dq0 [n, H] and
    dk / dv [n*S, H] plus their first-order bounds from e_dctx."""
    H = heads * 64
    q, k, v = _split_qkv(qkv, nseq, S, heads)
    q0 = q[:, :, 0]                                                   # n, heads, 64
    s = torch.einsum("nhd,nhsd->nhs", q0, k) / 8.0
    s = s.masked_fill(am.view(nseq, 1, S) == 0, float("-inf"))
    p = torch.softmax(s, -1)
    pm = p * mult0
    ctx = torch.einsum("nhs,nhsd->nhd", pm, v).reshape(nseq, H)
    if dctx is None:
        return p, ctx
    dO, eO = dctx.view(nseq, heads, 64), e_dctx.view(nseq, heads, 64)
    dpm = torch.einsum("nhd,nhsd->nhs", dO, v) * mult0
    edp = torch.einsum("nhd,nhsd->nhs", eO, v.abs()) * mult0
    ds = p * (dpm - (p * dpm).sum(-1, keepdim=True)) / 8.0
    eds = p * (2 ** -12 * (dpm.abs() + (p * dpm.abs()).sum(-1, keepdim=True)) + edp
               + (p * edp).sum(-1, keepdim=True)) / 8.0
    dq0 = torch.einsum("nhs,nhsd->nhd", ds, k)
    edq0 = torch.einsum("nhs,nhsd->nhd", eds, k.abs())
    dk = ds[..., None] * q0[:, :, None, :]
    edk = eds[..., None] * q0.abs()[:, :, None, :]
    dv = pm[..., None] * dO[:, :, None, :]
    edv = pm[..., None] * eO[:, :, None, :]
    return p, ctx, (dq0, edq0), (dk, edk), (dv, edv)


# ------------------------------------------------------------------ model, tokens, masks
def _config(kind, H, heads, I, L, S):
    cfg = dict(vocab_size=96, hidden_size=H, num_hidden_layers=L, num_attention_heads=heads, intermediate_size=I,
               max_position_embeddings=S + 2)
    if kind == "roberta":
        cfg.update(model_type="roberta", pad_token_id=1, layer_norm_eps=1e-5, type_vocab_size=1)
    return cfg


def _model(kind, H, heads, I, L, S, p, lean):
    from dpr_scale_b200.models.hf_model import HFEncoder
    enc = HFEncoder.from_config(_config(kind, H, heads, I, L, S), dropout=p, seed=H + L)
    with torch.no_grad():                 # non-zero biases / LayerNorm parameters
        gen = torch.Generator().manual_seed(H * 7 + I)
        for prm in enc.parameters():
            prm.add_(0.02 * torch.randn(prm.shape, generator=gen))
    enc = enc.cuda().train()
    enc.lean_activations = lean
    return enc


def _tokens(kind, nseq, S):
    """Ragged lengths (one sequence full, one of length 1), pad ids past each length, ids from a 96-word vocabulary
    (every id repeats), BERT: two segments."""
    pad = 1 if kind == "roberta" else 0
    gen = torch.Generator().manual_seed(nseq * 1000 + S)
    lens = torch.randint(max(1, S // 4), S + 1, (nseq,), generator=gen)
    lens[0] = S
    if nseq > 2:
        lens[2] = 1
    ids = torch.randint(3, 96, (nseq, S), generator=gen)
    am = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    tok = {"input_ids": ids * am + pad * (1 - am), "attention_mask": am}
    if kind == "bert":
        tok["token_type_ids"] = (torch.arange(S) >= S // 2).long().expand(nseq, S) * am
    return tok


def _masks(p, seed, nseq, S, H, heads, L):
    """float64 multipliers keep / (1 - p) of the four dropout sites on the device (ones when p = 0)."""
    from dpr_scale_b200 import ops
    T = nseq * S
    if p == 0:
        one = torch.ones(T, H, dtype=torch.float64, device="cuda")
        att = torch.ones(nseq, heads, S, S, dtype=torch.float64, device="cuda")
        return {"emb": one, **{l: {"attn": att, "attn_out": one, "ffn_out": one} for l in range(L)}}
    sc = 1.0 / (1.0 - round(p * 65536) / 65536.0)
    m = lambda rows, cols, l, site: ops.dropout_mask(rows, cols, p, seed, l, site).double() * sc
    return {"emb": m(T, H, 0, 0), **{l: {"attn": m(nseq * heads * S, S, l, 1).view(nseq, heads, S, S),
                                         "attn_out": m(T, H, l, 2), "ffn_out": m(T, H, l, 3)} for l in range(L)}}


def _layer_weights(enc, l):
    """float64 copies of layer l's weights as the kernels read them: the bf16 shadow of the matrices, the fp32 master of
    biases and LayerNorm parameters."""
    lt = enc.transformer.layout
    H, I = enc.config["hidden_size"], enc.config["intermediate_size"]
    b0 = lt.off_layer0 + l * lt.layer_stride

    def g(arena, name, shape):
        o = b0 + lt.rel(name)
        return _f64(arena[o:o + math.prod(shape)].view(shape))

    sh, ms = enc.shadow, enc.master
    a, o = "attention.self.", "attention.output."
    return dict(wqkv=g(sh, a + "query.weight", (3 * H, H)), bqkv=g(ms, a + "query.bias", (3 * H,)),
                wo=g(sh, o + "dense.weight", (H, H)), bo=g(ms, o + "dense.bias", (H,)),
                ln1g=g(ms, o + "LayerNorm.weight", (H,)), ln1b=g(ms, o + "LayerNorm.bias", (H,)),
                w1=g(sh, "intermediate.dense.weight", (I, H)), b1=g(ms, "intermediate.dense.bias", (I,)),
                w2=g(sh, "output.dense.weight", (H, I)), b2=g(ms, "output.dense.bias", (H,)),
                ln2g=g(ms, "output.LayerNorm.weight", (H,)), ln2b=g(ms, "output.LayerNorm.bias", (H,)))


class Run:
    """One training forward + bucketed backward of a case, with everything the checks read (device tensors)."""

    def __init__(self, case, lean, pruned=True):
        from dpr_scale_b200 import ops
        kind, H, heads, I, L, nseq, S, p = CASES[case]
        self.case, self.lean, self.pruned = case, lean, pruned
        self.kind, self.H, self.heads, self.I, self.L, self.nseq, self.S, self.p = kind, H, heads, I, L, nseq, S, p
        self.T = nseq * S
        enc = self.enc = _model(kind, H, heads, I, L, S, p, lean)
        tok = _tokens(kind, nseq, S)
        self.eps = enc.config["layer_norm_eps"]
        ids, tt, pos, am, _, _ = enc._prep_tokens(tok)
        self.ids, self.tt, self.pos, self.am = ids.flatten(), tt.flatten(), pos.flatten(), am
        gen = torch.Generator().manual_seed(S + H)
        self.dpooled = (torch.randint(-2, 3, (nseq, H), generator=gen).float().exp2()
                        * (2 * torch.randint(0, 2, (nseq, H), generator=gen) - 1)).cuda()
        enc.zero_grad()
        pooled, state = enc._run_forward(tok, True, train_dropout=True, force_seed=DROP_SEED)
        torch.cuda.synchronize()
        self.pooled = pooled
        lay, nbytes = _layout(H, I, L, heads, nseq, S, 2 if lean else 1)
        assert state.b.workspace_bytes >= nbytes
        v = _views(state.ws, state.b.workspace, lay)
        self.fwd = {k: t.clone() for k, t in v.items() if k not in ("gA", "gB", "gB2", "gH", "gQKV")}
        p_run, seed = enc.last_dropout
        assert seed == DROP_SEED and (p_run > 0) == (p > 0)
        self.masks = _masks(p_run, seed, nseq, S, H, heads, L)
        # weights as the kernels read them: bf16 shadow for the matrices, fp32 master for the rest
        lt = enc.transformer.layout
        self.lw = [_layer_weights(enc, l) for l in range(L)]
        e = lambda name: enc.master[lt.by_name[name][1]:lt.by_name[name][1] + math.prod(lt.by_name[name][0])].view(lt.by_name[name][0])
        self.word, self.ptab, self.ttab = (e("embeddings." + n + "_embeddings.weight") for n in ("word", "position", "token_type"))
        self.embg, self.embb = (_f64(e("embeddings.LayerNorm." + n)) for n in ("weight", "bias"))
        # backward, one layer per call; the hook snapshots the scratch and the finished layer's gradients
        self.snap = {}
        layer_of = {}
        for l in range(L):
            layer_of[lt.off_layer0 + (l + 1) * lt.layer_stride] = l

        def grad_sync(e_, lo, hi):
            l = layer_of[hi]
            s = {k: v[k].clone() for k in ("gA", "gB", "gB2", "gH", "gQKV")}
            if lean:
                s["ctx_t"], s["hact_t"] = v["ctx_t"].clone(), v["hact_t"].clone()
            b0 = lt.off_layer0 + l * lt.layer_stride
            s["grads"] = enc.grads[b0:b0 + lt.layer_stride].clone()
            if l == 0:
                s["emb_grads"] = enc.grads[:lt.off_layer0].clone()
            self.snap[l] = s

        enc.bwd_chunk_layers, enc.grad_sync = 1, grad_sync
        enc._run_backward(state, self.dpooled)
        torch.cuda.synchronize()
        state.release()
        assert sorted(self.snap) == list(range(L))
        self.lt = lt

    def grad(self, l, name, shape):
        o = self.lt.rel(name)
        return self.snap[l]["grads"][o:o + math.prod(shape)].view(shape)

    def emb_grad(self, name):
        shape, o = self.lt.by_name[name]
        return self.snap[0]["emb_grads"][o:o + math.prod(shape)].view(shape)

    def is_pruned(self, l):
        return self.pruned and l == self.L - 1


# ------------------------------------------------------------------ forward stages
def _embed_check(run, r):
    f = run.fwd
    E = ((run.word[run.ids] + run.ttab[run.tt]) + run.ptab[run.pos]).double()      # the kernel's fp32 (w + t) + p
    refg, e = _ln_fwd(r, "emb", E, f["emb_stats"], run.embg, run.embb, run.eps, f["x0"], run.masks["emb"])
    return _residual(refg, e)


def _layer_fwd_check(run, r, l, x_in, rA, tamper=None, out_override=None):
    """Every saved activation of layer l from the GPU's inputs to each stage; returns the rebuilt rA of the next layer
    (and its bound).  rA = (fp16 rebuild, bound) of this layer's residual input."""
    f, w, m = run.fwd, run.lw[l], run.masks[l]
    slot = l
    T, H, S, nseq, heads = run.T, run.H, run.S, run.nseq, run.heads
    tag = f"L{l}"
    pruned = run.is_pruned(l)
    X = _f64(x_in)
    qkv = f[("qkv", slot)]
    ref = X @ w["wqkv"].T + w["bqkv"]
    r.check(f"{tag}.qkv", qkv, ref, _store(ref, (H + 2) * U * (X.abs() @ w["wqkv"].abs().T + w["bqkv"].abs()), "bf16"))
    am = run.am
    m_ao, m_ffn = m["attn_out"], m["ffn_out"]
    rArows, eArows = rA
    if tamper == "attn_out_mask_of_ffn":
        m_ao = m_ffn
    if pruned:
        R = nseq
        rows = slice(0, R)
        probs = f[("lse", slot)].view(nseq, heads, S)
        p, cref = _cls_attn(qkv, am, m["attn"][:, :, 0, :], nseq, S, heads)
        r.check(f"{tag}.probs", probs, p, torch.full_like(p, 1e-5))
        ctx = f[("ctx", slot)][:R]
        r.problems(f"{tag}.ctx", _f64(ctx).view(R, heads, 1, 64), cref.view(R, heads, 1, 64), 2 ** -7, 1e-4)
        m_ao, m_ffn = m_ao[::S], m_ffn[::S]
        rArows, eArows = rArows[::S], eArows[::S]
    else:
        R, rows = T, slice(0, T)
        # lean: the shared buffer holds the last layer's ctx only; layer l's is the backward's re-run (bitwise full's)
        ctx = run.snap[l]["ctx_t"] if run.lean else f[("ctx", slot)]
        _attn_fwd_check(r, tag, qkv, am, m["attn"], ctx, f[("lse", slot)], nseq, S, heads)
    C = _f64(ctx)
    v = C @ w["wo"].T + w["bo"]
    ref = v * m_ao + rArows
    E = (H + 2) * U * (C.abs() @ w["wo"].abs().T + w["bo"].abs()) * m_ao + U * (v * m_ao).abs() + eArows + U * ref.abs()
    r.check(f"{tag}.z1", f[("z1", slot)][rows], ref, _store(ref, E, "fp16"))
    Z1 = _f64(f[("z1", slot)][rows])
    refg, e = _ln_fwd(r, f"{tag}.ln1", Z1, f[("stats1", slot)][rows], w["ln1g"], w["ln1b"], run.eps, f[("x1", slot)][rows])
    rB, eB = _residual(refg, e)
    X1 = _f64(f[("x1", slot)][rows])
    pre = X1 @ w["w1"].T + w["b1"]
    Epre = (H + 2) * U * (X1.abs() @ w["w1"].abs().T + w["b1"].abs())
    g, d = _gelu64(pre)
    mufu = 128 * U * (1 + pre.abs())
    hact = f[("hact", slot)][rows]
    if not (run.lean and not pruned):      # lean: the shared buffer holds the last layer's values only
        r.check(f"{tag}.hact", hact, g, _store(g, GELU_FIT + 1.13 * Epre + mufu, "bf16"))
    if ("hpre", slot) in f:
        if run.lean:
            r.check(f"{tag}.hpre(pre)", f[("hpre", slot)][rows], pre, _store(pre, Epre, "bf16"))
        else:
            r.check(f"{tag}.hpre(gelu')", f[("hpre", slot)][rows], d, _store(d, DGELU_FIT + 0.8 * Epre + mufu, "bf16"))
    if not (run.lean and not pruned):
        Hc = _f64(hact)
        v = Hc @ w["w2"].T + w["b2"]
        ref = v * m_ffn + rB
        E = (run.I + 2) * U * (Hc.abs() @ w["w2"].abs().T + w["b2"].abs()) * m_ffn + U * (v * m_ffn).abs() + eB + U * ref.abs()
        r.check(f"{tag}.z2", f[("z2", slot)][rows], ref, _store(ref, E, "fp16"))
    Z2 = _f64(f[("z2", slot)][rows])
    out = f[("out", slot)][rows] if out_override is None else out_override
    refg, e = _ln_fwd(r, f"{tag}.ln2", Z2, f[("stats2", slot)][rows], w["ln2g"], w["ln2b"], run.eps, out)
    if l == run.L - 1 and out_override is None:
        cls = refg if pruned else refg[::S]
        r.check(f"{tag}.pooled", run.pooled, cls, e if pruned else e[::S])
    return _residual(refg, e, "bf16" if tamper == "residual_bf16" else "fp16")


def _forward_check(run, r, tamper=None, upto=None):
    rA = _embed_check(run, r)
    x = run.fwd["x0"]
    for l in range(run.L if upto is None else upto):
        rA = _layer_fwd_check(run, r, l, x, rA, tamper)
        x = run.fwd[("out", l)]
    return rA


# ------------------------------------------------------------------ backward stages
def _layer_bwd_check(run, r, l, tamper=None):
    f, w, m, sn = run.fwd, run.lw[l], run.masks[l], run.snap[l]
    T, H, I, S, nseq, heads, p = run.T, run.H, run.I, run.S, run.nseq, run.heads, run.p
    tag = f"L{l}"
    pruned = run.is_pruned(l)
    R = nseq if pruned else T
    rows = slice(0, R)
    m_ao, m_ffn = (m["attn_out"][::S], m["ffn_out"][::S]) if pruned else (m["attn_out"], m["ffn_out"])
    G = lambda name, shape: run.grad(l, name, shape)
    # upstream gradient of the layer output
    if l == run.L - 1:
        dy = _f64(run.dpooled)
        if not pruned:
            full = torch.zeros(T, H, dtype=torch.float64, device="cuda")
            full[::S] = dy
            dy = full
    else:
        dy = _f64(run.snap[l + 1]["gA"])
    # LN2 backward (dz2 is overwritten by LN1's backward: rebuilt, its bound carried)
    Z2 = _f64(f[("z2", l)][rows])
    xg2, dz2, e2 = _ln_bwd(Z2, f[("stats2", l)][rows], w["ln2g"], dy)
    r.check(f"{tag}.dln2g", G("output.LayerNorm.weight", (H,)), (dy * xg2).sum(0), _rowsum_bound((dy * xg2).abs()))
    r.check(f"{tag}.dln2b", G("output.LayerNorm.bias", (H,)), dy.sum(0), _rowsum_bound(dy.abs()))
    Edz2 = _store(dz2, e2, "bf16")                       # the bf16 gB the later stages read
    D2 = dz2 * m_ffn if p > 0 else dz2
    ED2 = _store(D2, e2 * m_ffn, "bf16") if p > 0 else Edz2
    r.check(f"{tag}.db2", G("output.dense.bias", (H,)), D2.sum(0), ED2.sum(0) + _rowsum_bound(D2.abs() + ED2))
    # FFN
    if run.lean and not pruned:
        Hc, pre16 = _f64(sn["hact_t"][rows]), _f64(f[("hpre", l)][rows])
        g16, _ = _gelu64(pre16)
        r.check(f"{tag}.hact(rebuilt)", Hc, g16, _store(g16, GELU_FIT + 128 * U * (1 + pre16.abs()), "bf16"))
    else:
        Hc = _f64(f[("hact", l)][rows])
    r.check(f"{tag}.dW2", G("output.dense.weight", (H, I)), D2.T @ Hc,
            ED2.T @ Hc.abs() + (R + 2) * U * ((D2.abs() + ED2).T @ Hc.abs()))
    if run.lean:
        _, gp = _gelu64(_f64(f[("hpre", l)][rows]))
        egp = DGELU_FIT + 128 * U * (1 + _f64(f[("hpre", l)][rows]).abs())
    else:
        gp, egp = _f64(f[("hpre", l)][rows]), 0.0
    DW = D2 @ w["w2"]
    eDW = ED2 @ w["w2"].abs() + (H + 2) * U * ((D2.abs() + ED2) @ w["w2"].abs())
    ref = DW * gp
    GH = sn["gH"][rows]
    r.check(f"{tag}.gH", GH, ref, _store(ref, eDW * gp.abs() + DW.abs() * egp + U * ref.abs(), "bf16"))
    GH = _f64(GH)
    r.check(f"{tag}.db1", G("intermediate.dense.bias", (I,)), GH.sum(0), _rowsum_bound(GH.abs()))
    X1 = _f64(f[("x1", 0 if tamper == "dw1_x1_of_other_layer" and l == 1 else l)][rows])
    r.check(f"{tag}.dW1", G("intermediate.dense.weight", (I, H)), GH.T @ X1, (R + 2) * U * (GH.abs().T @ X1.abs()))
    # dx1 = gH W1 + dz2 (overwritten: rebuilt) and the LN1 backward it feeds
    dx1 = GH @ w["w1"] + dz2
    edx1 = _store(dx1, (I + 2) * U * (GH.abs() @ w["w1"].abs() + dz2.abs() + Edz2) + Edz2, "bf16")
    Z1 = _f64(f[("z1", l)][rows])
    xg1, dz1, e1 = _ln_bwd(Z1, f[("stats1", l)][rows], w["ln1g"], dx1, edx1)
    r.check(f"{tag}.gB(dz1)", sn["gB"][rows], dz1, _store(dz1, e1, "bf16"))
    if p > 0:
        r.check(f"{tag}.gB2(dz1m)", sn["gB2"][rows], dz1 * m_ao, _store(dz1 * m_ao, e1 * m_ao, "bf16"))
    r.check(f"{tag}.dln1g", G("attention.output.LayerNorm.weight", (H,)), (dx1 * xg1).sum(0),
            (edx1 * xg1.abs()).sum(0) + _rowsum_bound((dx1 * xg1).abs() + edx1 * xg1.abs()))
    r.check(f"{tag}.dln1b", G("attention.output.LayerNorm.bias", (H,)), dx1.sum(0),
            edx1.sum(0) + _rowsum_bound(dx1.abs() + edx1))
    GL = _f64(sn["gB2" if p > 0 else "gB"][rows])
    r.check(f"{tag}.dbo", G("attention.output.dense.bias", (H,)), GL.sum(0), _rowsum_bound(GL.abs()))
    if run.lean and not pruned:
        if l in getattr(run, "full_ctx", {}):
            r.exact(f"{tag}.ctx(rebuilt)==full", sn["ctx_t"], run.full_ctx[l])
        C = _f64(sn["ctx_t"])
    else:
        C = _f64(f[("ctx", l)][rows])
    GLw = _f64(sn["gB"][rows]) if tamper == "dwo_from_gB" else GL
    r.check(f"{tag}.dWo", G("attention.output.dense.weight", (H, H)), GLw.T @ C, (R + 2) * U * (GLw.abs().T @ C.abs()))
    # dctx = gLin Wo (overwritten by dqkv's producer: rebuilt) and the attention backward
    dctx = GL @ w["wo"]
    edctx = _store(dctx, (H + 2) * U * (GL.abs() @ w["wo"].abs()), "bf16")
    qkv = f[("qkv", l)]
    GQ = sn["gQKV"]
    if pruned:
        _, _, (dq0, edq0), (dk, edk), (dv, edv) = _cls_attn(qkv, run.am, m["attn"][:, :, 0, :], nseq, S, heads, dctx, edctx)
        got = _f64(GQ).view(nseq, S, 3, heads, 64)
        r.problems(f"{tag}.dq0", got[:, 0, 0][:, :, None], dq0[:, :, None], 2 ** -7, 1e-5, edq0[:, :, None])
        r.problems(f"{tag}.dk", got[:, :, 1].transpose(1, 2), dk, 2 ** -7, 1e-5, edk)
        r.problems(f"{tag}.dv", got[:, :, 2].transpose(1, 2), dv, 2 ** -7, 1e-5, edv)
        r.add(f"{tag}.dq_rows>0==0", 0.0 if float(got[:, 1:, 0].abs().max()) == 0.0 else float("inf"))
    else:
        ctx = sn["ctx_t"] if run.lean else f[("ctx", l)]
        _attn_bwd_check(r, tag, qkv, run.am, m["attn"], ctx, dctx, edctx, GQ, nseq, S, heads)
    GQ = _f64(GQ)
    r.check(f"{tag}.dbqkv", G("attention.self.query.bias", (3 * H,)), GQ.sum(0), _rowsum_bound(GQ.abs()))
    X = _f64(run.fwd["x0"] if l == 0 else run.fwd[("out", l - 1)])
    r.check(f"{tag}.dWqkv", G("attention.self.query.weight", (3 * H, H)), GQ.T @ X, (T + 2) * U * (GQ.abs().T @ X.abs()))
    # dx = dqkv Wqkv + dz1 (the pruned layer: dz1 added on the CLS rows r * S only)
    Y = GQ @ w["wqkv"]
    eY = (3 * H + 2) * U * (GQ.abs() @ w["wqkv"].abs())
    B = _f64(sn["gB"][rows])
    if pruned:
        # gA = bf16(dqkv Wqkv), then add_rows: row r * S += dz1[r] with a second bf16 rounding
        ref, bound = Y.clone(), _store(Y, eY, "bf16")
        cls = torch.arange(R, device="cuda") * (1 if tamper == "cls_residual_stride_H" else S)
        new = Y[cls] + B
        ref[cls] = new
        bound[cls] = _store(new, bound[cls] + U * new.abs(), "bf16")
    else:
        ref = Y + B
        bound = _store(ref, eY + (3 * H + 2) * U * B.abs(), "bf16")
    r.check(f"{tag}.gA(dx)", sn["gA"], ref, bound)


def _embed_bwd_check(run, r):
    H = run.H
    dy = _f64(run.snap[0]["gA"]) * run.masks["emb"]
    E = ((run.word[run.ids] + run.ttab[run.tt]) + run.ptab[run.pos]).double()
    xg, dz, e = _ln_bwd(E, run.fwd["emb_stats"], run.embg, dy)
    r.check("emb.dln_g", run.emb_grad("embeddings.LayerNorm.weight"), (dy * xg).sum(0), _rowsum_bound((dy * xg).abs()))
    r.check("emb.dln_b", run.emb_grad("embeddings.LayerNorm.bias"), dy.sum(0), _rowsum_bound(dy.abs()))
    for name, idx, table in (("word", run.ids, run.word), ("position", run.pos, run.ptab),
                             ("token_type", run.tt, run.ttab)):
        n = table.shape[0]
        ref = torch.zeros(n, H, dtype=torch.float64, device="cuda").index_add_(0, idx, dz)
        ea = torch.zeros_like(ref).index_add_(0, idx, e)
        aa = torch.zeros_like(ref).index_add_(0, idx, dz.abs() + e)
        cnt = torch.bincount(idx, minlength=n).double()[:, None]
        r.check(f"emb.d{name}", run.emb_grad(f"embeddings.{name}_embeddings.weight"), ref, ea + (cnt + 4) * U * aa)


def _backward_check(run, r, tamper=None):
    for l in range(run.L - 1, -1, -1):
        _layer_bwd_check(run, r, l, tamper)
    _embed_bwd_check(run, r)


# ------------------------------------------------------------------ tests
_RUNS = {}


def _pair(case):
    """(full, lean) runs of a case, same weights, tokens and dropout seed (cached for the module)."""
    if case not in _RUNS:
        _RUNS.clear()
        full = Run(case, lean=False)
        lean = Run(case, lean=True)
        lean.full_ctx = {l: full.fwd[("ctx", l)] for l in range(full.L - 1)}
        _RUNS[case] = (full, lean)
    return _RUNS[case]


def _check_case(case, pruned=True):
    full, lean = (_pair(case) if pruned else (Run(case, False, pruned), Run(case, True, pruned)))
    if not pruned:
        lean.full_ctx = {l: full.fwd[("ctx", l)] for l in range(full.L)}
    out = []
    for run in (full, lean):
        r = Ratios()
        _forward_check(run, r)
        _backward_check(run, r)
        mode = "lean" if run.lean else "full"
        r.report(f"{case} {mode}{'' if pruned else ' unpruned'}")
        out.append(r)
    # full vs lean: every saved forward activation but hpre (and the shared ctx / hact buffers) bitwise
    r = Ratios()
    for key, t in full.fwd.items():
        name = key[0] if isinstance(key, tuple) else key
        if name in ("hpre", "ctx", "hact", "rA", "rB"):
            continue
        if pruned and isinstance(key, tuple) and key[1] == full.L - 1 and name != "qkv" and name != "lse":
            lean_t, t = lean.fwd[key][:full.nseq], t[:full.nseq]      # the pruned layer writes its R = nseq rows
        else:
            lean_t = lean.fwd[key]
        r.exact(f"lean==full {key}", lean_t, t)
    last = full.L - 1
    R = full.nseq if pruned else full.T
    r.exact("lean==full ctx(last)", lean.fwd["ctx_t"][:R], full.fwd[("ctx", last)][:R])
    r.exact("lean==full hact(last)", lean.fwd["hact_t"][:R], full.fwd[("hact", last)][:R])
    r.exact("lean==full pooled", lean.pooled, full.pooled)
    out.append(r)
    for x in out:
        x.assert_ok()


@pytest.mark.skipif(os.environ.get("DPRB_NO_CLS_PRUNE") is not None, reason="DPRB_NO_CLS_PRUNE is set")
@pytest.mark.parametrize("case", list(CASES))
def test_encoder_stages_match_float64(case):
    _check_case(case)


def _unpruned_child(case):
    _check_case(case, pruned=False)


def test_unpruned_last_layer_stages_match_float64():
    """DPRB_NO_CLS_PRUNE=1 (read once per process): the last layer runs on every row, in a child process."""
    env = dict(os.environ, DPRB_NO_CLS_PRUNE="1")
    code = "from tests.test_encoder_stages_gpu import _unpruned_child; _unpruned_child('tiny-S37')"
    p = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    print(p.stdout[-4000:])
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]


def test_fwd_tokens_last_layer_matches_float64():
    """dprb_encoder_fwd_tokens (save = 0: two slots, layer l in slot l & 1; eval): the last layer's saved activations
    in slot (L - 1) & 1 and the caller's tokens buffer, from the previous layer's output in the other slot.  The last
    layer is never pruned here."""
    from types import SimpleNamespace
    from dpr_scale_b200.models.citadel_models.colbert_model import encode_tokens
    kind, H, heads, I, L, nseq, S, _ = CASES["h320-S200"]
    enc = _model(kind, H, heads, I, L, S, 0.0, False).eval()
    tok = _tokens(kind, nseq, S)
    hidden, am, _, _ = encode_tokens(enc, tok)
    torch.cuda.synchronize()
    ws = enc._ws_cache[torch.cuda.current_stream().cuda_stream]
    v = _views(ws, (ws.data_ptr() + 255) & ~255, _layout(H, I, L, heads, nseq, S, 0)[0])
    cur, prev = (L - 1) & 1, (L - 2) & 1
    lw = _layer_weights(enc, L - 1)
    run = SimpleNamespace(L=L, H=H, I=I, S=S, nseq=nseq, heads=heads, T=nseq * S, p=0.0, lean=False,
                          eps=enc.config["layer_norm_eps"], am=am, masks=_masks(0.0, 0, nseq, S, H, heads, L),
                          is_pruned=lambda l: False, pooled=None, lw={L - 1: lw},
                          fwd={(k[0], L - 1): t for k, t in v.items() if isinstance(k, tuple) and k[1] == cur})
    r = Ratios()
    # the last layer's residual input: the fp16 rebuild of the previous layer's LayerNorm (the other slot)
    wp = _layer_weights(enc, L - 2)
    refg, e = _ln_fwd(r, f"L{L - 2}.ln2", _f64(v[("z2", prev)]), v[("stats2", prev)], wp["ln2g"], wp["ln2b"],
                      run.eps, v[("out", prev)])
    _layer_fwd_check(run, r, L - 1, v[("out", prev)], _residual(refg, e), out_override=hidden)
    r.report("fwd_tokens h320-S200")
    r.assert_ok()


# ------------------------------------------------------------------ negative controls
CONTROLS = {   # tamper: the stage that must see it
    "residual_bf16": "L1.z1",
    "attn_out_mask_of_ffn": "L0.z1",
    "dwo_from_gB": "L0.dWo",
    "cls_residual_stride_H": "L2.gA(dx)",
    "dw1_x1_of_other_layer": "L1.dW1",
}


@pytest.mark.skipif(os.environ.get("DPRB_NO_CLS_PRUNE") is not None, reason="DPRB_NO_CLS_PRUNE is set")
@pytest.mark.parametrize("tamper", list(CONTROLS))
def test_negative_control_exceeds_its_gate(tamper):
    """A plausibly wrong host-side reference (the library and device are untouched) must put its stage over the gate."""
    full, _ = _pair("tiny-S37")
    r = Ratios()
    if tamper in ("residual_bf16", "attn_out_mask_of_ffn"):
        _forward_check(full, r, tamper)
    else:
        _backward_check(full, r, tamper)
    stage = CONTROLS[tamper]
    print(f"control {tamper}: {stage} {r.worst[stage]:.3g}x gate")
    assert r.worst[stage] > 1.0
