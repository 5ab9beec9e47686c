"""The trainable heads on top of the encoder against float64: HFEncoder's projection (``_ProjectFn``: Linear +
LayerNorm, eps = nn.LayerNorm's 1e-5) and the cross-encoder's grouped cross-entropy head (``_GroupCE``), at the widths
and row counts they accept, plus the autograd glue around them.

u = 2^-24 (fp32 unit roundoff), b = 2^-8 (bf16), |A||B| a product of magnitudes, K the terms of a sum.  Every gate is
per element: |GPU - float64| <= bound, with the bound derived as below (no cosine, no global rel-L2).

1. Stage by stage.  Each stage's float64 reference is fed the GPU's own rounded inputs to that stage, read from
   ``out.grad_fn.saved_tensors`` (x16, w16, z, stats; dpre, drop_in) or, for the projection's dz, from the ln_bwd call
   of its backward.
   * an fp32 GEMM or column sum with K terms, split-K atomics included: (K + 2) u sum|terms|;
   * a bf16 store on top of an fp32 bound E: b |ref| + (1 + b) E;
   * LayerNorm forward on the GPU's z (P columns, fp32 statistics): mean within E_mu = u (sum|z| + |mu|); rstd within
     rel_r = (P + 12) u + (E_mu r)^2 / 2 relative (P-term sums, rsqrtf's 2 ulp); out within
     |g| r E_mu + (rel_r + 3u) |g xhat| + u |out|;
   * LayerNorm backward on the GPU's z and statistics: r (u sum|g dy| + (P + 5) u mean|g dy xhat| |xhat|
     + 6u (|g dy| + |s1| + |xhat s2|)) before the bf16 store; dgamma (N + 4) u sum|dy xhat|, dbeta and dbias (N + 1) u;
   * the group CE kernel: tanhf within 4u |t|; logits (H + 2) u (sum|t w| + |b|) plus the propagated pre-activation
     error; softmax probabilities (G + 8) u p; 1 - t^2 within 10u absolute; dpre 3u relative before its bf16 store.
2. End to end against float64 autograd of the head (oracle.encoder.layer_norm, oracle.cross_encoder_train.head_ce) on
   the fp32 input leaf: the input and the weight are each rounded to bf16 (b relative), and that error, with the stage
   bounds above, is carried through the head to first order with the magnitudes of its exact Jacobians (LayerNorm:
   |g| r (e_i + mean e + |xhat_i| mean(|xhat| e)); softmax: p_n (e_n + sum_m p_m e_m); tanh: (1 - t^2) e).

Glue: a stride-0 (out.sum()), non-contiguous ((out.t() @ M).sum()) and scaled (0.37 * loss) upstream gradient; the
encoder body receives bitwise the head's dx; a second backward with retain_graph=True gives the same gradients; the
eval-mode group_ce and CrossEncoder.forward give the same logits.  Each test prints its worst error / gate per tensor.

Worst error / gate measured on an H100 80GB HBM3 (700 W limit), over every case of each sweep:
  projection stages     z 0.99, dz 1.00 (bf16 stores: half an ulp reaches b |x|, so these approach 1 by
                        construction), mean 0.01, rstd 0.18, out 0.14, dgamma 0.33, dbias 0.10, dW 0.46, dx 0.20
  projection end to end out 0.13, dgamma 0.04, dbias 0.17, dW 0.14, dx 0.19; the glue cases stay below 0.14
  group CE stages       x16 1.00 and dpre 0.98 (bf16 stores), logits 0.001, dW_dense 0.37, db_dense 0.08, dx 0.011,
                        loss, dW_out and db_out below 0.001
  group CE end to end   p = 0: logits 0.013, dW_dense 0.011, dx 0.021, dW_out 0.008;
                        p = 0.1: logits 0.012, dW_dense 0.067, dx 0.030, dW_out 0.013
The head's gradients sit at rel-L2 <= 8.6e-3 (dx 8.5e-3) without dropout and <= 8.4e-3 (dx 6.4e-3) with it, except the
dense bias gradient at p = 0 (3.0e-2 against 8.4e-3): each group's softmax gradient sums to zero, so that column sum
cancels, and dropout masks break the cancellation.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
BF = 2.0 ** -8
EPS = 1e-5          # nn.LayerNorm's default: HFEncoder's project[1].eps
SCALE = 0.37
SCALE32 = float(torch.tensor(SCALE, dtype=torch.float32))   # what autograd hands backward
SEED = 0x5EED

# (N rows, H, P): every P with a small and a large N; P = 8 and P = 776 with H = 1024
PROJ_CASES = [(1, 1024, 8), (8200, 1024, 8), (2, 128, 16), (1000, 768, 16), (7, 768, 32), (8200, 128, 32),
              (64, 1024, 64), (1000, 128, 64), (65, 768, 120), (1000, 1024, 120), (129, 128, 128), (8200, 768, 128),
              (1, 768, 200), (1000, 128, 200), (2, 1024, 256), (1000, 768, 256), (7, 128, 320), (8200, 1024, 320),
              (65, 768, 768), (1000, 1024, 768), (129, 1024, 776), (1000, 768, 776), (64, 768, 1024),
              (8200, 1024, 1024)]
# (B groups, G pairs per group, H): every B x G, H cycling through 128 / 768 / 1024
CE_CASES = [(B, G, H) for i, (B, G) in enumerate((B, G) for B in (1, 3, 37) for G in (2, 7, 64))
            for H in ((128, 768, 1024)[i % 3],)]


def _f64(t):
    return t.detach().to("cuda", torch.float64)


def _check(ratios, name, got, ref, bound):
    got = _f64(got)
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite values"
    err = (got - ref).abs()
    bound = torch.broadcast_to(bound, err.shape)
    ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    ratios[name] = max(ratio, ratios.get(name, 0.0))
    over = err > bound
    assert not bool(over.any()), f"{name}: {int(over.sum())} of {err.numel()} elements over the gate (worst {ratio:.3g}x)"


def _report(case, ratios, extra=""):
    print(f"{case}: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()) + extra)


def _mean(t):
    return t.mean(1, keepdim=True)


# ------------------------------------------------------------------ projection: Linear + LayerNorm
def _proj_inputs(N, H, P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, generator=g)
    x[1::3] *= 1e-3 / (0.02 * H ** 0.5)          # these rows' z has a standard deviation near 1e-3: eps matters
    W = 0.02 * torch.randn(P, H, generator=g)     # HFEncoder's init of the projection
    b = 1e-3 * torch.randn(P, generator=g)
    gamma = 1.0 + 0.1 * torch.randn(P, generator=g)
    beta = 0.1 * torch.randn(P, generator=g)
    # upstream gradient of +-2^k: exact in fp32 after any scaling by a float32 factor
    R = torch.randint(-2, 3, (N, P), generator=g).float().exp2() * (2 * torch.randint(0, 2, (N, P), generator=g) - 1)
    return x, W, b, gamma, beta, R


def _proj_forward(x, W, b, gamma, beta):
    from dpr_scale_b200.models.hf_model import _ProjectFn
    leaves = [t.cuda().requires_grad_(True) for t in (x, W, b, gamma, beta)]
    return leaves, _ProjectFn.apply(*leaves, EPS)


def _ln_fwd_bounds(zabs_sum, mu, r, xh, g, be, P):
    """(E_mu, rel_r, out bound) of the fp32 LayerNorm forward (docstring, section 1)."""
    e_mu = U * (zabs_sum + mu.abs())
    rel_r = (P + 12) * U + 0.5 * (e_mu * r) ** 2
    out = xh * g + be
    return e_mu, rel_r, g.abs() * r * e_mu + (rel_r + 3 * U) * (xh * g).abs() + U * out.abs()


def _ln_bwd_fp32(r, xh, gd, s1, s2, P):
    """Bound of the fp32 LayerNorm backward before its bf16 store (docstring, section 1)."""
    return r * (U * gd.abs().sum(1, keepdim=True) + (P + 5) * U * _mean((gd * xh).abs()) * xh.abs()
                + 6 * U * (gd.abs() + s1.abs() + (xh * s2).abs()))


@pytest.mark.parametrize("N,H,P", PROJ_CASES)
def test_projection_stages_match_float64(N, H, P, monkeypatch):
    from dpr_scale_b200 import ops
    x, W, b, gamma, beta, R = _proj_inputs(N, H, P, N * 7 + H + P)
    leaves, out = _proj_forward(x, W, b, gamma, beta)
    x16, w16, z, stats, _ = out.grad_fn.saved_tensors
    seen = []
    real_ln_bwd = ops.ln_bwd

    def ln_bwd(*a, **k):
        dz = real_ln_bwd(*a, **k)
        seen.append(dz)
        return dz

    monkeypatch.setattr(ops, "ln_bwd", ln_bwd)
    out.backward(R.cuda())
    torch.cuda.synchronize()
    assert len(seen) == 1
    X, Wt, Z, b64, g64, be64, d = (_f64(t) for t in (x16, w16, z, b, gamma, beta, R))
    r = {}
    # Linear: z = bf16(x16 w16^T + b)
    zr = X @ Wt.T + b64
    e = (H + 2) * U * (X.abs() @ Wt.abs().T + b64.abs())
    _check(r, "z", Z, zr, BF * zr.abs() + (1 + BF) * e)
    # LayerNorm forward on the GPU's z
    mu = _mean(Z)
    rs = (_mean((Z - mu) ** 2) + EPS).rsqrt()
    xh = (Z - mu) * rs
    e_mu, rel_r, e_out = _ln_fwd_bounds(Z.abs().sum(1, keepdim=True), mu, rs, xh, g64, be64, P)
    _check(r, "mean", stats[:, :1], mu, e_mu)
    _check(r, "rstd", stats[:, 1:], rs, rel_r * rs)
    _check(r, "out", out, xh * g64 + be64, e_out)
    # LayerNorm backward on the GPU's z and statistics
    mg, rg = _f64(stats[:, :1]), _f64(stats[:, 1:])
    xg = (Z - mg) * rg
    gd = g64 * d
    s1, s2 = _mean(gd), _mean(gd * xg)
    dzr = rg * (gd - s1 - xg * s2)
    _check(r, "dz", seen[0], dzr, BF * dzr.abs() + (1 + BF) * _ln_bwd_fp32(rg, xg, gd, s1, s2, P))
    D = _f64(seen[0])
    _check(r, "dgamma", leaves[3].grad, (d * xg).sum(0), (N + 4) * U * (d * xg).abs().sum(0))
    _check(r, "dbeta", leaves[4].grad, d.sum(0), (N + 1) * U * d.abs().sum(0))
    _check(r, "dbias", leaves[2].grad, D.sum(0), (N + 1) * U * D.abs().sum(0))
    # wgrad (split-K) and dgrad GEMMs on the GPU's dz
    _check(r, "dW", leaves[1].grad, D.T @ X, (N + 2) * U * (D.abs().T @ X.abs()))
    _check(r, "dx", leaves[0].grad, D @ Wt, (P + 2) * U * (D.abs() @ Wt.abs()))
    _report(f"projection stages N={N} H={H} P={P}", r)


def _proj_end_to_end(r, leaves, out, x, W, b, gamma, beta, d):
    """Check the GPU's out and gradients against float64 autograd at the fp32 inputs, upstream gradient d (float64)."""
    from oracle.encoder import layer_norm
    N, H = x.shape
    P = W.shape[0]
    x, W, b, gamma, beta = (_f64(t).requires_grad_(True) for t in (x, W, b, gamma, beta))
    ref = layer_norm(x @ W.T + b, gamma, beta, EPS)
    ref.backward(d)
    with torch.no_grad():
        A = x.abs() @ W.abs().T
        z = x @ W.T + b
        e_acc = BF * (2 + BF) * A + (H + 2) * U * ((1 + BF) ** 2 * A + b.abs())
        Ez = e_acc + BF * (z.abs() + e_acc)
        mu = _mean(z)
        rs = (_mean((z - mu) ** 2) + EPS).rsqrt()
        xh = (z - mu) * rs
        g = gamma
        e_mu, rel_r, e_out32 = _ln_fwd_bounds((z.abs() + Ez).sum(1, keepdim=True), mu, rs, xh, g, beta, P)
        rho = rs * _mean(xh.abs() * Ez) + rel_r                              # relative error of rstd
        Exh = rs * (Ez + _mean(Ez) + e_mu) + xh.abs() * rho
        _check(r, "out", out, ref.detach(), g.abs() * Exh + e_out32)
        gd = g * d
        s1, s2 = _mean(gd), _mean(gd * xh)
        dz = rs * (gd - s1 - xh * s2)
        Edz = (dz.abs() * rho + rs * (Exh * s2.abs() + xh.abs() * _mean(gd.abs() * Exh))
               + _ln_bwd_fp32(rs, xh, gd, s1, s2, P))
        Edz = Edz + BF * (dz.abs() + Edz)
        Dm, Xm, Wm = dz.abs() + Edz, (1 + BF) * x.abs(), (1 + BF) * W.abs()
        _check(r, "dgamma", leaves[3].grad, gamma.grad,
               (d.abs() * Exh).sum(0) + (N + 4) * U * (d.abs() * (xh.abs() + Exh)).sum(0))
        _check(r, "dbeta", leaves[4].grad, beta.grad, (N + 1) * U * d.abs().sum(0))
        _check(r, "dbias", leaves[2].grad, b.grad, Edz.sum(0) + (N + 1) * U * Dm.sum(0))
        _check(r, "dW", leaves[1].grad, W.grad,
               Edz.T @ Xm + BF * (dz.abs().T @ x.abs()) + (N + 2) * U * (Dm.T @ Xm))
        _check(r, "dx", leaves[0].grad, x.grad, Edz @ Wm + BF * (dz.abs() @ W.abs()) + (P + 2) * U * (Dm @ Wm))


@pytest.mark.parametrize("N,H,P", PROJ_CASES)
def test_projection_end_to_end_matches_float64(N, H, P):
    x, W, b, gamma, beta, R = _proj_inputs(N, H, P, N * 7 + H + P)
    leaves, out = _proj_forward(x, W, b, gamma, beta)
    out.backward(R.cuda())
    torch.cuda.synchronize()
    r = {}
    _proj_end_to_end(r, leaves, out, x, W, b, gamma, beta, _f64(R))
    _report(f"projection end to end N={N} H={H} P={P}", r)


@pytest.mark.parametrize("upstream", ["sum", "transposed", "scaled"])
@pytest.mark.parametrize("N,H,P", [(65, 768, 120), (1000, 128, 776)])
def test_projection_upstream_gradients(N, H, P, upstream):
    """A stride-0, a non-contiguous and a scaled upstream gradient give the float64 gradients, and dx bitwise equals
    the one of the same upstream gradient given as a dense contiguous tensor."""
    x, W, b, gamma, beta, R = _proj_inputs(N, H, P, 31 * N + P)
    M = torch.randint(-4, 5, (N, 3), generator=torch.Generator().manual_seed(N)).float() / 4
    leaves, out = _proj_forward(x, W, b, gamma, beta)
    if upstream == "sum":
        loss, d = out.sum(), torch.ones(N, P)
    elif upstream == "transposed":
        loss, d = (out.t() @ M.cuda()).sum(), M.sum(1, keepdim=True).expand(N, P)
    else:
        s = torch.tensor(SCALE, dtype=torch.float32)
        loss, d = s.cuda() * (out * R.cuda()).sum(), R * s                 # exact: R holds +-2^k
    loss.backward()
    torch.cuda.synchronize()
    r = {}
    _proj_end_to_end(r, leaves, out, x, W, b, gamma, beta, _f64(d))
    dense, out2 = _proj_forward(x, W, b, gamma, beta)
    out2.backward(d.contiguous().cuda())
    torch.cuda.synchronize()
    assert torch.equal(leaves[0].grad, dense[0].grad)
    _report(f"projection upstream={upstream} N={N} H={H} P={P}", r)


def test_projection_second_backward_gives_the_same_gradients():
    x, W, b, gamma, beta, R = _proj_inputs(129, 768, 200, 3)
    leaves, out = _proj_forward(x, W, b, gamma, beta)
    loss = SCALE * (out * R.cuda()).sum()
    loss.backward(retain_graph=True)
    first = [t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    loss.backward()
    torch.cuda.synchronize()
    assert torch.equal(leaves[0].grad, first[0])                    # dz and the dgrad GEMM are deterministic
    r = {}
    _proj_end_to_end(r, leaves, out, x, W, b, gamma, beta, _f64(R) * SCALE32)
    _report("projection second backward", r)


# ------------------------------------------------------------------ cross-encoder head: grouped cross-entropy
def _ce_inputs(B, G, H, seed):
    g = torch.Generator().manual_seed(seed)
    N = B * G
    cls = torch.randn(N, H, generator=g)
    Wd = 0.02 * torch.randn(H, H, generator=g)
    bd = 0.02 * torch.randn(H, generator=g)
    Wo = 0.4 * torch.randn(1, H, generator=g)          # 20x the 0.02 init, as the model tests scale it
    bo = 0.1 * torch.randn(1, generator=g)
    labels = torch.randint(0, G, (B,), generator=g)
    return cls, Wd, bd, Wo, bo, labels


def _ce_masks(kind, N, H, p):
    """The head's replayed dropout multipliers (float64 [N, H]): site 4 after tanh, site 5 (RoBERTa) before the dense
    layer."""
    from dpr_scale_b200 import ops
    from dpr_scale_b200.models.citadel_models.cross_encoder import _keep_scale
    one = torch.ones(N, H, dtype=torch.float64, device="cuda")
    if p == 0:
        return one, one
    mh = _f64(ops.dropout_mask(N, H, p, SEED, 0, ops.DROP_SITE_HEAD)) * _keep_scale(p)
    mi = _f64(ops.dropout_mask(N, H, p, SEED, 0, ops.DROP_SITE_HEAD_IN)) * _keep_scale(p) if kind == "roberta" else one
    return mh, mi


def _ce_forward(kind, cls, Wd, bd, Wo, bo, labels, G, p):
    from dpr_scale_b200.models.citadel_models.cross_encoder import _GroupCE
    leaves = [t.cuda().requires_grad_(True) for t in (cls, Wd, bd, Wo, bo)]
    p_in = p if kind == "roberta" else 0.0
    loss, logits = _GroupCE.apply(*leaves, labels.cuda(), G, p, p_in, SEED)
    return leaves, loss, logits


def _ce_chain(X, Wd, bd, Wo, bo, labels, G, mh, e_pre):
    """float64 closed form of the head from the dense layer's input X on, with first-order bounds of the GPU's values
    given a bound e_pre of the error of its pre-activation (docstring, section 1)."""
    import torch.nn.functional as F
    N, H = X.shape
    B = N // G
    pre = X @ Wd.T + bd
    t = torch.tanh(pre)
    tm = t * mh
    one_t2 = 1 - t * t
    e_t = one_t2 * e_pre + 4 * U * t.abs()
    logits = tm @ Wo.T + bo
    e_l = (Wo.abs() * mh * e_t).sum(1, keepdim=True) + (H + 2) * U * ((tm * Wo).abs().sum(1, keepdim=True) + bo.abs())
    lg, el = logits.view(B, G), e_l.view(B, G)
    p = torch.softmax(lg, 1)
    onehot = F.one_hot(labels.to(X.device), G).double()
    e_p = p * (el + (p * el).sum(1, keepdim=True)) + (G + 8) * U * p
    gc, e_g = ((p - onehot) / B).view(N, 1), (e_p / B).view(N, 1)
    dpre = gc * Wo * one_t2 * mh
    e_dpre = (e_g * Wo.abs() * one_t2 + gc.abs() * Wo.abs() * (2 * t.abs() * e_t + 10 * U)) * mh + 3 * U * dpre.abs()
    loss = (torch.logsumexp(lg, 1) - (lg * onehot).sum(1)).mean()
    return dict(
        logits=(logits.view(-1), e_l.view(-1)),
        loss=(loss, ((p * el).sum(1) + (onehot * el).sum(1)).mean() + (G + B + 8) * U * (lg.abs().max() + loss.abs())),
        dpre=(dpre, e_dpre + BF * (dpre.abs() + e_dpre)),
        dWo=((gc * tm).sum(0, keepdim=True),
             (e_g * tm.abs() + gc.abs() * mh * e_t).sum(0, keepdim=True) + (N + 2) * U * (gc * tm).abs().sum(0, keepdim=True)),
        dbo=(gc.sum(0), e_g.sum(0) + (N + 1) * U * gc.abs().sum(0)))


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,G,H", CE_CASES)
@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_group_ce_head_stages_match_float64(kind, B, G, H, p):
    N = B * G
    cls, Wd, bd, Wo, bo, labels = _ce_inputs(B, G, H, 1000 * B + 10 * G + H)
    leaves, loss, logits = _ce_forward(kind, cls, Wd, bd, Wo, bo, labels, G, p)
    x16, w16, dpre, dw_out, db_out, drop_in = loss.grad_fn.saved_tensors
    assert (drop_in is not None) == (kind == "roberta" and p > 0)
    loss.backward()
    torch.cuda.synchronize()
    mh, mi = _ce_masks(kind, N, H, p)
    X, Wt, bd64, Wo64, bo64 = (_f64(t) for t in (x16, w16, bd, Wo, bo))
    r = {}
    xin = _f64(cls) * mi                                   # the dense layer's input: the dropped CLS rows, in bf16
    _check(r, "x16", X, xin, (BF + 2 * U) * xin.abs())
    c = _ce_chain(X, Wt, bd64, Wo64, bo64, labels, G, mh, (H + 2) * U * (X.abs() @ Wt.abs().T + bd64.abs()))
    for name, got in (("logits", logits), ("loss", loss), ("dpre", dpre), ("dWo", leaves[3].grad),
                      ("dbo", leaves[4].grad)):
        _check(r, name, got, *c[name])
    D = _f64(dpre)
    _check(r, "dWd", leaves[1].grad, D.T @ X, (N + 2) * U * (D.abs().T @ X.abs()))
    _check(r, "dbd", leaves[2].grad, D.sum(0), (N + 1) * U * D.abs().sum(0))
    dxr = (D @ Wt) * mi
    _check(r, "dx", leaves[0].grad, dxr, (H + 2) * U * (D.abs() @ Wt.abs()) * mi + U * dxr.abs())
    _report(f"group CE stages {kind} B={B} G={G} H={H} p={p}", r)


def _ce_end_to_end(r, kind, leaves, loss, logits, cls, Wd, bd, Wo, bo, labels, G, p, g=1.0):
    """The GPU's loss, logits and gradients of g * loss against float64 autograd of the head at the fp32 CLS rows.
    Returns the rel-L2 of each gradient but db_out, whose reference is zero (a group's softmax gradient sums to 0)."""
    from oracle.cross_encoder_train import head_ce
    from tests import rerank_cases
    from tests.util import rel_l2
    N, H = cls.shape
    mh, mi = _ce_masks(kind, N, H, p)
    x = _f64(cls).requires_grad_(True)
    Wd64, bd64, Wo64, bo64 = (_f64(t).requires_grad_(True) for t in (Wd, bd, Wo, bo))
    if kind == "bert":
        names = ("transformer.bert.pooler.dense.", "transformer.classifier.")
    else:
        names = ("transformer.classifier.dense.", "transformer.classifier.out_proj.")
    sd = {names[0] + "weight": Wd64, names[0] + "bias": bd64, names[1] + "weight": Wo64, names[1] + "bias": bo64}
    ref_loss, ref_logits = head_ce(sd, rerank_cases.ORACLE_CFG[kind], x, labels.cuda(), G,
                                   head_in=mi if kind == "roberta" and p > 0 else None, head=mh if p > 0 else None)
    (g * ref_loss).backward()
    with torch.no_grad():
        xin = x * mi
        bx = BF + 2 * U                                     # x16 against the exact dropped rows
        A = xin.abs() @ Wd64.abs().T
        e_pre = (bx + BF + bx * BF) * A + (H + 2) * U * ((1 + bx) * (1 + BF) * A + bd64.abs())
        c = _ce_chain(xin, Wd64, bd64, Wo64, bo64, labels, G, mh, e_pre)
        _check(r, "logits", logits, ref_logits, c["logits"][1])
        _check(r, "loss", loss, ref_loss, c["loss"][1])
        dpre, e_dpre = (g * v for v in c["dpre"])
        Dm, Xm, Wm = dpre.abs() + e_dpre, (1 + bx) * xin.abs(), (1 + BF) * Wd64.abs()
        grads = ((leaves[0], x, (e_dpre @ Wm + BF * (dpre.abs() @ Wd64.abs()) + (H + 2) * U * (Dm @ Wm)) * mi
                  + 2 * U * x.grad.abs()),
                 (leaves[1], Wd64, e_dpre.T @ Xm + bx * (dpre.abs().T @ xin.abs()) + (N + 2) * U * (Dm.T @ Xm) + U * Wd64.grad.abs()),
                 (leaves[2], bd64, e_dpre.sum(0) + (N + 1) * U * Dm.sum(0) + U * bd64.grad.abs()),
                 (leaves[3], Wo64, g * c["dWo"][1] + U * Wo64.grad.abs()),
                 (leaves[4], bo64, g * c["dbo"][1] + U * bo64.grad.abs()))
        rel = {}
        for (got, ref, bound), name in zip(grads, ("dx", "dWd", "dbd", "dWo", "dbo")):
            _check(r, name, got.grad, ref.grad, bound)
            if name != "dbo":
                rel[name] = rel_l2(got.grad.double().cpu(), ref.grad.cpu())
    return rel


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,G,H", CE_CASES)
@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_group_ce_head_end_to_end_matches_float64(kind, B, G, H, p):
    cls, Wd, bd, Wo, bo, labels = _ce_inputs(B, G, H, 1000 * B + 10 * G + H)
    leaves, loss, logits = _ce_forward(kind, cls, Wd, bd, Wo, bo, labels, G, p)
    loss.backward()
    torch.cuda.synchronize()
    r = {}
    rel = _ce_end_to_end(r, kind, leaves, loss, logits, cls, Wd, bd, Wo, bo, labels, G, p)
    _report(f"group CE end to end {kind} B={B} G={G} H={H} p={p}", r,
            " | rel-L2 " + ", ".join(f"{k} {v:.1e}" for k, v in rel.items()))


def _ce_close(a, b, D, X, g):
    """|a - b| within two fp32 GEMM / column-sum bounds (split-K atomics sum in any order) and one rounding."""
    N = D.shape[0]
    return (_f64(a) - _f64(b)).abs() <= 2 * (N + 2) * U * g * (D.abs().T @ X.abs() if X is not None
                                                                  else D.abs().sum(0)) + U * _f64(a).abs()


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_group_ce_scaled_loss_scales_every_gradient(kind):
    """Gradients of 0.37 * loss are float32(0.37) x those of loss: bitwise where the arithmetic is the same (dx, the
    label projection), to fp32 rounding where split-K atomics sum in another order (the dense layer)."""
    B, G, H, p = 3, 7, 768, 0.1
    inputs = _ce_inputs(B, G, H, 17)
    plain, loss, _ = _ce_forward(kind, *inputs, G, p)
    x16, dpre = loss.grad_fn.saved_tensors[0], loss.grad_fn.saved_tensors[2]
    loss.backward()
    scaled, loss2, logits2 = _ce_forward(kind, *inputs, G, p)
    (SCALE * loss2).backward()
    torch.cuda.synchronize()
    s = torch.tensor(SCALE, dtype=torch.float32, device="cuda")
    for i in (0, 3, 4):
        assert torch.equal(scaled[i].grad, plain[i].grad * s), i
    D, X = _f64(dpre), _f64(x16)
    assert bool(_ce_close(scaled[1].grad, plain[1].grad * s, D, X, SCALE).all())
    assert bool(_ce_close(scaled[2].grad, plain[2].grad * s, D, None, SCALE).all())
    r = {}
    rel = _ce_end_to_end(r, kind, scaled, loss2, logits2, *inputs, G, p, g=float(s))
    _report(f"group CE 0.37 * loss {kind}", r, " | rel-L2 " + ", ".join(f"{k} {v:.1e}" for k, v in rel.items()))


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_group_ce_second_backward_gives_the_same_gradients(kind):
    """backward scales the saved label-projection gradients by the upstream gradient: a second backward through the
    same graph (retain_graph=True) must see them unscaled."""
    B, G, H, p = 3, 7, 128, 0.1
    inputs = _ce_inputs(B, G, H, 23)
    leaves, loss, _ = _ce_forward(kind, *inputs, G, p)
    x16, dpre = loss.grad_fn.saved_tensors[0], loss.grad_fn.saved_tensors[2]
    (SCALE * loss).backward(retain_graph=True)
    first = [t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    (SCALE * loss).backward()
    torch.cuda.synchronize()
    for i in (0, 3, 4):
        assert torch.equal(leaves[i].grad, first[i]), i
    D, X = _f64(dpre), _f64(x16)
    assert bool(_ce_close(leaves[1].grad, first[1], D, X, SCALE).all())
    assert bool(_ce_close(leaves[2].grad, first[2], D, None, SCALE).all())


# ------------------------------------------------------------------ the handoff into the encoder body
def _hook_first_arg(monkeypatch, module, name, seen):
    """Replace module.name (an autograd Function) by one that records the gradient of its first argument."""
    real = getattr(module, name)

    class Hooked:
        @staticmethod
        def apply(first, *args):
            first.register_hook(lambda grad: seen.append(grad.detach().clone()))
            return real.apply(first, *args)

    monkeypatch.setattr(module, name, Hooked)


def _record_dpooled(monkeypatch, enc, got):
    orig = enc._run_backward

    def run_backward(state, dpooled, sync=True):
        got.append(dpooled.detach().clone())
        return orig(state, dpooled, sync)

    monkeypatch.setattr(enc, "_run_backward", run_backward)


def _match_by_rows(seen, got, rows):
    assert len(seen) == len(got) == len(rows), (len(seen), len(got))
    for n in rows:
        a = [t for t in seen if t.shape[0] == n]
        b = [t for t in got if t.shape[0] == n]
        assert len(a) == len(b) == 1
        assert a[0].dtype == b[0].dtype == torch.float32 and torch.equal(a[0], b[0]), n


@pytest.mark.parametrize("shared", [False, True])
def test_encoder_receives_the_projection_dx_bitwise(monkeypatch, shared):
    import torch.nn.functional as F
    from dpr_scale_b200.models import hf_model
    cfg = dict(vocab_size=96, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
               max_position_embeddings=48)
    q_enc = hf_model.HFEncoder.from_config(cfg, dropout=0.1, projection_dim=64, seed=1).cuda().train()
    c_enc = q_enc if shared else hf_model.HFEncoder.from_config(cfg, dropout=0.1, projection_dim=64, seed=2).cuda().train()
    seen, got = [], []
    _hook_first_arg(monkeypatch, hf_model, "_ProjectFn", seen)
    for enc in {id(e): e for e in (q_enc, c_enc)}.values():
        _record_dpooled(monkeypatch, enc, got)
    g = torch.Generator().manual_seed(5)

    def toks(n):
        ids = torch.randint(3, 96, (n, 16), generator=g)
        am = torch.ones(n, 16, dtype=torch.int64)
        am[0, 10:] = 0
        return {"input_ids": (ids * am).cuda(), "token_type_ids": torch.zeros_like(ids).cuda(),
                "attention_mask": am.cuda()}

    q, c = q_enc(toks(4)), c_enc(toks(8))
    loss = F.cross_entropy(q @ c.t(), torch.arange(4, device="cuda") * 2)
    (SCALE * loss).backward()
    torch.cuda.synchronize()
    _match_by_rows(seen, got, (4, 8))


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_encoder_receives_the_group_ce_dx_bitwise(monkeypatch, kind):
    from dpr_scale_b200.models.citadel_models import cross_encoder
    from tests.test_cross_encoder_train_gpu import _tiny, _tokens
    m, _ = _tiny(kind, 0.1)
    m.train()
    seen, got = [], []
    _hook_first_arg(monkeypatch, cross_encoder, "_GroupCE", seen)
    _record_dpooled(monkeypatch, m._body, got)
    tok = {k: v.cuda() for k, v in _tokens(kind, 12, 24, 9).items()}
    loss, _ = m.group_ce(tok, torch.tensor([0, 3, 1]), 4)
    (SCALE * loss).backward()
    torch.cuda.synchronize()
    _match_by_rows(seen, got, (12,))


@pytest.mark.parametrize("kind", ["bert", "roberta"])
def test_eval_group_ce_logits_match_forward(kind):
    """Validation metrics come from group_ce in eval mode, reranking from forward (seqcls_head_fwd): same logits within
    two fp32 dot-product bounds (|tanh| <= 1)."""
    from tests.test_cross_encoder_train_gpu import _tiny, _tokens
    m, _ = _tiny(kind, 0.1)
    m.eval()
    tok = {k: v.cuda() for k, v in _tokens(kind, 12, 24, 11).items()}
    with torch.no_grad():
        _, logits = m.group_ce(tok, torch.tensor([0, 3, 1]), 4)
        fwd = m(tok)
    out = m._head_linears()[1]
    H = m.config["hidden_size"]
    bound = 2 * (H + 6) * U * (_f64(out.weight).abs().sum() + _f64(out.bias).abs().sum())
    r = {}
    _check(r, "logits", logits, _f64(fwd[:, 0]), bound)
    _report(f"eval group_ce vs forward {kind}", r)
