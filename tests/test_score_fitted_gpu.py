"""The fused scoring + cross-entropy kernels (dprb_score_tc_fwd / _bwd) on the batches a retriever in training sees:
every label the argmax of its row by a margin, per-row losses far below 1, |logit| in the hundreds (raw CLS dot
products at temperature 1) or normalized embeddings at inv_t 20 / 100.  Each query row of dq and each column of dc is
compared with float64 autograd of cross_entropy(q c^T inv_t), against that row's own max (check_fitted documents the
gates), next to torch's fp32 cross_entropy on the CPU on the same inputs.

The generator is tested without a GPU (test_fitted_batch_regime): the regimes below are what it claims."""
import math

import pytest
import torch

U = 2.0 ** -24                  # fp32 unit roundoff
EPS_ROW = 2.0 ** -20            # 8 ulp of 1: what fp32 p and p - 1 of one row can be off by
LOGIT_TOL = (1e-5, 1e-3)        # bf16x3 logits: 1e-5 |logit| + 1e-3 (include/dprb.h, score_tc.cu)
F32_FACTOR = 4.0                # a row of dq / dc may be this many times worse than fp32 torch beyond its bound

Q_REG, C_REG, D_REG = 160, 300, 768
REGIMES = {
    "raw20": dict(logit_max=20.0, margin=(3.0, 10.0), spread=2.0),
    "raw80": dict(logit_max=80.0, margin=(5.0, 20.0), spread=3.0),
    "raw250": dict(logit_max=250.0, margin=(5.0, 20.0), spread=4.0),
    "raw250_inv_t_0.125": dict(logit_max=250.0, inv_t=0.125, margin=(5.0, 20.0), spread=4.0),
    "norm_inv_t20": dict(normalized=True, inv_t=20.0, margin=(6.0, 12.0), common=0.2),
    "norm_inv_t100": dict(normalized=True, inv_t=100.0, margin=(5.0, 20.0)),
    "mixed250": dict(logit_max=250.0, margin=(5.0, 20.0), spread=4.0, fitted=0.5),
}


def _bisect(gap, target, lo, hi, iters=80):
    """Per-row root of the increasing-through-the-bracket gap(t) = target over [lo, hi] (float64 vectors)."""
    assert bool((gap(lo) < target).all() and (gap(hi) > target).all()), "margin outside the reachable range"
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        below = gap(mid) < target
        lo, hi = torch.where(below, mid, lo), torch.where(below, hi, mid)
    return 0.5 * (lo + hi)


def fitted_batch(Q, C, d, *, logit_max=250.0, inv_t=1.0, normalized=False, margin=(5.0, 20.0), spread=4.0,
                 common=0.5, fitted=1.0, label_lo=0, seed=0):
    """Seeded fp32 q [Q, d], c [C, d] and int64 labels [Q]; logits s = q c^T * inv_t.

    The first round(fitted * Q) rows are fitted: the label is the argmax of the row by a margin drawn uniformly from
    `margin` (logit units).  The other rows keep a random label, as in a batch the model does not fit yet.  Labels
    are drawn from [label_lo, C).
      unnormalized: the logits of a row spread ~ N(0, spread^2) about a per-row offset that puts the row's largest
        |logit| at U(0.6, 1) * logit_max (one row in four negative): the shared direction raw CLS embeddings carry.
        inv_t only rescales q, so |logit| and inv_t are set independently.
      normalized: unit q and c rows whose cosines share `common` (cos ~ common between unrelated rows); logit_max is
        not used, |logit| <= inv_t.
    Built in float64 in d - 1 coordinates and turned by a random orthogonal matrix, so every coordinate carries a part
    of the shared direction.  The last coordinate is a probe that leaves every logit as it is: q there is 0 and c is 1,
    so dq_i there is scale * sum_j W_ij, the row sum of W.  Returns q, c, labels, `fitted` (bool [Q]) and the
    float64 logits and margins of the fp32 q, c."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    d -= 1
    rows = torch.arange(Q)
    labels = torch.randint(label_lo, C, (Q,), generator=g)
    fit = rows < int(round(fitted * Q))
    want = margin[0] + (margin[1] - margin[0]) * torch.rand(Q, generator=g, dtype=f64)
    onehot = torch.nn.functional.one_hot(labels, C).bool()

    def gap_of(s):
        return s[rows, labels] - s.masked_fill(onehot, -math.inf).amax(1)

    if normalized:
        a, b = math.sqrt(common), math.sqrt(1.0 - common)
        y = torch.randn(C, d - 1, generator=g, dtype=f64)
        x = torch.randn(Q, d - 1, generator=g, dtype=f64)
        cf = torch.cat([torch.full((C, 1), a, dtype=f64), b * y / y.norm(dim=1, keepdim=True)], 1)
        qf = torch.cat([torch.full((Q, 1), a, dtype=f64), b * x / x.norm(dim=1, keepdim=True)], 1)
        G, H = qf @ cf.T, cf[labels] @ cf.T          # q.c_j and c_label.c_j
        tt = torch.zeros(Q, dtype=f64)
        if bool(fit.any()):
            Gf, Hf, n = G[fit], H[fit], int(fit.sum())
            lab_f, rows_f, oh_f = labels[fit], torch.arange(n), onehot[fit]
            glab = Gf[rows_f, lab_f]

            def gap(t):   # inv_t (cos_label - max other cos) of normalize(q + t c_label)
                s = (Gf + t[:, None] * Hf) / torch.sqrt(1.0 + 2.0 * t * glab + t * t)[:, None]
                return inv_t * (s[rows_f, lab_f] - s.masked_fill(oh_f, -math.inf).amax(1))

            tt[fit] = _bisect(gap, want[fit], torch.full((n,), -0.5, dtype=f64), torch.full((n,), 50.0, dtype=f64))
        qf = qf + tt[:, None] * cf[labels]
        qf = qf / qf.norm(dim=1, keepdim=True)
        qscale = 1.0
    else:
        y = torch.randn(C, d - 1, generator=g, dtype=f64) / math.sqrt(d - 1)
        x = torch.randn(Q, d - 1, generator=g, dtype=f64) * spread
        step = y[labels] / (y[labels] ** 2).sum(1, keepdim=True)      # raises the label's logit by 1 per unit t
        G, H = x @ y.T, step @ y.T
        tt = torch.zeros(Q, dtype=f64)
        if bool(fit.any()):
            Gf, Hf = G[fit], H[fit]
            lab_f, rows_f = labels[fit], torch.arange(int(fit.sum()))
            oh_f = onehot[fit]

            def gap(t):
                s = Gf + t[:, None] * Hf
                return s[rows_f, lab_f] - s.masked_fill(oh_f, -math.inf).amax(1)

            n = int(fit.sum())
            tt[fit] = _bisect(gap, want[fit], torch.full((n,), -400.0, dtype=f64), torch.full((n,), 800.0, dtype=f64))
        x = x + tt[:, None] * step
        s0 = x @ y.T
        top = logit_max * (0.6 + 0.4 * torch.rand(Q, generator=g, dtype=f64))
        neg = torch.rand(Q, generator=g) < 0.25
        off = torch.where(neg, -top - s0.amin(1), top - s0.amax(1))
        qf = torch.cat([off[:, None], x], 1)
        cf = torch.cat([torch.ones(C, 1, dtype=f64), y], 1)
        qscale = 1.0 / inv_t
    R, _ = torch.linalg.qr(torch.randn(d, d, generator=g, dtype=f64))
    q = torch.cat([qf @ R * qscale, torch.zeros(Q, 1, dtype=f64)], 1).float()
    c = torch.cat([cf @ R, torch.ones(C, 1, dtype=f64)], 1).float()
    s = q.double() @ c.double().T * inv_t
    return {"q": q, "c": c, "labels": labels, "fitted": fit, "logits": s, "margin": gap_of(s)}


def _regime_batch(name, seed=1):
    kw = dict(REGIMES[name])
    return fitted_batch(Q_REG, C_REG, D_REG, seed=seed, **kw), kw


@pytest.mark.parametrize("name", sorted(REGIMES))
def test_fitted_batch_regime(name):
    """CPU: the generator makes the regime it claims - fitted rows peak on their label by a margin in range, the
    logit range is the requested one, the per-row loss of fitted rows is small and random rows peak elsewhere."""
    b, kw = _regime_batch(name)
    s, lab, fit, mg = b["logits"], b["labels"], b["fitted"], b["margin"]
    assert int(fit.sum()) == round(kw.get("fitted", 1.0) * Q_REG)
    assert bool((s[fit].argmax(1) == lab[fit]).all())
    lo, hi = kw["margin"]
    assert float(mg[fit].min()) >= lo - 1e-3 and float(mg[fit].max()) <= hi + 1e-3, (float(mg[fit].min()),
                                                                                     float(mg[fit].max()))
    inv_t = kw.get("inv_t", 1.0)
    amax = float(s.abs().max())
    if kw.get("normalized"):
        assert 0.5 * inv_t <= amax <= inv_t * (1 + 1e-5), amax
        assert torch.allclose(b["q"][:, :-1].double().norm(dim=1), torch.ones(Q_REG, dtype=torch.float64), atol=1e-6)
        assert torch.allclose(b["c"][:, :-1].double().norm(dim=1), torch.ones(C_REG, dtype=torch.float64), atol=1e-6)
    else:
        assert 0.9 * kw["logit_max"] <= amax <= kw["logit_max"] * (1 + 1e-5), amax
        assert float(s.abs().amax(1).min()) >= 0.5 * kw["logit_max"]     # every row at that magnitude, not a few
    assert bool((b["q"][:, -1] == 0).all() and (b["c"][:, -1] == 1).all())
    loss = torch.logsumexp(s, 1) - s[torch.arange(Q_REG), lab]
    assert float(loss[fit].median()) < 0.1 and float(loss[fit].max()) < 1.0 and float(loss[fit].min()) > 0.0
    if not bool(fit.all()):
        assert float((s[~fit].argmax(1) != lab[~fit]).double().mean()) > 0.9
        assert float(loss[~fit].median()) > 1.0


# ------------------------------------------------------------------ GPU: kernel against float64
def _kernel(q, c, labels, inv_t, q0, nq, c0, nc, pair_mask):
    """Training-form forward, backward, then an evaluation-form forward (logits) on the SAME workspace, whose row
    counters the first call left for reuse.  Everything on the device, returned on the CPU."""
    from dpr_scale_b200 import _lib, ops
    dev = "cuda"
    lib = _lib.load()
    Q, d = q.shape
    C = c.shape[0]
    qd, cd, ld = q.to(dev), c.to(dev), labels.to(dev)
    pm = None if pair_mask is None else pair_mask.to(torch.uint8).to(dev)
    nbytes = int(lib.dprb_score_tc_workspace_bytes(Q, C, d, nq, nc))
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    base, room = ws.data_ptr() + (-ws.data_ptr()) % 256, nbytes

    def fwd(want_logits):
        lse = torch.empty(Q, device=dev)
        loss = torch.zeros(1, device=dev)
        logits = torch.empty(Q, C, device=dev) if want_logits else None
        ops.check(lib.dprb_score_tc_fwd(ops._ptr(qd), ops._ptr(cd), None, ops._ptr(pm), ops._ptr(ld), float(inv_t),
                                        ops._ptr(lse), ops._ptr(loss), ops._ptr(logits), Q, C, d, nq, nc, base, room,
                                        ops._stream()), "dprb_score_tc_fwd")
        return lse, loss, logits

    lse, loss, _ = fwd(False)
    dq = torch.empty(nq, d, device=dev)
    dc = torch.empty(nc, d, device=dev)
    ops.check(lib.dprb_score_tc_bwd(None, ops._ptr(pm), ops._ptr(ld), ops._ptr(lse), 1.0, float(inv_t), ops._ptr(dq),
                                    ops._ptr(dc), Q, C, d, q0, nq, c0, nc, base, room, ops._stream()),
              "dprb_score_tc_bwd")
    lse2, loss2, logits = fwd(True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in dict(lse=lse, loss=loss, dq=dq, dc=dc, lse2=lse2, loss2=loss2,
                                        logits=logits).items()}


def _reference(q, c, labels, inv_t, pair_mask, dtype):
    qr = q.to(dtype).requires_grad_(True)
    cr = c.to(dtype).requires_grad_(True)
    s = qr @ cr.T * inv_t
    if pair_mask is not None:
        s = s.masked_fill(pair_mask, -math.inf)
    loss = torch.nn.functional.cross_entropy(s, labels)
    loss.backward()
    zero = torch.zeros_like
    return s.detach(), loss.detach(), zero(qr) if qr.grad is None else qr.grad, zero(cr) if cr.grad is None else cr.grad


def _row_gate(name, got, ref, ref32, bound, res, bad):
    """Rows of got [n, d] against float64 ref: max_k (|got - ref| - bound)_+ <= F32_FACTOR * (fp32 torch's error of
    that row, at least 1 ulp of the row's max).  Keeps the worst row's ratio and the per-row median relative errors of
    the kernel and of fp32 torch."""
    err = (got.double() - ref).abs()
    rmax = ref.abs().amax(1)
    e32 = (ref32.double() - ref).abs().amax(1)
    excess = (err - bound).clamp_min(0).amax(1)
    allowed = F32_FACTOR * torch.maximum(e32, U * rmax)
    ratio = torch.where(excess > 0, excess / allowed, torch.zeros_like(excess))
    live = rmax > 0
    res[name + "_ratio"] = float(ratio.max()) if len(ratio) else 0.0
    res[name + "_median_rel"] = float((err.amax(1)[live] / rmax[live]).median()) if bool(live.any()) else 0.0
    res[name + "_median_rel_fp32"] = float((e32[live] / rmax[live]).median()) if bool(live.any()) else 0.0
    if res[name + "_ratio"] > 1.0:
        i = int(ratio.argmax())
        bad.append(f"{name}: row {i} exceeds its bound by {float(excess[i]):.3e} > {F32_FACTOR} x fp32 error "
                   f"{float(e32[i]):.3e} (row max {float(rmax[i]):.3e}; {res[name + '_ratio']:.1f} x gate)")


def check_fitted(q, c, labels, inv_t, q0=0, nq=None, c0=0, nc=None, pair_mask=None, res=None):
    """dprb_score_tc_fwd / _bwd against float64 autograd of mean cross_entropy(q c^T inv_t) (pair_mask: True -> -inf).
    Fills `res` with the error figures and raises AssertionError listing every gate exceeded.

    With s the logits, P = softmax(s), W = P - onehot(label), scale = inv_t / Q:  dq = scale W c, dc = scale W^T q.
    The row's logit errors e_ij are measured from the logits the kernel returns (gated first at the documented
    1e-5 |logit| + 1e-3): ds_i = max_j |e_ij| and their spread r_i = max_j e_ij - min_j e_ij.  An error common to
    the row leaves softmax and loss alone; to first order the errors move W_ij = p_j - onehot by
    p_j (e_j - sum_l p_l e_l), at most r_i |W_ij| (the label's term is p_lab sum_j p_j (e_lab - e_j)
    <= r_i p_lab (1 - p_lab)).  So the kernel's W differs from float64 by at most
        D_ij = (r_i + kappa) |W_ij| + EPS_ROW (P_ij + onehot_ij)
    kappa = 2^-17 + (max(Q, C) / 16 + 8) 2^-24: the bf16 hi + lo split of W (2^-18 |W|), the dropped lo x m product of
    the GEMM (2^-18), and its fp32 accumulation over K / 16 k-steps plus the split-K atomics;  EPS_ROW = 2^-20, 8 ulp
    of 1, is what fp32 p_j = 2^((s2_j - M) - lg2 L) and p - 1 can give (ex2 / log1p to a few ulp, L accumulated
    in fp32).  Gates:
      * logits: per row, max |err| <= 1e-5 max|s_i| + 1e-3; masks identical (-inf where masked);
      * invariant (c0 = 0, nc = C): rows of W sum to 0 whatever the logit error, so sum_j dc_j = 0 exactly; per
        coordinate k,  |sum_j dc_jk| <= scale sum_i (EPS_ROW + kappa sum_j |W_ij|) |q_ik|.  The same per row where the
        batch has fitted_batch's probe coordinate (q 0, c 1):  |dq_i / scale| there <= EPS_ROW + kappa sum_j |W_ij|.
        A lse rounded at the logit's magnitude scales a whole row of P by 1 + eta, eta ~ ulp(|logit|), and fails
        these wherever eta outgrows EPS_ROW;
      * dq rows / dc columns: beyond scale (D |c|)_ik resp. scale (D^T |q|)_jk elementwise, a row's max error may be
        at most F32_FACTOR x fp32 torch's max error of that row (_row_gate);
      * loss_sum / Q relative to the loss itself: per row |d loss_i| <= r_i (1 - p_lab) + 8 ulp(loss_i), plus
        (8 + Q / 32) ulp of the mean for the fp32 warp sums and atomics;
      * lse per row: ds_i + 4 ulp(|lse_i|) + 8 ulp(1);
      * a second forward on the same workspace (evaluation form, logits) gives bitwise the same lse."""
    res = {} if res is None else res
    Q, d = q.shape
    C = c.shape[0]
    nq = Q if nq is None else nq
    nc = C if nc is None else nc
    k = _kernel(q, c, labels, inv_t, q0, nq, c0, nc, pair_mask)
    s, loss64, dq64, dc64 = _reference(q, c, labels, inv_t, pair_mask, torch.float64)
    _, loss32, dq32, dc32 = _reference(q, c, labels, inv_t, pair_mask, torch.float32)
    bad = []
    fin = torch.isfinite(s)
    assert torch.equal(torch.isfinite(k["logits"]), fin), "logits: masked entries differ"
    assert torch.isfinite(k["dq"]).all() and torch.isfinite(k["dc"]).all(), "non-finite gradients"
    e = k["logits"].double() - s
    zero = torch.zeros((), dtype=torch.float64)
    srow = torch.where(fin, s.abs(), zero).amax(1)
    ds = torch.where(fin, e.abs(), zero).amax(1)
    spread = torch.where(fin, e, -math.inf).amax(1) - torch.where(fin, e, math.inf).amin(1)
    res["logit_spread_rel"] = float((spread / srow).max())
    res["logit_err_rel"] = float((ds / srow).max())
    r = float((ds / (LOGIT_TOL[0] * srow + LOGIT_TOL[1])).max())
    res["logit_ratio"] = r
    if r > 1.0:
        bad.append(f"logits: {r:.2f} x gate")

    P = torch.softmax(s, 1)
    onehot = torch.nn.functional.one_hot(labels, C).double()
    W = P - onehot
    Wa = W.abs()
    scale = inv_t / Q
    kappa = 2.0 ** -17 + (max(Q, C) / 16 + 8) * U
    D = (spread[:, None] + kappa) * Wa + EPS_ROW * (P + onehot)
    qa, ca = q.double().abs(), c.double().abs()
    _row_gate("dq", k["dq"], dq64[q0:q0 + nq], dq32[q0:q0 + nq], scale * D[q0:q0 + nq] @ ca, res, bad)
    _row_gate("dc", k["dc"], dc64[c0:c0 + nc], dc32[c0:c0 + nc], scale * D[:, c0:c0 + nc].T @ qa, res, bad)

    if bool((q[:, -1] == 0).all() and (c[:, -1] == 1).all()):
        sig = k["dq"][:, -1].double() / scale
        tol = EPS_ROW + kappa * Wa[q0:q0 + nq].sum(1)
        res["w_rowsum_ratio"], res["w_rowsum_max"] = float((sig.abs() / tol).max()), float(sig.abs().max())
        if res["w_rowsum_ratio"] > 1.0:
            bad.append(f"sum_j W_ij: {res['w_rowsum_max']:.3e}, {res['w_rowsum_ratio']:.1f} x gate")
    if c0 == 0 and nc == C:
        tol = scale * ((EPS_ROW + kappa * Wa.sum(1))[:, None] * qa).sum(0)
        sdc = k["dc"].double().sum(0).abs()
        ratio = torch.where(tol > 0, sdc / tol, torch.where(sdc > 0, math.inf, 0.0))   # tol 0: q is 0 there
        res["dc_sum_ratio"], res["dc_sum_max"] = float(ratio.max()), float(sdc.max())
        if res["dc_sum_ratio"] > 1.0:
            bad.append(f"sum_j dc_j: {res['dc_sum_max']:.3e}, {res['dc_sum_ratio']:.1f} x gate")

    rows = torch.arange(Q)
    lse64 = torch.logsumexp(s, 1)
    li = lse64 - s[rows, labels]
    ltol = float((spread * (1 - P[rows, labels]) + 8 * U * li).mean()) + (8 + Q / 32) * U * float(loss64)
    for tag in ("loss", "loss2"):
        e = abs(float(k[tag]) / Q - float(loss64))
        res[tag + "_err"], res[tag + "_ratio"] = e, (e / ltol if ltol > 0 else (0.0 if e == 0 else math.inf))
        if e > ltol:
            bad.append(f"{tag}: mean {float(k[tag]) / Q:.9e} vs {float(loss64):.9e}: {e / ltol:.1f} x gate")
    res["loss"], res["loss_err_fp32"] = float(loss64), abs(float(loss32) - float(loss64))
    lerr = (k["lse"].double() - lse64).abs()
    r = float((lerr / (ds + 4 * U * lse64.abs() + 8 * U)).max())
    res["lse_ratio"], res["lse_err"] = r, float(lerr.max())
    if r > 1.0:
        bad.append(f"lse: {res['lse_err']:.3e}, {r:.1f} x gate")
    assert torch.equal(k["lse2"], k["lse"]), "a second forward on the same workspace changed lse"
    res["_kernel"] = k
    assert not bad, "; ".join(bad)
    return res


def _report(res):
    return {k: v for k, v in res.items() if not k.startswith("_")}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(REGIMES))
def test_fitted_regime(name):
    b, kw = _regime_batch(name)
    res = check_fitted(b["q"], b["c"], b["labels"], kw.get("inv_t", 1.0))
    print(name, _report(res))


# windows (q0, nq, c0, nc) off the 128 boundaries; the first ends inside the last partial row and column tiles
WINDOWS = {"to_end": (37, 263, 130, 203), "inner": (5, 200, 1, 250)}


@pytest.mark.gpu
@pytest.mark.parametrize("window", sorted(WINDOWS))
@pytest.mark.parametrize("fitted", [1.0, 0.0], ids=["fitted", "random"])
def test_local_windows(window, fitted):
    b = fitted_batch(300, 333, 256, fitted=fitted, seed=2)
    q0, nq, c0, nc = WINDOWS[window]
    check_fitted(b["q"], b["c"], b["labels"], 1.0, q0, nq, c0, nc)


@pytest.mark.gpu
@pytest.mark.parametrize("fitted", [1.0, 0.0], ids=["fitted", "random"])
def test_label_in_last_partial_tile(fitted):
    """Every label in columns [256, 333): the last, partial column tile (C % 4 != 0: the scalar logits store)."""
    b = fitted_batch(200, 333, 256, fitted=fitted, label_lo=256, seed=3)
    check_fitted(b["q"], b["c"], b["labels"], 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("fitted", [1.0, 0.0], ids=["fitted", "random"])
def test_pair_mask_only_label_left(fitted):
    """Even rows: a pair_mask that leaves only the label.  Their softmax is exactly onehot: W row, dq row and loss are
    exactly 0 and lse is exactly the label's logit.  Odd rows: 20 % of the columns masked."""
    Q, C = 96, 200
    b = fitted_batch(Q, C, 256, fitted=fitted, seed=4)
    g = torch.Generator().manual_seed(40)
    pm = torch.rand(Q, C, generator=g) < 0.2
    pm[0::2] = True
    pm[torch.arange(Q), b["labels"]] = False
    res = check_fitted(b["q"], b["c"], b["labels"], 1.0, pair_mask=pm)
    k = res["_kernel"]
    assert float(k["dq"][0::2].abs().max()) == 0.0, "a row with only its label left has a nonzero dq"
    lab_logit = k["logits"][torch.arange(Q), b["labels"]]
    assert torch.equal(k["lse"][0::2], lab_logit[0::2]), "lse of a label-only row is not the label's logit"
    even = check_fitted(b["q"][0::2].contiguous(), b["c"], b["labels"][0::2].contiguous(), 1.0, pair_mask=pm[0::2])
    k = even["_kernel"]
    assert float(k["loss"]) == 0.0 and float(k["loss2"]) == 0.0, "label-only rows have a nonzero loss"
    assert float(k["dq"].abs().max()) == 0.0 and float(k["dc"].abs().max()) == 0.0


@pytest.mark.gpu
def test_two_equal_maxima():
    """Fitted rows whose label column gets an exact copy, so they peak twice (p = 1/2 each, loss ln 2 + ...): the copy
    in the label's own 32-column chunk, in the next 128-column tile and in the one after."""
    Q, C = 128, 300
    b = fitted_batch(Q, C, 256, seed=5)
    q, c, labels = b["q"], b["c"].clone(), b["labels"]
    free = sorted(set(range(C)) - set(labels.tolist()))
    tiles = [(0, 128), (128, 256), (256, C)]
    pairs = []
    k0s = list(dict.fromkeys(labels.tolist()))[:3]
    for shift, k0 in enumerate(k0s):
        lo, hi = ((k0 // 32) * 32, (k0 // 32) * 32 + 32) if shift == 0 else tiles[(k0 // 128 + shift) % 3]
        k1 = next(j for j in free if lo <= j < hi)
        free.remove(k1)
        c[k1] = c[k0]
        pairs.append((k0, k1))
    res = check_fitted(q, c, labels, 1.0)
    k = res["_kernel"]
    s = q.double() @ c.double().T
    for k0, k1 in pairs:
        r = labels == k0
        assert bool((s[r, k1] == s[r].amax(1)).all()), "a copied label column is not a second maximum"
        assert torch.equal(k["logits"][r, k0], k["logits"][r, k1]), "copies of one column got different logits"
