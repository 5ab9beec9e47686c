"""The optimizer kernels of csrc/optim.cu (global-norm sum of squares, AdamW, LAMB, MADGRAD) against float64, stage by
stage, at full model arena layouts and across the launch switches of the host code.

Every step restarts the float64 restatement from the kernel's own fp32 state before that step, so errors never compound
across steps, and each stage is gated by a bound counted from its own fp32 roundings (u = 2^-24; a correctly rounded
operation is off by at most u relative; cbrtf is documented at 1 ulp, i.e. 2u).  The betas, eps, lr, weight decay and
max_norm go to the oracle as the fp32 values the C ABI receives.  Stages:

  * clip multiplier: gmul = grad_scale * min(1, max_norm / (sqrt(sumsq) * grad_scale + 1e-6)) in float64 from the
    kernel's own sumsq.  With the clip active the kernel's fp32 gmul carries up to 5u (sqrt, two products, sum,
    division), so g * gmul carries eg = 6u; with the clip off or clamped to 1, gmul is grad_scale exactly (eg = 0).
  * AdamW / LAMB moments: m' = b1 m + (1 - b1) g gmul within (2 |b1 m| + (2 + eg) |(1 - b1) g gmul|) u;
    v' = b2 v + (1 - b2) (g gmul)^2 within (2 |b2 v| + (3 + 2 eg) (1 - b2) (g gmul)^2) u.
  * AdamW p', from the kernel's m' and v': pd = p (1 - lr wd), upd = lr / bc1 * m' / (sqrt(v') / sqrt(bc2) + eps),
    p' = pd - upd within (4 |pd| + 9 |upd|) u: two roundings in 1 - lr wd and one in the product; sqrt, the bc2_rsqrt
    constant, its product, + eps, the division, the bc1 constant, lr / bc1 and the final product (8); the difference (1).
  * LAMB trust (LambPlan.trust_scale), against float64 norms of the kernel's p and of u rebuilt in float64 from the
    kernel's m' and v'.  Each element's u = m / (sqrt(v) + eps) + wd p is off by at most 4u A with A = |m / (sqrt(v) +
    eps)| + |wd p|, so each u^2 by 9u A^2.  The fp32 sums follow one fixed order: per thread, 8 float4 iterations of
    a 4-term sum (3 + 8 additions), a warp tree (5), the 8 warp partials of the block in sequence (7), each lane's run
    over the segment's chunks (ceil(chunks / 32) - 1), a warp tree (5): depth D = ceil(chunks / 32) + 27.  So
    ||p|| is within ((D + 1) / 2 + 1) u, ||u|| within ((9 sum A^2 / sum u^2 + D) / 2 + 1) u, and step_size * trust
    within their sum + 3u (the division, the fp32 step size, the product).  Trust 1 (adam, ||p|| = 0 or ||u|| = 0) must
    give step_size rounded once.
  * LAMB p' = p - k u with the kernel's own k = step_size * trust: within (|p| + 6 |k| A) u.
  * MADGRAD, g'' = g gmul + wd p (off by cg u A, A = |g gmul| + |wd p|, cg = eg + 2 with decay, eg without):
    nu' = nu + lamb g''^2 within (|nu| + (2 cg + 4) lamb A^2) u, s' = s + lamb g'' within (|s| + (cg + 3) lamb A) u;
    p' from the kernel's nu', s' with q = s / (cbrt(nu) + eps) (qc = 4u): momentum 0 rebuilds x0 = p + q(nu, s), and
    z = x0 - q(nu', s') is within (2 |p| + 6 |q0| + 5 |q1|) u; momentum m uses the stored x0 and p' = m p + (1 - m) z
    is within (2 |m p| + (1 - m) (4 |x0| + 8 |q1|)) u.
  * the bf16 shadow equals p'.to(bfloat16) bit for bit, and the gradient arena is left unchanged.
  * sumsq: Wilkinson's bound for non-negative terms, (terms per thread + 4 + tree depth 8 + atomics) u of the float64
    sum, also when several calls accumulate into one non-zero buffer as the fused optimizers' clip does.

The wrappers (FusedAdamW, FusedLamb, FusedMADGRAD) are checked the same way on a tiny encoder with a projection head at
grad_scale 1/2, the arena path with fp32 betas and the per-tensor torch path with the Python floats it is given; every
scalar the torch path casts to fp32 adds one rounding to each term (cu = 1), and its norms, whose summation order is
torch's, take Wilkinson's n u.

Every case prints its worst error as a share of each gate.  Launch facts come from this device's SM count: the LAMB chunk
kernels run min(nchunks, sms * 8) CTAs and the trust kernel one warp per segment; the AdamW and MADGRAD loops run
sms * 8 blocks of 256 threads over float4s, so a second pass starts at n = 4 * sms * 8 * 256 + 4.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
TINY = 2.0 ** -146          # covers roundings in the subnormal range, where the relative model does not hold
SLICE = 1 << 24             # float64 oracle slices: 128 MB per tensor


def F32(x):
    return float(np.float32(x))


B1, B2 = F32(0.9), F32(0.999)
CHUNK = 8192                # ops.LAMB_CHUNK
BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2)
ROBERTA_LARGE = dict(vocab_size=50265, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                     intermediate_size=4096, max_position_embeddings=514, type_vocab_size=1)
LAYOUTS = {"bert-base": (BERT_BASE, 108_891_648, 197, 13_401), "roberta-large": (ROBERTA_LARGE, 354_310_144, 389, 43_456)}


def _sms():
    from dpr_scale_b200 import _lib
    return _lib.load().dprb_num_sms()


def _layout_sizes(name):
    from dpr_scale_b200.models.hf_model import ParamLayout
    cfg, total, nseg, nchunks = LAYOUTS[name]
    sizes = [math.prod(s) for _, s, _ in ParamLayout(dict(cfg, layer_norm_eps=1e-12)).entries]
    assert sum(sizes) == total and len(sizes) == nseg and sum(-(-s // CHUNK) for s in sizes) == nchunks
    return sizes


class Shares(dict):
    """Worst |got - want| / gate per stage, kept on the device until the case ends."""

    def add(self, name, got, want, gate):
        err = (got.double() - want).abs()
        self.setdefault(name, []).append((err / (gate + TINY)).max())

    def equal(self, name, ok):
        self.setdefault(name, []).append(torch.zeros((), device=DEV) if ok else torch.full((), math.inf, device=DEV))

    def done(self, label):
        out = {k: float(torch.stack(v).max()) for k, v in self.items()}
        print(f"{label}: " + " ".join(f"{k} {v:.3f}" for k, v in sorted(out.items())))
        bad = {k: v for k, v in out.items() if not v <= 1.0}
        assert not bad, (label, bad)
        return out


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _logmag(n, gen, lo, hi):
    """random signs, magnitudes log-uniform over [10^lo, 10^hi]"""
    e = torch.rand(n, device=DEV, generator=gen).mul_(hi - lo).add_(lo)
    return torch.pow(10.0, e).mul_(torch.randn(n, device=DEV, generator=gen).sign_())


def _grad(n, gen, zero_share=0.05):
    g = torch.randn(n, device=DEV, generator=gen).mul_(3.0)
    g[torch.rand(n, device=DEV, generator=gen) < zero_share] = 0.0      # unused rows: exact-zero gradients
    return g


def _sumsq64(t):
    return sum(float(t[i:i + SLICE].double().square().sum()) for i in range(0, t.numel(), SLICE))


CLIPS = ["off-null", "off-zero", "active", "inactive"]


def _clip(g, clip, gs):
    """-> (device sum of squares or None, max_norm) for one branch of clip_gmul"""
    from dpr_scale_b200 import ops
    if clip == "off-null":
        return None, 1.0
    ss = torch.zeros(1, device=DEV)
    ops.sumsq(g, ss)
    total = math.sqrt(_sumsq64(g)) * gs
    return ss, {"off-zero": 0.0, "active": F32(0.5 * total), "inactive": F32(2.0 * total)}[clip]


def _gmul(ss, gs, max_norm):
    """float64 clip multiplier from the kernel's own fp32 sum of squares -> (gmul, eg in u)"""
    if ss is None or max_norm <= 0:
        return gs, 0
    coef = max_norm / (math.sqrt(float(ss)) * gs + F32(1e-6))
    return (gs, 0) if coef >= 1.0 else (gs * coef, 6)


# ------------------------------------------------------------------ stage restatements (flat slices)
def _adamw_stages(res, pre, post, g, gmul, eg, lr, b1, b2, eps, wd, step, cu=0):
    p0, m0, v0 = (t.double() for t in pre)
    p1, m1, v1 = post
    gg = g.double() * gmul
    t1, t2 = b1 * m0, (1 - b1) * gg
    res.add("m", m1, t1 + t2, ((2 + cu) * t1.abs() + (2 + eg + cu) * t2.abs()) * U)
    t1, t2 = b2 * v0, (1 - b2) * gg * gg
    res.add("v", v1, t1 + t2, ((2 + cu) * t1 + (3 + 2 * eg + cu) * t2) * U)
    pd = p0 * (1 - lr * wd)
    upd = lr / (1 - b1 ** step) * m1.double() / (v1.double().sqrt() / math.sqrt(1 - b2 ** step) + eps)
    res.add("p", p1, pd - upd, ((4 + cu) * pd.abs() + (9 + cu) * upd.abs()) * U)


def _madgrad_stages(res, pre, post, g, x0, gmul, eg, lr, mom, wd, eps, k, root_u=2, cu=0):
    p0, nu0, s0 = (t.double() for t in pre)
    p1, nu1, s1 = post
    lam = (lr + eps) * math.sqrt(k + 1)
    gg = g.double() * gmul
    a = gg.abs()
    if wd != 0:
        gg = gg + wd * p0
        a = a + (wd * p0).abs()
    cg = eg + (2 if wd != 0 else 0) + cu
    res.add("nu", nu1, nu0 + lam * gg * gg, ((1 + cu) * nu0 + (2 * cg + 4 + cu) * lam * a * a) * U)
    res.add("s", s1, s0 + lam * gg, ((1 + cu) * s0.abs() + (cg + 3 + cu) * lam * a) * U)
    qc = root_u + 2 + cu
    q1 = s1.double() / (nu1.double().pow(1 / 3) + eps)
    if mom == 0:
        q0 = s0 / (nu0.pow(1 / 3) + eps)
        res.add("p", p1, p0 + q0 - q1, ((2 + cu) * p0.abs() + (qc + 2) * q0.abs() + (qc + 1) * q1.abs()) * U)
    else:
        x0 = x0.double()
        ck = 1 - mom
        res.add("p", p1, mom * p0 + ck * (x0 - q1),
                ((2 + cu) * (mom * p0).abs() + ck * ((4 + cu) * x0.abs() + (qc + 4) * q1.abs())) * U)


def _lamb_u(p0, m1, v1, eps, wd):
    q = m1.double() / (v1.double().sqrt() + eps)
    w = wd * p0.double()
    return q + w, q.abs() + w.abs()


def _trust_rel(depth, aa, uu):
    """relative bound of step_size * trust for sum-of-squares depth `depth` (see the module docstring)"""
    return ((depth + 1) / 2 + 1 + (9 * aa / uu + depth) / 2 + 1 + 3) * U


# ------------------------------------------------------------------ AdamW and MADGRAD over one flat arena
def _adamw_case(label, n, step, wd, clip="active", gs=1.0, seed=0, lr=1e-3, eps=1e-8):
    from dpr_scale_b200 import ops
    gen = _gen(seed)
    p = _logmag(n, gen, -5, 0)               # many |p| below the update, where the bias corrections show
    g = _grad(n, gen)
    if step == 1:
        m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    else:
        m = torch.randn(n, device=DEV, generator=gen).mul_(2 * (1 - B1 ** (step - 1)))
        v = torch.randn(n, device=DEV, generator=gen).mul_(3).square_().mul_(1 - B2 ** (step - 1))
        unused = g == 0
        m[unused] = 0.0
        v[unused] = 0.0
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ss, max_norm = _clip(g, clip, gs)
    pre = (p.clone(), m.clone(), v.clone())
    g0 = g.clone()
    lr_, eps_, wd_ = F32(lr), F32(eps), F32(wd)
    ops.adamw_step(p, g, m, v, shadow, lr_, B1, B2, eps_, wd_, step, gs, ss, max_norm)
    gmul, eg = _gmul(ss, gs, max_norm)
    res = Shares()
    for i in range(0, n, SLICE):
        sl = slice(i, i + SLICE)
        _adamw_stages(res, [t[sl] for t in pre], (p[sl], m[sl], v[sl]), g[sl], gmul, eg, lr_, B1, B2, eps_, wd_, step)
        res.equal("shadow", torch.equal(shadow[sl], p[sl].to(torch.bfloat16)))
    res.equal("grad", torch.equal(g, g0))
    return res.done(f"adamw {label} n={n} step={step} wd={wd} clip={clip} grad_scale={gs}")


def _madgrad_case(label, n, k, mom, wd, clip="active", gs=1.0, seed=1, lr=1e-2, eps=1e-6):
    from dpr_scale_b200 import ops
    gen = _gen(seed)
    p = _logmag(n, gen, -4, 0)
    g = _grad(n, gen)
    tiny = torch.rand(n, device=DEV, generator=gen) < 0.01
    g[tiny] = 1e-25                          # g * g underflows: nu' stays 0 while s' moves
    if k == 0:
        nu, s = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    else:
        nu = torch.randn(n, device=DEV, generator=gen).mul_(3).square_().mul_(0.01 * (k + 1))
        s = torch.randn(n, device=DEV, generator=gen).mul_(0.03 * math.sqrt(k + 1))
        fresh = (g == 0) | tiny                # rows no step has touched: nu = s = 0, denominator cbrt(0) + eps
        nu[fresh] = 0.0
        s[fresh] = 0.0
    x0 = (p + torch.randn(n, device=DEV, generator=gen).mul_(0.01)) if mom else None
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ss, max_norm = _clip(g, clip, gs)
    pre = (p.clone(), nu.clone(), s.clone())
    g0 = g.clone()
    lr_, eps_, wd_, mom_ = F32(lr), F32(eps), F32(wd), F32(mom)
    ops.madgrad_step(p, g, nu, s, x0, shadow, lr_, mom_, wd_, eps_, k, gs, ss, max_norm)
    gmul, eg = _gmul(ss, gs, max_norm)
    res = Shares()
    for i in range(0, n, SLICE):
        sl = slice(i, i + SLICE)
        _madgrad_stages(res, [t[sl] for t in pre], (p[sl], nu[sl], s[sl]), g[sl], x0[sl] if mom else None, gmul, eg,
                        lr_, mom_, wd_, eps_, k)
        res.equal("shadow", torch.equal(shadow[sl], p[sl].to(torch.bfloat16)))
    res.equal("grad", torch.equal(g, g0))
    if k > 0 and wd == 0:
        assert bool(((nu == 0) & (s != 0)).any())  # the cbrt(0) + eps denominator met a moving s
    return res.done(f"madgrad {label} n={n} k={k} momentum={mom} wd={wd} clip={clip} grad_scale={gs}")


def _stream_sizes():
    b4 = 4 * _sms() * 8 * 256      # one pass of the grid-stride loop, in elements
    return {"n=1": 1, "n=2": 2, "n=3": 3, "n=4": 4, "n=5": 5, "4B-1": b4 - 1, "4B": b4, "4B+3": b4 + 3,
            "4B+4": b4 + 4, "4B+5": b4 + 5, "bert-base+1": 108_891_649, "bert-base+3": 108_891_651,
            "roberta-large+1": 354_310_145, "roberta-large+3": 354_310_147}


SIZE_IDS = ["n=1", "n=2", "n=3", "n=4", "n=5", "4B-1", "4B", "4B+3", "4B+4", "4B+5", "bert-base+1", "bert-base+3",
            "roberta-large+1", "roberta-large+3"]


@pytest.mark.parametrize("size", SIZE_IDS)
def test_adamw_and_madgrad_sizes(size):
    n = _stream_sizes()[size]
    _adamw_case(size, n, 3, 0.01)
    _madgrad_case(size, n, 1, 0.9, 0.01)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("step", [1, 2, 3, 10, 1000, 100000])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_adamw_schedule(step, wd):
    _adamw_case("4B+5", _stream_sizes()["4B+5"], step, wd, seed=step)


@pytest.mark.parametrize("k", [0, 1, 10, 1000])
@pytest.mark.parametrize("mom", [0.0, 0.9])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_madgrad_schedule(k, mom, wd):
    # k = 0 is the first step, where the warmup holds lr at 0 and lr + eps drives the update
    _madgrad_case("4B+5", _stream_sizes()["4B+5"], k, mom, wd, lr=0.0 if k == 0 else 1e-2, seed=k + 7)


# ------------------------------------------------------------------ LAMB
def _lamb_case(label, sizes, mode, steps=2, seed=3, clip="active", gs=1.0, wd=0.01, zero_norm=(), zero_grad=(),
               repeat=False, lr=1e-2, eps=1e-6):
    from dpr_scale_b200 import ops
    plan = ops.LambPlan(sizes, DEV)
    n, nseg = plan.numel, plan.nseg
    offs = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    per = [-(-s // CHUNK) for s in sizes]
    grid = min(plan.nchunks, _sms() * 8)
    lane_runs = -(-max(per) // 32)
    clamp = 2.0 if mode == "debias" else 10.0
    adam, debias = mode == "adam", mode == "debias"
    gen = _gen(seed)
    p = torch.randn(n, device=DEV, generator=gen)
    targets = [0.3, 3.0, 0.8, 20.0]          # ||p|| / clamp: both sides of the clamp
    for i in range(nseg):
        p[offs[i]:offs[i + 1]].mul_(targets[i % 4] * clamp / math.sqrt(sizes[i]))
    for i in zero_norm:
        p[offs[i]:offs[i + 1]] = 0.0
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    lr_, eps_, wd_ = F32(lr), F32(eps), F32(wd)
    res = Shares()
    for step in range(1, steps + 1):
        g = _grad(n, gen)
        for i in zero_grad:
            g[offs[i]:offs[i + 1]] = 0.0
        ss, max_norm = _clip(g, clip, gs)
        pre = (p.clone(), m.clone(), v.clone())
        g0 = g.clone()
        ops.lamb_step(p, g, m, v, shadow, plan, lr_, B1, B2, eps_, wd_, clamp, adam, debias, step, gs, ss, max_norm)
        scale = plan.trust_scale().double()
        if repeat:                         # the same inputs and sumsq give the same bits
            out = (p.clone(), m.clone(), v.clone(), shadow.clone(), plan.trust_scale().clone())
            p.copy_(pre[0]), m.copy_(pre[1]), v.copy_(pre[2])
            ops.lamb_step(p, g, m, v, shadow, plan, lr_, B1, B2, eps_, wd_, clamp, adam, debias, step, gs, ss,
                          max_norm)
            res.equal("repeat", all(torch.equal(a, b) for a, b in
                                    zip(out, (p, m, v, shadow, plan.trust_scale()))))
        gmul, eg = _gmul(ss, gs, max_norm)
        step_size = lr_ * (math.sqrt(1 - B2 ** step) / (1 - B1 ** step) if debias else 1.0)
        pp = _lamb_arena_check(res, sizes, pre, (p, m, v), g, gmul, eg, scale, step_size, eps_, wd_, clamp, adam)
        res.equal("shadow", torch.equal(shadow, p.to(torch.bfloat16)))
        res.equal("grad", torch.equal(g, g0))
        for i in zero_norm if step == 1 else ():   # the first step moves p off zero
            res.equal("trust1", float(scale[i]) == F32(step_size))
        for i in zero_grad:
            res.equal("trust1", wd != 0 or adam or float(scale[i]) == F32(step_size))
    clamped = int((pp.sqrt() > clamp).sum())
    return res.done(f"lamb {label} mode={mode} nseg={nseg} nchunks={plan.nchunks} grid={grid} "
                    f"chunk passes per CTA={-(-plan.nchunks // grid)} max chunks per segment={max(per)} "
                    f"chunk runs per lane={lane_runs} segments above the clamp={clamped}/{nseg}")


@pytest.mark.parametrize("layout", ["bert-base", "roberta-large"])
@pytest.mark.parametrize("mode", ["default", "debias", "adam"])
def test_lamb_real_layouts(layout, mode):
    sizes = _layout_sizes(layout)
    # segment 1 (position embeddings, more than 32 chunks) gets no gradient; segment 2 (token types) is all zero.
    # Default mode runs without decay, so the gradient-free segment has u = 0 and trust 1.
    kw = {"default": dict(wd=0.0, clip="active", gs=1.0), "debias": dict(wd=0.01, clip="inactive", gs=0.125),
          "adam": dict(wd=0.01, clip="off-null", gs=1.0)}[mode]
    _lamb_case(layout, sizes, mode, zero_norm=(2,), zero_grad=(1,), repeat=layout == "bert-base", **kw)
    torch.cuda.empty_cache()


def _fill_chunks(head, nchunks):
    """`head` segments, then one-chunk segments of assorted sizes until the plan has exactly `nchunks` chunks"""
    left = nchunks - sum(-(-s // CHUNK) for s in head)
    assert left >= 0
    return list(head) + [[CHUNK, 4100, CHUNK - 4, 20, 4][i % 5] for i in range(left)]


def _switch_sizes(case):
    grid = _sms() * 8
    head = [33 * CHUNK, 32 * CHUNK, 4, 12]
    return {
        "chunks=grid-1": lambda: _fill_chunks(head, grid - 1),
        "chunks=grid": lambda: _fill_chunks(head, grid),
        "chunks=grid+1": lambda: _fill_chunks(head, grid + 1),
        "segments of 32 and 33 chunks": lambda: [32 * CHUNK, 32 * CHUNK + 4, 33 * CHUNK, 4, 8],
        "nseg=1": lambda: [70 * CHUNK + 12],
        "nseg=8": lambda: [4 * (1 + (i * 7919) % 9000) for i in range(8)],
        "nseg=9": lambda: [4 * (1 + (i * 7919) % 9000) for i in range(8)] + [40 * CHUNK],
        "nseg=17": lambda: [4 * (1 + (i * 7919) % 9000) for i in range(16)] + [CHUNK + 4],
        "4-element segments": lambda: [4] * 50 + [8, 4, 12, 4],
    }[case]()


@pytest.mark.parametrize("case", ["chunks=grid-1", "chunks=grid", "chunks=grid+1", "segments of 32 and 33 chunks",
                                  "nseg=1", "nseg=8", "nseg=9", "nseg=17", "4-element segments"])
def test_lamb_switches(case):
    sizes = _switch_sizes(case)
    if case.startswith("chunks="):
        want = _sms() * 8 + {"chunks=grid-1": -1, "chunks=grid": 0, "chunks=grid+1": 1}[case]
        assert sum(-(-s // CHUNK) for s in sizes) == want
    for mode in ("default", "debias"):
        _lamb_case(case, sizes, mode, seed=len(sizes))


# ------------------------------------------------------------------ clip branches, all three optimizers
@pytest.mark.parametrize("clip", CLIPS)
@pytest.mark.parametrize("gs", [1.0, 0.125])
def test_clip_branches(clip, gs):
    n = _stream_sizes()["4B+5"]
    _adamw_case("4B+5", n, 2, 0.01, clip=clip, gs=gs)
    _madgrad_case("4B+5", n, 3, 0.0, 0.01, clip=clip, gs=gs)
    _lamb_case("uneven", [768, 4, 8192, 8196, 36, 3 * 8192 + 4, 100004, 65536], "default", clip=clip, gs=gs)


# ------------------------------------------------------------------ sumsq
def _sumsq_gate_terms(n, sms):
    n4 = n >> 2
    grid = max(1, min(-(-n4 // 256), sms * 8))
    per_thread = -(-n4 // (grid * 256)) + 3 + 1 + (1 if n & 3 else 0)   # float4 runs, 4-term sum, square, tail
    return per_thread, grid


def _sumsq_data(n, seed):
    gen = _gen(seed)
    x = _logmag(n, gen, -8, 3)
    x[torch.rand(n, device=DEV, generator=gen) < 0.05] = 0.0
    x[torch.randint(0, n, (max(1, n // 100000),), device=DEV, generator=gen)] = 1e6   # a few that dominate
    return x


@pytest.mark.parametrize("size", ["n=1", "n=5", "4B-1", "4B+5", "bert-base+3", "roberta-large+3"])
def test_sumsq(size):
    from dpr_scale_b200 import ops
    n = _stream_sizes()[size]
    x = _sumsq_data(n, 5)
    out = torch.zeros(1, device=DEV)
    ops.sumsq(x, out)
    want = _sumsq64(x)
    per_thread, grid = _sumsq_gate_terms(n, _sms())
    gate = (per_thread + 8 + grid) * U * want
    share = abs(float(out) - want) / gate
    print(f"sumsq {size}: n={n} grid={grid} |err| / gate {share:.4f} (gate {gate / want:.2e} relative)")
    assert share <= 1.0


def test_sumsq_accumulates_like_the_clip():
    """two encoder arenas, then the extra tensors, into one buffer that starts non-zero"""
    from dpr_scale_b200 import ops
    sms = _sms()
    parts = [_sumsq_data(n, 10 + i) for i, n in enumerate([4 * sms * 8 * 256 + 5, 3_000_001, 8192, 64, 5])]
    start = F32(123.456)
    out = torch.full((1,), start, device=DEV)
    for x in parts:
        ops.sumsq(x, out)
    want = start + sum(_sumsq64(x) for x in parts)
    terms = [_sumsq_gate_terms(x.numel(), sms) for x in parts]
    gate = (max(t[0] for t in terms) + 8 + sum(t[1] for t in terms) + 1) * U * want
    share = abs(float(out) - want) / gate
    print(f"sumsq accumulated over {len(parts)} calls: |err| / gate {share:.4f}")
    assert share <= 1.0


# ------------------------------------------------------------------ the wrappers at grad_scale 1/2
@pytest.mark.parametrize("which", ["adamw", "lamb", "madgrad"])
@pytest.mark.parametrize("clip", ["inactive", "active"])
def test_wrappers_at_half_grad_scale(which, clip):
    """The trainer sets grad_scale = 1/world_size; two ranks give 1/2.  Arena path and per-tensor path (_extra_coef)
    against float64, three steps on the same gradients, each step from the optimizer's own state."""
    from dpr_scale_b200.optim import FusedAdamW, FusedLamb, FusedMADGRAD
    from tests.test_optim_gpu import _task_with_projection
    task, batch = _task_with_projection()
    encs = [task.query_encoder, task.context_encoder]
    lr, wd, gs = 1e-2, 0.01, 0.5
    if which == "adamw":
        opt = FusedAdamW(task.parameters(), lr=lr, weight_decay=wd, grad_scale=gs)
    elif which == "lamb":
        opt = FusedLamb(task.parameters(), lr=lr, eps=1e-6, weight_decay=wd, grad_scale=gs)
    else:
        opt = FusedMADGRAD(task.parameters(), lr=lr, momentum=0.9, weight_decay=wd, grad_scale=gs)
    opt.attach_encoders(encs)
    opt.zero_grad()
    task.training_step(batch, 0).backward()
    arena_ids = {id(p) for e in encs for _, p, _ in e.transformer.arena_params()}
    extra = [p for p in task.parameters() if id(p) not in arena_ids and p.grad is not None]
    assert extra                                                 # the projection heads take the per-tensor path
    total = math.sqrt(sum(_sumsq64(e.grads) for e in encs) + sum(_sumsq64(p.grad) for p in extra)) * gs
    opt.max_grad_norm = {"active": 0.5, "inactive": 2.0}[clip] * total
    b1, b2 = opt.param_groups[0]["betas"] if which != "madgrad" else (0.9, 0.999)
    eps = opt.param_groups[0]["eps"]
    res = Shares()
    for step in range(1, 4):
        pre_arena = [(e.master.clone(), [t.clone() if isinstance(t, torch.Tensor) else t
                                         for t in opt._arena_state.get(id(e), ())]) for e in encs]
        pre_extra = [(p.detach().clone(), {k: t.clone() for k, t in opt.state[p].items()}) for p in extra]
        with torch.no_grad():
            opt.step()
        ss = opt.last_sumsq
        gmul, eg = _gmul(ss, gs, F32(opt.max_grad_norm))
        assert (eg == 0) == (clip == "inactive")
        for e, (p0, st0) in zip(encs, pre_arena):
            st = opt._arena_state[id(e)]
            z = torch.zeros_like(p0)
            if which == "adamw":
                m0, v0 = st0 if st0 else (z, z)
                _adamw_stages(res, (p0, m0, v0), (e.master, st[0], st[1]), e.grads, gmul, eg, F32(lr), F32(b1),
                              F32(b2), F32(eps), F32(wd), step)
            elif which == "lamb":
                m0, v0 = st0[:2] if st0 else (z, z)
                sizes = [math.prod(s) for _, s, _ in e.transformer.layout.entries]
                _lamb_arena_check(res, sizes, (p0, m0, v0), (e.master, st[0], st[1]), e.grads, gmul, eg,
                                  st[2].trust_scale().double(), F32(lr), F32(eps), F32(wd), 10.0)
            else:
                nu0, s0 = st0[:2]
                _madgrad_stages(res, (p0, nu0, s0), (e.master, st[0], st[1]), e.grads, st[2], gmul, eg, F32(lr),
                                F32(0.9), F32(wd), F32(eps), step - 1)
            res.equal("shadow", torch.equal(e.shadow, e.master.to(torch.bfloat16)))
        gmul_t, eg_t = gmul, eg          # _extra_coef repeats the kernel's fp32 clip arithmetic
        for p, (p0, st0) in zip(extra, pre_extra):
            st = opt.state[p]
            p1, g = p.detach().view(-1), p.grad.view(-1)
            p0 = p0.view(-1)
            if which == "adamw":
                m0, v0 = (st0["m"].view(-1), st0["v"].view(-1)) if st0 else (torch.zeros_like(p0),) * 2
                _adamw_stages(res, (p0, m0, v0), (p1, st["m"].view(-1), st["v"].view(-1)), g, gmul_t, eg_t, lr, b1,
                              b2, eps, wd, step, cu=1)
            elif which == "lamb":
                m0, v0 = ((st0["exp_avg"].view(-1), st0["exp_avg_sq"].view(-1)) if st0 else
                          (torch.zeros_like(p0),) * 2)
                _lamb_tensor_check(res, (p0, m0, v0), (p1, st["exp_avg"].view(-1), st["exp_avg_sq"].view(-1)), g,
                                   gmul_t, eg_t, lr, b1, b2, eps, wd, 10.0)
            else:
                nu0, s0 = ((st0["grad_sum_sq"].view(-1), st0["s"].view(-1)) if "grad_sum_sq" in st0 else
                           (torch.zeros_like(p0),) * 2)
                nu1 = st["grad_sum_sq"].view(-1).double()
                # torch takes nu ** (1/3) through powf (4 ulp) with the exponent in fp32
                root_u = 8 + torch.where(nu1 > 0, nu1.clamp(min=1e-300).log().abs(), torch.zeros_like(nu1)) * \
                    abs(F32(1 / 3) - 1 / 3) / U
                _madgrad_stages(res, (p0, nu0, s0), (p1, st["grad_sum_sq"].view(-1), st["s"].view(-1)), g,
                                st["x0"].view(-1), gmul_t, eg_t, lr, 0.9, wd, eps, step - 1, root_u=root_u, cu=1)
    res.done(f"{which} wrappers, grad_scale 1/2, clip {clip}, 3 steps")


def _lamb_arena_check(res, sizes, pre, post, g, gmul, eg, scale, step_size, eps, wd, clamp, adam=False):
    """LAMB stages over an arena of segments, given the kernel's per-segment step_size * trust; -> ||p||^2 per
    segment"""
    offs = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    pp, uu, aa = [], [], []
    for i in range(len(sizes)):
        sl = slice(offs[i], offs[i + 1])
        p0 = pre[0][sl]
        gg = g[sl].double() * gmul
        t1, t2 = B1 * pre[1][sl].double(), (1 - B1) * gg
        res.add("m", post[1][sl], t1 + t2, (2 * t1.abs() + (2 + eg) * t2.abs()) * U)
        t1, t2 = B2 * pre[2][sl].double(), (1 - B2) * gg * gg
        res.add("v", post[2][sl], t1 + t2, (2 * t1 + (3 + 2 * eg) * t2) * U)
        u, a = _lamb_u(p0, post[1][sl], post[2][sl], eps, wd)
        pp.append(p0.double().square().sum())
        uu.append(u.square().sum())
        aa.append(a.square().sum())
        res.add("p", post[0][sl], p0.double() - scale[i] * u, (p0.double().abs() + 6 * scale[i].abs() * a) * U)
    pp, uu, aa = torch.stack(pp), torch.stack(uu), torch.stack(aa)
    one = (pp == 0) | (uu == 0) | adam
    trust = torch.where(one, torch.ones_like(pp), pp.sqrt().clamp(max=clamp) / uu.sqrt().clamp(min=1e-300))
    chunks = [-(-s // CHUNK) for s in sizes]
    depth = torch.tensor([-(-c // 32) + 27 for c in chunks], dtype=torch.float64, device=DEV)
    rel = torch.where(one, torch.full_like(pp, U), _trust_rel(depth, aa, uu.clamp(min=1e-300)))
    res.add("trust", scale, step_size * trust, rel * step_size * trust)
    return pp


def _lamb_tensor_check(res, pre, post, g, gmul, eg, lr, b1, b2, eps, wd, clamp):
    """the per-tensor torch path: moments as the kernel's (cu = 1); p' against the float64 trust, whose error under
    torch's own summation order is taken as Wilkinson's n u"""
    p0, m0, v0 = (t.double() for t in pre)
    p1, m1, v1 = post
    gg = g.double() * gmul
    t1, t2 = b1 * m0, (1 - b1) * gg
    res.add("m", m1, t1 + t2, (3 * t1.abs() + (3 + eg) * t2.abs()) * U)
    t1, t2 = b2 * v0, (1 - b2) * gg * gg
    res.add("v", v1, t1 + t2, (3 * t1 + (4 + 2 * eg) * t2) * U)
    u, a = _lamb_u(p0, m1, v1, eps, wd)
    pp, uu, aa = p0.square().sum(), u.square().sum(), a.square().sum()
    one = bool(pp == 0) or bool(uu == 0)
    trust = 1.0 if one else float(min(float(pp.sqrt()), clamp) / uu.sqrt())
    tau = 0.0 if one else float(_trust_rel(p0.numel() + 2, aa, uu)) + 2 * U
    k = lr * trust
    res.add("p", p1, p0 - k * u, (2 * p0.abs() + 7 * abs(k) * a) * U + tau * abs(k) * u.abs())
