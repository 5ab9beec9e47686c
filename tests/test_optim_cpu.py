"""CPU tests of the LAMB and MADGRAD optimizers: the float64 oracles (MADGRAD against the reference's own optimizer,
tests/golden/optim_madgrad.npz; LAMB against hand-computed single steps), the per-tensor path of FusedLamb /
FusedMADGRAD, the LAMB chunk plan, config composition and keyword checks."""
import math

import numpy as np
import pytest
import torch

from oracle import optim as oopt
from tests.util import load_golden

B1, B2 = 0.9, 0.999
C1 = (1 - B1) / math.sqrt(1 - B2)   # |u| of every element after the first step when eps = 0 and wd = 0


def _madgrad_cases():
    g = load_golden("optim_madgrad.npz")
    names = sorted({k.split("/")[0] for k in g if "/" in k})
    return g, names


def test_madgrad_oracle_matches_reference_golden():
    g, names = _madgrad_cases()
    assert set(names) == {"m09_wd", "m0_wd", "m09", "m0_eps"}
    lrs = g["lrs"].tolist()
    assert lrs[0] == 0.0                                        # a warmup step with the scheduled rate at 0
    for name in names:
        momentum, wd, eps = g[f"{name}/hyper"].tolist()
        ps = [g[f"{name}/p0/{i}"].double().clone() for i in range(int(g["num_params"]))]
        states = [oopt.madgrad_state(p, momentum) for p in ps]
        for k, lr in enumerate(lrs):
            for i, (p, st) in enumerate(zip(ps, states)):
                oopt.madgrad_step(p, g[f"{name}/g/{k}/{i}"].double(), st, k, lr, momentum, wd, eps)
                want = g[f"{name}/p/{k}/{i}"].double()
                assert torch.allclose(p, want, rtol=1e-5, atol=1e-6), (name, k, i, float((p - want).abs().max()))
                if k == 0:
                    assert not torch.equal(p, g[f"{name}/p0/{i}"].double())   # lr = 0 still moves p (lr + eps)
        for i, st in enumerate(states):
            assert torch.allclose(st["grad_sum_sq"], g[f"{name}/grad_sum_sq/{i}"].double(), rtol=1e-5, atol=1e-9)
            assert torch.allclose(st["s"], g[f"{name}/s/{i}"].double(), rtol=1e-5, atol=1e-9)


def _t(xs):
    return torch.tensor(xs, dtype=torch.float64)


def _lamb_one(p, g, **kw):
    p, g = _t(p), _t(g)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    trust = oopt.lamb_step(p, g, m, v, 1, 0.01, B1, B2, **kw)
    return p, trust


def test_lamb_oracle_first_step_closed_form():
    # eps = 0, wd = 0: u = C1 * sign(g), so trust * u = ||p|| / sqrt(n) * sign(g)
    p, trust = _lamb_one([3.0, -4.0, 0.0, 0.0], [1.0, -2.0, 0.5, -0.1], eps=0.0)
    assert trust == pytest.approx(5.0 / (C1 * 2.0), rel=1e-12)
    want = _t([3.0, -4.0, 0.0, 0.0]) - 0.01 * 2.5 * _t([1.0, -1.0, 1.0, -1.0])
    assert torch.allclose(p, want, rtol=0, atol=1e-12)
    # weight decay enters u before the norm: u = C1 * sign(g) + wd * p
    p, trust = _lamb_one([3.0, 4.0], [1.0, 1.0], eps=0.0, weight_decay=0.5)
    u = _t([C1 + 1.5, C1 + 2.0])
    assert trust == pytest.approx(5.0 / float(u.norm()), rel=1e-12)
    assert torch.allclose(p, _t([3.0, 4.0]) - 0.01 * trust * u, rtol=0, atol=1e-12)


def test_lamb_oracle_zero_weight_norm_gives_trust_one():
    p, trust = _lamb_one([0.0, 0.0, 0.0, 0.0], [1.0, -1.0, 2.0, -3.0], eps=0.0)
    assert trust == 1.0
    assert torch.allclose(p, -0.01 * C1 * _t([1.0, -1.0, 1.0, -1.0]), rtol=0, atol=1e-12)
    p, trust = _lamb_one([1.0, 2.0], [0.0, 0.0], eps=1e-8)            # u = 0 -> trust 1, p unchanged
    assert trust == 1.0 and torch.equal(p, _t([1.0, 2.0]))


def test_lamb_oracle_weight_norm_clamp():
    p, trust = _lamb_one([12.0, 16.0], [1.0, 1.0], eps=0.0)            # ||p|| = 20 -> clamped to 10
    assert trust == pytest.approx(10.0 / (C1 * math.sqrt(2.0)), rel=1e-12)
    assert torch.allclose(p, _t([12.0, 16.0]) - 0.01 * 10.0 / math.sqrt(2.0), rtol=0, atol=1e-12)
    p, trust = _lamb_one([12.0, 16.0], [1.0, 1.0], eps=0.0, clamp_value=30.0)
    assert trust == pytest.approx(20.0 / (C1 * math.sqrt(2.0)), rel=1e-12)


def test_lamb_oracle_debias_and_adam():
    step_size = 0.01 * math.sqrt(1 - B2) / (1 - B1)
    p, trust = _lamb_one([3.0, -4.0, 0.0, 0.0], [1.0, -2.0, 0.5, -0.1], eps=0.0, debias=True)
    want = _t([3.0, -4.0, 0.0, 0.0]) - step_size * 2.5 * _t([1.0, -1.0, 1.0, -1.0])
    assert torch.allclose(p, want, rtol=0, atol=1e-12)
    p, trust = _lamb_one([3.0, -4.0], [1.0, -2.0], eps=0.0, adam=True)
    assert trust == 1.0
    assert torch.allclose(p, _t([3.0 - 0.01 * C1, -4.0 + 0.01 * C1]), rtol=0, atol=1e-12)


def _seeded_params(seed, shapes=((6, 5), (17,), (3, 4))):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes], g


def test_fused_madgrad_tensor_path_matches_reference_golden():
    """Without arenas every parameter takes FusedMADGRAD's per-tensor path: it must reproduce the reference."""
    from dpr_scale_b200.optim import FusedMADGRAD
    g, names = _madgrad_cases()
    for name in names:
        momentum, wd, eps = g[f"{name}/hyper"].tolist()
        params = [torch.nn.Parameter(g[f"{name}/p0/{i}"].clone()) for i in range(int(g["num_params"]))]
        opt = FusedMADGRAD(params, lr=1e-2, momentum=momentum, weight_decay=wd, eps=eps)
        for k, lr in enumerate(g["lrs"].tolist()):
            opt.param_groups[0]["lr"] = lr
            for i, p in enumerate(params):
                p.grad = g[f"{name}/g/{k}/{i}"].clone()
            opt.step()
            for i, p in enumerate(params):
                assert torch.allclose(p.detach(), g[f"{name}/p/{k}/{i}"], rtol=1e-6, atol=1e-7), (name, k, i)
        assert opt.param_groups[0]["k"] == len(g["lrs"])


@pytest.mark.parametrize("kw", [dict(), dict(weight_decay=0.01, debias=True), dict(adam=True, clamp_value=0.5)])
def test_fused_lamb_tensor_path_matches_oracle(kw):
    from dpr_scale_b200.optim import FusedLamb
    params, g = _seeded_params(3)
    ref = [p.detach().double().clone() for p in params]
    mom = [(torch.zeros_like(r), torch.zeros_like(r)) for r in ref]
    opt = FusedLamb(params, lr=0.02, eps=1e-6, max_grad_norm=1.0, grad_scale=0.5, **kw)
    for step in range(1, 4):
        grads = [torch.randn(p.shape, generator=g) * 2 for p in params]
        for p, gr in zip(params, grads):
            p.grad = gr.clone()
        opt.step()
        total = math.sqrt(sum(float(((0.5 * gr.double()) ** 2).sum()) for gr in grads))
        coef = 0.5 * min(1.0, 1.0 / (total + 1e-6))
        for r, (m, v), gr in zip(ref, mom, grads):
            oopt.lamb_step(r, coef * gr.double(), m, v, step, 0.02, eps=1e-6, **kw)
    for p, r in zip(params, ref):
        assert torch.allclose(p.detach().double(), r, rtol=1e-5, atol=1e-6)


def test_lamb_plan_chunks_never_straddle_segments():
    from dpr_scale_b200 import ops
    sizes = [768, 8192, 8196, 20, 3 * 8192 + 4, 4]
    pl = ops.LambPlan(sizes, "cpu", chunk=8192)
    plan = pl.plan.numpy()
    C, S = pl.nchunks, pl.nseg
    off, seg, seg_chunk = plan[:C + 1], plan[C + 1:2 * C + 1], plan[2 * C + 1:]
    assert S == len(sizes) and C == 1 + 1 + 2 + 1 + 4 + 1 and len(seg_chunk) == S + 1
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    assert off[0] == 0 and off[-1] == bounds[-1] and (np.diff(off) > 0).all() and (np.diff(off) <= 8192).all()
    assert (off % 4 == 0).all()
    for c in range(C):
        s = seg[c]
        assert bounds[s] <= off[c] and off[c + 1] <= bounds[s + 1]
        assert seg_chunk[s] <= c < seg_chunk[s + 1]
    assert pl.workspace.numel() >= 4 * (2 * C + S)
    with pytest.raises(ValueError):
        ops.LambPlan([768, 6], "cpu")            # segment not a multiple of 4
    with pytest.raises(ValueError):
        ops.LambPlan([], "cpu")


def test_optim_configs_compose_to_the_fused_classes():
    from dpr_scale_b200.optim import FusedLamb, FusedMADGRAD
    from dpr_scale_b200.utils.config import compose, instantiate
    params = [torch.nn.Parameter(torch.zeros(4))]
    cfg = compose("config", ["task/optim=lamb"])
    o = cfg.task.optim
    assert o._target_ == "dpr_scale_b200.optim.FusedLamb"
    assert o.lr == 1e-5 and list(o.betas) == [0.9, 0.999] and o.eps == 1e-8 and o.weight_decay == 0
    opt = instantiate(o, params)
    assert isinstance(opt, FusedLamb) and opt.param_groups[0]["lr"] == 1e-5 and opt.param_groups[0]["eps"] == 1e-8
    assert opt.clamp_value == 10 and opt.adam is False and opt.debias is False
    cfg = compose("config", ["task/optim=madgrad"])
    o = cfg.task.optim
    assert o._target_ == "dpr_scale_b200.optim.FusedMADGRAD"
    assert o.lr == 1e-3 and o.eps == 1e-6 and o.weight_decay == 0 and o.momentum == 0.9
    opt = instantiate(o, params)
    assert isinstance(opt, FusedMADGRAD)
    grp = opt.param_groups[0]
    assert (grp["lr"], grp["eps"], grp["weight_decay"], grp["momentum"], grp["k"]) == (1e-3, 1e-6, 0, 0.9, 0)


def test_unsupported_keywords_and_values_raise():
    from dpr_scale_b200.optim import FusedAdamW, FusedLamb, FusedMADGRAD
    params = [torch.nn.Parameter(torch.zeros(4))]
    with pytest.raises(ValueError):
        FusedMADGRAD(params, decouple_decay=True)
    with pytest.raises(ValueError):
        FusedAdamW(params, amsgrad=True)
    for bad in (dict(lr=0.0), dict(eps=-1.0), dict(betas=(1.0, 0.999)), dict(weight_decay=-0.1),
                dict(clamp_value=-1.0)):
        with pytest.raises(ValueError):
            FusedLamb(params, **bad)
    for bad in (dict(lr=0.0), dict(momentum=1.0), dict(weight_decay=-0.1), dict(eps=-1.0)):
        with pytest.raises(ValueError):
            FusedMADGRAD(params, **bad)
