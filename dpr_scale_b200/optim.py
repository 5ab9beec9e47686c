"""Fused optimizers over the flat parameter arenas: the reference's three choices (conf/task/optim/adamw.yaml,
lamb.yaml, madgrad.yaml) executed by sm_90a kernels, one per encoder arena, with Lightning's global-norm clip
(``gradient_clip_val``, conf/trainer/gpu_1_host.yaml:8) and the bf16 shadow refresh folded in and no host sync.

- FusedAdamW: torch.optim.AdamW semantics, one kernel.
- FusedLamb: torch_optimizer.Lamb (0.3.x) semantics, trust ratio per parameter tensor (one ParamLayout entry).
- FusedMADGRAD: dpr_scale/optim/madgrad.py (dense branch) semantics, one kernel.

They are ``torch.optim.Optimizer`` subclasses so ``LambdaLR`` (dpr_task.py:144) drives ``param_groups[0]['lr']``
unchanged.  Parameters that are not arena-backed (the optional projection head) take a per-tensor torch path with the
same math.
"""
import math

import torch

from . import ops


class _ArenaOptimizer(torch.optim.Optimizer):
    """Encoder registration, the arena / extra-parameter split and the clip sum of squares shared by the fused
    optimizers.  Subclasses implement ``step``."""

    def __init__(self, params, defaults, max_grad_norm, grad_scale):
        super().__init__(params, defaults)
        self.max_grad_norm = float(max_grad_norm)
        self.grad_scale = float(grad_scale)  # e.g. 1/world_size after a SUM all-reduce
        self._encoders = []
        self._arena_state = {}
        self._step = 0
        self._sumsq = None
        self.last_sumsq = None

    def attach_encoders(self, encoders):
        """Register arena-backed encoders (dpr_scale_b200.models.hf_model.HFEncoder); de-duplicated."""
        seen = set()
        self._encoders = []
        for e in encoders:
            if id(e) not in seen:
                seen.add(id(e))
                self._encoders.append(e)

    def _arena_ptrs(self):
        s = set()
        for e in self._encoders:
            for _, p, _ in e.transformer.arena_params():
                s.add(id(p))
        return s

    def zero_grad(self, set_to_none: bool = False):
        for e in self._encoders:
            e.zero_grad()
        arena = self._arena_ptrs()
        for g in self.param_groups:
            for p in g["params"]:
                if id(p) not in arena:
                    p.grad = None

    def _extra_and_sumsq(self):
        """-> (parameters outside the arenas that have a gradient, device-side sum of squares of every gradient for the
        clip, or None when clipping is off)."""
        arena = self._arena_ptrs()
        extra = [p for g in self.param_groups for p in g["params"] if id(p) not in arena and p.grad is not None]
        dev = self._encoders[0].master.device if self._encoders else (extra[0].device if extra else None)
        sumsq = None
        if self.max_grad_norm > 0 and dev is not None:
            if self._sumsq is None or self._sumsq.device != dev:
                self._sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
            sumsq = self._sumsq
            sumsq.zero_()
            for e in self._encoders:
                ops.sumsq(e.grads, sumsq)
            for p in extra:
                ops.sumsq(p.grad.contiguous().view(-1), sumsq) if p.grad.is_cuda and p.grad.dtype == torch.float32 \
                    else sumsq.add_(p.grad.float().pow(2).sum())
            self.last_sumsq = sumsq
        return extra, sumsq

    def _extra_coef(self, sumsq):
        """The kernels' gradient multiplier for the per-tensor path: grad_scale times the clip coefficient."""
        coef = self.grad_scale
        if sumsq is not None:
            total = sumsq.sqrt() * self.grad_scale
            coef = self.grad_scale * torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0)
        return coef


class FusedAdamW(_ArenaOptimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 max_grad_norm=0.0, grad_scale=1.0):
        if amsgrad:
            raise ValueError("FusedAdamW: amsgrad is not supported (reference config uses amsgrad: false)")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults, max_grad_norm, grad_scale)

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._step += 1
        group = self.param_groups[0]
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        extra, sumsq = self._extra_and_sumsq()
        for e in self._encoders:
            st = self._arena_state.get(id(e))
            if st is None or st[0].device != e.master.device:
                st = (torch.zeros_like(e.master), torch.zeros_like(e.master))
                self._arena_state[id(e)] = st
            ops.adamw_step(e.master, e.grads, st[0], st[1], e.shadow, lr, b1, b2, eps, wd, self._step,
                           self.grad_scale, sumsq, self.max_grad_norm)
            e.mark_shadow_fresh()
        if extra:
            coef = self._extra_coef(sumsq)
            for p in extra:
                st = self.state[p]
                if not st:
                    st["m"], st["v"] = torch.zeros_like(p), torch.zeros_like(p)
                g = p.grad * coef
                p.mul_(1.0 - lr * wd)
                st["m"].mul_(b1).add_(g, alpha=1.0 - b1)
                st["v"].mul_(b2).addcmul_(g, g, value=1.0 - b2)
                denom = st["v"].sqrt() / math.sqrt(1.0 - b2 ** self._step) + eps
                p.addcdiv_(st["m"], denom, value=-lr / (1.0 - b1 ** self._step))
        return loss


class FusedLamb(_ArenaOptimizer):
    """torch_optimizer.Lamb: Adam moments without bias correction, u = m / (sqrt(v) + eps) + wd * p, and a per-tensor
    trust ratio min(||p||, clamp_value) / ||u||.  The arena kernels reduce the norms in a fixed order, so given the
    same gradients and clip sum of squares the update is bitwise repeatable and no rank-dependent bit enters the trust
    ratios."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0, clamp_value=10, adam=False,
                 debias=False, max_grad_norm=0.0, grad_scale=1.0):
        betas = tuple(betas)
        if lr <= 0.0:
            raise ValueError(f"FusedLamb: invalid learning rate {lr}")
        if eps < 0.0:
            raise ValueError(f"FusedLamb: invalid epsilon {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"FusedLamb: invalid betas {betas}")
        if weight_decay < 0:
            raise ValueError(f"FusedLamb: invalid weight_decay {weight_decay}")
        if clamp_value < 0.0:
            raise ValueError(f"FusedLamb: invalid clamp value {clamp_value}")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults, max_grad_norm, grad_scale)
        self.clamp_value = float(clamp_value)
        self.adam = bool(adam)
        self.debias = bool(debias)

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._step += 1
        group = self.param_groups[0]
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        extra, sumsq = self._extra_and_sumsq()
        for e in self._encoders:
            st = self._arena_state.get(id(e))
            if st is None or st[0].device != e.master.device:
                # one segment per parameter tensor, in arena order (ParamLayout packs them back to back)
                plan = ops.LambPlan([math.prod(s) for _, s, _ in e.transformer.layout.entries], e.master.device)
                st = (torch.zeros_like(e.master), torch.zeros_like(e.master), plan)
                self._arena_state[id(e)] = st
            ops.lamb_step(e.master, e.grads, st[0], st[1], e.shadow, st[2], lr, b1, b2, eps, wd, self.clamp_value,
                          self.adam, self.debias, self._step, self.grad_scale, sumsq, self.max_grad_norm)
            e.mark_shadow_fresh()
        if extra:
            coef = self._extra_coef(sumsq)
            step_size = lr
            if self.debias:
                step_size = lr * math.sqrt(1.0 - b2 ** self._step) / (1.0 - b1 ** self._step)
            for p in extra:
                st = self.state[p]
                if not st:
                    st["exp_avg"], st["exp_avg_sq"] = torch.zeros_like(p), torch.zeros_like(p)
                g = p.grad * coef
                st["exp_avg"].mul_(b1).add_(g, alpha=1.0 - b1)
                st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1.0 - b2)
                u = st["exp_avg"] / st["exp_avg_sq"].sqrt().add(eps)
                if wd != 0:
                    u.add_(p, alpha=wd)
                w_norm = p.norm().clamp(0, self.clamp_value)
                u_norm = u.norm()
                trust = torch.where((w_norm == 0) | (u_norm == 0), torch.ones_like(w_norm), w_norm / u_norm)
                if self.adam:
                    trust = torch.ones_like(trust)
                p.sub_(u * (trust * step_size))
        return loss


class FusedMADGRAD(_ArenaOptimizer):
    """dpr_scale/optim/madgrad.py (dense gradients): dual averaging with a cube-root denominator.  Its quirks are kept:
    the step uses lr + eps (so it is not zero while warmup holds the scheduled lr at 0), lamb = (lr + eps) * sqrt(k + 1)
    with k counting steps from 0, weight decay is coupled (g += wd * p), and with momentum != 0 x0 is the parameters'
    value when the optimizer is built."""

    def __init__(self, params, lr=1e-2, momentum=0.9, weight_decay=0, eps=1e-6, k=0, decouple_decay=False,
                 max_grad_norm=0.0, grad_scale=1.0):
        if decouple_decay:
            raise ValueError("FusedMADGRAD: decouple_decay is not supported (the reference's MADGRAD couples decay)")
        if momentum < 0 or momentum >= 1:
            raise ValueError(f"FusedMADGRAD: momentum {momentum} must be in the range [0,1)")
        if lr <= 0:
            raise ValueError(f"FusedMADGRAD: learning rate {lr} must be positive")
        if weight_decay < 0:
            raise ValueError(f"FusedMADGRAD: weight decay {weight_decay} must be non-negative")
        if eps < 0:
            raise ValueError("FusedMADGRAD: eps must be non-negative")
        defaults = dict(lr=lr, eps=eps, momentum=momentum, weight_decay=weight_decay, k=int(k))
        super().__init__(params, defaults, max_grad_norm, grad_scale)
        self.momentum = float(momentum)
        if self.momentum != 0:
            for g in self.param_groups:
                for p in g["params"]:
                    self.state[p]["x0"] = p.detach().clone()

    def attach_encoders(self, encoders):
        """Registers the encoders and gathers the x0 snapshots of their parameters into one flat copy per arena."""
        super().attach_encoders(encoders)
        for e in self._encoders:
            if id(e) in self._arena_state:
                continue
            x0 = None
            if self.momentum != 0:
                x0 = torch.empty_like(e.master)
                for _, p, off in e.transformer.arena_params():
                    snap = self.state[p].pop("x0", None) if p in self.state else None
                    x0[off:off + p.numel()].copy_((snap if snap is not None else p.detach()).view(-1))
            self._arena_state[id(e)] = (torch.zeros_like(e.master), torch.zeros_like(e.master), x0)

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        group = self.param_groups[0]
        lr, eps, wd, mom, k = group["lr"], group["eps"], group["weight_decay"], group["momentum"], group["k"]
        extra, sumsq = self._extra_and_sumsq()
        for e in self._encoders:
            st = self._arena_state.get(id(e))
            if st is None or st[0].device != e.master.device:
                st = (torch.zeros_like(e.master), torch.zeros_like(e.master),
                      e.master.detach().clone() if mom != 0 else None)
                self._arena_state[id(e)] = st
            ops.madgrad_step(e.master, e.grads, st[0], st[1], st[2], e.shadow, lr, mom, wd, eps, k, self.grad_scale,
                             sumsq, self.max_grad_norm)
            e.mark_shadow_fresh()
        if extra:
            coef = self._extra_coef(sumsq)
            lamb = (lr + eps) * math.sqrt(k + 1)
            for p in extra:
                st = self.state[p]
                if "grad_sum_sq" not in st:
                    st["grad_sum_sq"], st["s"] = torch.zeros_like(p), torch.zeros_like(p)
                    if mom != 0 and "x0" not in st:
                        st["x0"] = p.detach().clone()
                g = p.grad * coef
                if wd != 0:
                    g.add_(p, alpha=wd)
                nu, s = st["grad_sum_sq"], st["s"]
                x0 = st["x0"] if mom != 0 else p.addcdiv(s, nu.pow(1 / 3).add_(eps), value=1)
                nu.addcmul_(g, g, value=lamb)
                s.add_(g, alpha=lamb)
                z = x0.addcdiv(s, nu.pow(1 / 3).add_(eps), value=-1)
                if mom == 0:
                    p.copy_(z)
                else:
                    p.mul_(mom).add_(z, alpha=1 - mom)
        group["k"] = k + 1
        return loss
