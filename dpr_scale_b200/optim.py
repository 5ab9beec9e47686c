"""FusedAdamW — torch.optim.AdamW semantics (conf/task/optim/adamw.yaml of the reference) executed by ONE
sm_90a kernel per encoder arena: global-norm clip (Lightning's ``gradient_clip_val``,
conf/trainer/gpu_1_host.yaml:8) + decoupled-weight-decay Adam + bf16 shadow refresh, no host sync.

It is a ``torch.optim.Optimizer`` so ``LambdaLR`` (dpr_task.py:144) drives ``param_groups[0]['lr']`` unchanged.
Parameters that are not arena-backed (the optional projection head) take a plain per-tensor path.
"""
import math

import torch

from . import ops


class FusedAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 max_grad_norm=0.0, grad_scale=1.0):
        if amsgrad:
            raise ValueError("FusedAdamW: amsgrad is not supported (reference config uses amsgrad: false)")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay)
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

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self._step += 1
        group = self.param_groups[0]
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
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
        for e in self._encoders:
            st = self._arena_state.get(id(e))
            if st is None or st[0].device != e.master.device:
                st = (torch.zeros_like(e.master), torch.zeros_like(e.master))
                self._arena_state[id(e)] = st
            ops.adamw_step(e.master, e.grads, st[0], st[1], e.shadow, lr, b1, b2, eps, wd, self._step,
                           self.grad_scale, sumsq, self.max_grad_norm)
            e.mark_shadow_fresh()
        if extra:
            coef = self.grad_scale
            if sumsq is not None:
                total = sumsq.sqrt() * self.grad_scale
                coef = self.grad_scale * torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0)
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
