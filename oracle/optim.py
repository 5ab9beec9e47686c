"""float64 restatements of the LAMB and MADGRAD updates (next to task.adamw_step), per parameter tensor, in place.

lamb_step: torch_optimizer.Lamb 0.3.x as configured by conf/task/optim/lamb.yaml.
madgrad_step: the dense branch of dpr_scale/optim/madgrad.py as configured by conf/task/optim/madgrad.yaml.
"""
import math


def lamb_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0, clamp_value=10.0, adam=False,
              debias=False):
    """One LAMB update of one tensor; returns the trust ratio used."""
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    step_size = lr * (math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step) if debias else 1.0)
    u = m / (v.sqrt() + eps) + weight_decay * p
    w_norm = min(float(p.norm()), clamp_value)
    u_norm = float(u.norm())
    trust = 1.0 if (w_norm == 0 or u_norm == 0 or adam) else w_norm / u_norm
    p.sub_(step_size * trust * u)
    return trust


def madgrad_state(p, momentum):
    """The reference's initialize_state: zero sums, and x0 = p when momentum != 0."""
    st = {"grad_sum_sq": p.new_zeros(p.shape), "s": p.new_zeros(p.shape)}
    if momentum != 0:
        st["x0"] = p.clone()
    return st


def madgrad_step(p, g, state, k, lr, momentum=0.9, weight_decay=0.0, eps=1e-6):
    """One MADGRAD update of one tensor at step k (counting from 0)."""
    lamb = (lr + eps) * math.sqrt(k + 1)
    if weight_decay != 0:
        g = g + weight_decay * p
    nu, s = state["grad_sum_sq"], state["s"]
    x0 = state["x0"] if momentum != 0 else p + s / (nu ** (1 / 3) + eps)
    nu.add_(lamb * g * g)
    s.add_(lamb * g)
    z = x0 - s / (nu ** (1 / 3) + eps)
    if momentum == 0:
        p.copy_(z)
    else:
        p.mul_(momentum).add_((1 - momentum) * z)
