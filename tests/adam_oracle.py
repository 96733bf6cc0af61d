"""fp64 restatement of one fused optimiser update (sparf_b200.optim.FusedAdam.step, csrc/optim.cu::sparf_adam_step):
skip on a non-finite gradient, clip_grad_norm_, Adam (amsgrad=False, weight_decay=0), ExponentialLR x linear warm-up,
and the two step counters.  Pinned against torch's own optimiser in tests/test_adam_oracle_cpu.py.

All arithmetic is the textbook formula in float64; nothing mimics an fp32 rounding or an evaluation order.
"""
from dataclasses import dataclass

import torch


@dataclass
class Hyper:
    lr0: float
    gamma: float = 1.0
    warmup: float = 0.0         # 0: no warm-up
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    max_norm: float = 0.0       # 0: no clipping


def lr_at(h: Hyper, k: int) -> float:
    """Learning rate of iteration k (1-based): lr0 * gamma^(k-1) * min(1, k / warmup)."""
    lr = h.lr0 * h.gamma ** (k - 1)
    if h.warmup > 0:
        lr *= min(1.0, k / h.warmup)
    return lr


def clip_coef(h: Hyper, grad: torch.Tensor) -> float:
    """clip_grad_norm_'s factor: max_norm / (||g|| + 1e-6), at most 1 (1 without clipping)."""
    if h.max_norm <= 0:
        return 1.0
    return min(1.0, h.max_norm / (grad.double().norm().item() + 1e-6))


def step(h: Hyper, param, grad, exp_avg, exp_avg_sq, steps):
    """One update from (param, grad, exp_avg, exp_avg_sq) and steps = (updates taken, iterations seen).

    Returns float64 tensors (param, grad, exp_avg, exp_avg_sq) after the update, where grad is the clipped gradient,
    and the new steps.  A non-finite gradient skips everything but the iteration counter."""
    p, g, m, v = (x.double() for x in (param, grad, exp_avg, exp_avg_sq))
    t, k = int(steps[0]), int(steps[1])
    k += 1
    if not torch.isfinite(g).all():
        return p, g, m, v, (t, k)
    t += 1
    g = g * clip_coef(h, g)
    m = m + (1 - h.beta1) * (g - m)
    v = h.beta2 * v + (1 - h.beta2) * g * g
    bc1, bc2 = 1 - h.beta1 ** t, 1 - h.beta2 ** t
    denom = torch.sqrt(v) / bc2 ** 0.5 + h.eps
    p = p - lr_at(h, k) / bc1 * m / denom
    return p, g, m, v, (t, k)
