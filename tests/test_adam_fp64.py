"""One fused optimiser update (sparf_b200.optim.FusedAdam.step: csrc/optim.cu's grad_stats_kernel + adam_kernel) from a
random state against the fp64 restatement in tests/adam_oracle.py on the same fp32 inputs, element by element.

Gates, in units of u = 2^-24 (the fp32 unit round-off) of each quantity's natural scale, from the kernel's operations
(each rounded fp32 operation, and each fp32 rounding of an fp64 scalar, adds at most u/2 of its result):
  grad  B_G = 4 u |g|.  The clip factor max_norm / (norm + 1e-6) takes five roundings (the norm's cast to fp32 counts
        half through the square root): <= 2.25 u relative; applying it to g adds u/2.
  m     B_M = 8 u max(|m|, |g|).  m + w1 (g - m) (or g - (g - m)(1 - w1) for w1 >= 0.5): the clipped g carries 3 u,
        the rounding of w1, the subtraction, the product and the sum at most u each at this scale (|g - m| <= 2 scale,
        w1 <= 1): 6.5 u.
  v     B_V = 10 u max(|v|, g^2).  b2 v + w2 g^2 adds two non-negative terms: g^2 carries 2 * 3 u from the clip and
        u/2 from the square, each coefficient and product u/2 more, the sum u/2: <= 8 u of v' itself.
  p     B_P = 16 u (|p| + lr / bc1 * max(|m|, |g|) / denom).  denom = sqrt(v') / sqrt(bc2) + eps: v's 8 u halves through
        the square root, plus the root, the scalar sqrt(bc2), the division, eps and the sum: <= 6.5 u.  m' / denom then
        errs by <= 6.5 u of max(|m|, |g|) / denom plus 8 u of |m'| / denom, the fp32 step size and the product one u
        more: 15 u of the update's scale; the final sum u/2 of |p'|.
The scale of p is |p| plus the update's size at m's natural scale (not at |m'|, which may cancel to ~0).

Cases: n in {1, 255, 256, 257, T - 1, T + 1, 1.2 M} with T = 8 * 256 * (the device's SM count), the element count
above which the launch's num_sms * 8 blocks of 256 threads grid-stride (an H100 with 132 SMs: T = 270 336; every
default network is larger); w1 = 1 - beta1 below 0.5, and at and above 0.5 (the two branches of Tensor.lerp_);
clipping active, inactive and off; iteration k below and above the warm-up.  A NaN or a +Inf gradient skips the
update: param, exp_avg, exp_avg_sq and grad keep their bits, only the iteration counter advances, and the next finite
step matches the oracle again.  After every step scratch (the gradient statistics and the last-block-out counter) is
zero and the counters are the oracle's.

Worst error / gate over all cases, measured on an H100 80GB HBM3 (700 W power limit): grad 0.16, m 0.18, v 0.22,
p 0.21.
"""
import pytest
import torch

import adam_oracle as A

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
B_G, B_M, B_V, B_P = 4.0, 8.0, 10.0, 16.0

CONFIGS = {
    # beta1 0.9: w1 = 0.1 < 0.5; clip active; k = 5 < warm-up 50
    "w1_0.1_clip_warmup": dict(hyper=dict(lr0=1e-3, gamma=0.999, warmup=50.0, beta1=0.9, beta2=0.999, eps=1e-8),
                               clip=0.3, steps=(3, 4)),
    # beta1 0.3: w1 = 0.7 >= 0.5; clip inactive (max_norm 10x the norm); k = 41 > warm-up 10
    "w1_0.7_noclip_after_warmup": dict(hyper=dict(lr0=5e-3, gamma=0.97, warmup=10.0, beta1=0.3, beta2=0.9, eps=1e-6),
                                       clip=10.0, steps=(30, 40)),
    # beta1 0.5: w1 = 0.5 exactly (the >= branch); no clipping; first update (largest bias corrections)
    "w1_0.5_off_first": dict(hyper=dict(lr0=2e-3, gamma=1.0, beta1=0.5, beta2=0.99, eps=1e-8), clip=0.0, steps=(0, 0)),
}


def _threshold():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


def _sizes():
    T = _threshold()
    return [1, 255, 256, 257, T - 1, T + 1, 1_200_000]


def _state(n, seed):
    """Random fp32 (param, grad, exp_avg, exp_avg_sq) spanning three decades, with some exact zeros."""
    g = torch.Generator(device="cuda").manual_seed(seed)

    def mag():
        return 10.0 ** (-3 * torch.rand(n, device="cuda", generator=g))

    p = torch.randn(n, device="cuda", generator=g)
    grad = torch.randn(n, device="cuda", generator=g) * mag()
    m = 0.1 * torch.randn(n, device="cuda", generator=g) * mag()
    v = (torch.randn(n, device="cuda", generator=g) * mag()) ** 2
    grad[5::17] = 0
    m[7::23] = 0
    v[11::29] = 0
    return p, grad, m, v


def _fused(n, hyper, max_norm, state, steps):
    from sparf_b200.optim import FlatParameters, FusedAdam
    mod = torch.nn.Module()
    mod.p = torch.nn.Parameter(torch.zeros(n, device="cuda"))
    flat = FlatParameters([mod])
    adam = FusedAdam(flat, lr=hyper.lr0, betas=(hyper.beta1, hyper.beta2), eps=hyper.eps, gamma=hyper.gamma,
                     warmup_steps=hyper.warmup, max_norm=max_norm or None)
    p, grad, m, v = state
    flat.flat_param.copy_(p)
    flat.flat.copy_(grad)
    adam.exp_avg.copy_(m)
    adam.exp_avg_sq.copy_(v)
    adam.steps.copy_(torch.tensor(steps))
    return flat, adam


def _ratio(got, want, scale, bound):
    """max |got - want| / (bound u scale), elementwise (0 where both error and scale are 0)."""
    err = (got.double() - want).abs()
    lim = bound * ULP * scale
    assert torch.isfinite(err).all()
    return (err / lim.clamp_min(1e-300)).max().item() if (err > 0).any() else 0.0


def _check_step(flat, adam, hyper, state, steps):
    """One step of the fused kernels against the oracle; returns the worst ratio per quantity."""
    p0, g0, m0, v0 = (x.double() for x in state)
    adam.step()
    p, g, m, v, st = A.step(hyper, p0, g0, m0, v0, steps)
    assert adam.steps.tolist() == list(st)
    assert (adam.scratch.view(torch.int64) == 0).all(), adam.scratch
    t, k = st
    s_m = torch.maximum(m0.abs(), g0.abs())
    denom = torch.sqrt(v) / (1 - hyper.beta2 ** t) ** 0.5 + hyper.eps
    s_p = p0.abs() + A.lr_at(hyper, k) / (1 - hyper.beta1 ** t) * s_m / denom
    ratios = dict(grad=_ratio(flat.flat, g, g0.abs(), B_G), m=_ratio(adam.exp_avg, m, s_m, B_M),
                  v=_ratio(adam.exp_avg_sq, v, torch.maximum(v0, g0 * g0), B_V),
                  p=_ratio(flat.flat_param, p, s_p, B_P))
    return ratios


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("size", range(7), ids=["1", "255", "256", "257", "T-1", "T+1", "1.2M"])
def test_fused_adam_step_matches_fp64(size, config):
    n = _sizes()[size]
    c = CONFIGS[config]
    hyper = A.Hyper(**c["hyper"])
    state = _state(n, seed=size * 10 + list(CONFIGS).index(config))
    max_norm = c["clip"] * state[1].double().norm().item()
    hyper.max_norm = max_norm
    if max_norm:
        assert (A.clip_coef(hyper, state[1]) < 1) == (c["clip"] < 1)
    flat, adam = _fused(n, hyper, max_norm, state, c["steps"])
    ratios = _check_step(flat, adam, hyper, state, c["steps"])
    print("adam n=%-8d %-28s worst error / gate: %s" % (n, config, "  ".join("%s %.3f" % kv for kv in ratios.items())))
    for what, r in ratios.items():
        assert r <= 1.0, (what, r)
    if c["clip"] == 10.0:       # inactive clip: the gradient is left as it was
        assert torch.equal(flat.flat, state[1])


@pytest.mark.parametrize("bad", [float("nan"), float("inf")], ids=["nan", "inf"])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("size", [3, 5], ids=["257", "T+1"])
def test_fused_adam_skips_non_finite_gradient(size, where, bad):
    """A non-finite gradient anywhere (the first or the last block) skips the update bit for bit while the schedule
    advances; the next finite gradient is applied as the oracle applies it (the skip flag did not stick)."""
    n = _sizes()[size]
    c = CONFIGS["w1_0.1_clip_warmup"]
    hyper = A.Hyper(**c["hyper"])
    state = _state(n, seed=99 + size)
    hyper.max_norm = 0.3 * state[1].double().norm().item()
    flat, adam = _fused(n, hyper, hyper.max_norm, state, c["steps"])
    flat.flat[0 if where == "first" else n - 1] = bad
    before = [x.clone() for x in (flat.flat_param, flat.flat, adam.exp_avg, adam.exp_avg_sq)]
    adam.step()
    steps = (c["steps"][0], c["steps"][1] + 1)
    assert adam.steps.tolist() == list(steps)
    assert (adam.scratch.view(torch.int64) == 0).all(), adam.scratch
    after = (flat.flat_param, flat.flat, adam.exp_avg, adam.exp_avg_sq)
    for b, a in zip(before, after):
        assert torch.equal(b.view(torch.int32), a.view(torch.int32))
    flat.flat.copy_(state[1])
    state = (flat.flat_param.clone(), state[1], adam.exp_avg.clone(), adam.exp_avg_sq.clone())
    ratios = _check_step(flat, adam, hyper, state, steps)
    print("adam n=%-8d %s %-5s then finite: %s" % (n, where, bad, "  ".join("%s %.3f" % kv for kv in ratios.items())))
    for what, r in ratios.items():
        assert r <= 1.0, (what, r)
