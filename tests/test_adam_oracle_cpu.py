"""tests/adam_oracle.py against torch's own recipe in fp64 on the CPU: check for a non-finite gradient, then
torch.nn.utils.clip_grad_norm_ + torch.optim.Adam(foreach=False) with the warm-up factor applied to the group's lr for
the step, then ExponentialLR.step(), as the trainers do (and as tests/test_optim.py replays on the device)."""
import pytest
import torch

import adam_oracle as A


@pytest.mark.parametrize("max_norm,warmup,betas", [(0.0, 0.0, (0.9, 0.999)), (0.5, 0.0, (0.9, 0.999)),
                                                   (0.05, 6.0, (0.9, 0.999)), (0.05, 6.0, (0.3, 0.9))])
def test_adam_oracle_matches_torch_fp64(max_norm, warmup, betas):
    h = A.Hyper(lr0=1e-2, gamma=0.93, warmup=warmup, beta1=betas[0], beta2=betas[1], eps=1e-8, max_norm=max_norm)
    g = torch.Generator().manual_seed(5)
    shapes = [(7, 5), (5,), (3, 4, 2)]
    params = [torch.nn.Parameter(torch.randn(s, generator=g, dtype=torch.float64)) for s in shapes]
    opt = torch.optim.Adam(params, lr=h.lr0, betas=betas, eps=h.eps, foreach=False)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=h.gamma)
    flat = torch.cat([p.detach().reshape(-1) for p in params])
    m, v = torch.zeros_like(flat), torch.zeros_like(flat)
    steps = (0, 0)
    clipped = 0
    for it in range(1, 13):
        grads = [torch.randn(s, generator=g, dtype=torch.float64) * 10.0 ** (-(it % 4)) for s in shapes]
        if it == 5:
            grads[1][2] = float("nan")
        if it == 9:
            grads[2][0, 1, 1] = float("inf")
        for p, gr in zip(params, grads):
            p.grad = gr.clone()
        flat_g = torch.cat([gr.reshape(-1) for gr in grads])
        # torch
        lr_orig = opt.param_groups[0]["lr"]
        opt.param_groups[0]["lr"] = lr_orig * (min(1.0, it / warmup) if warmup else 1.0)
        finite = all(torch.isfinite(p.grad).all() for p in params)
        if finite:
            if max_norm:
                torch.nn.utils.clip_grad_norm_(params, max_norm)
            opt.step()
        torch_g = torch.cat([p.grad.reshape(-1) for p in params])
        clipped += finite and A.clip_coef(h, flat_g) < 1
        opt.zero_grad()
        opt.param_groups[0]["lr"] = lr_orig
        sched.step()
        # oracle
        flat, g_used, m, v, steps = A.step(h, flat, flat_g, m, v, steps)
        assert steps == (it - (it >= 5) - (it >= 9), it)
        want = torch.cat([p.detach().reshape(-1) for p in params])
        assert (flat - want).abs().max().item() <= 1e-13 * want.abs().max().item(), it
        st = [opt.state[p] for p in params]
        if st[0]:
            assert int(st[0]["step"]) == steps[0]
            want_m = torch.cat([s["exp_avg"].reshape(-1) for s in st])
            want_v = torch.cat([s["exp_avg_sq"].reshape(-1) for s in st])
            assert (m - want_m).abs().max().item() <= 1e-14 * want_m.abs().max().item(), it
            assert (v - want_v).abs().max().item() <= 1e-14 * want_v.abs().max().item(), it
        if finite:      # the clipped gradient, as clip_grad_norm_ leaves it in .grad
            assert (g_used - torch_g).abs().max().item() <= 1e-15 * flat_g.abs().max().item(), it
        else:           # untouched
            assert torch.equal(g_used.nan_to_num(), torch_g.nan_to_num()), it
    assert abs(A.lr_at(h, 12) - sched.get_last_lr()[0] * h.gamma ** -1) <= 1e-15
    assert (clipped > 0) == (max_norm > 0)


def test_adam_oracle_skips_non_finite_gradients():
    h = A.Hyper(lr0=1e-3, max_norm=1.0)
    x = torch.randn(10, dtype=torch.float64)
    for bad in (float("nan"), float("inf"), -float("inf")):
        g = x.clone()
        g[3] = bad
        p, g2, m, v, steps = A.step(h, x, g, x * 0.5, x * x, (4, 7))
        assert steps == (4, 8)
        assert torch.equal(p, x) and torch.equal(m, x * 0.5) and torch.equal(v, x * x)


def test_adam_oracle_schedule():
    h = A.Hyper(lr0=2e-3, gamma=0.9, warmup=4)
    assert [round(A.lr_at(h, k) / 2e-3, 12) for k in (1, 2, 4, 5)] == [0.25, round(0.9 * 0.5, 12), round(0.9 ** 3, 12),
                                                                       round(0.9 ** 4, 12)]
