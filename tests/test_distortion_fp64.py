"""The distortion regulariser (ops.distortion_loss, csrc/optim.cu) against the literal O(S^2) form of the oracle
(oracle.sparf_oracle.distortion_loss) evaluated in fp64, at the sample layouts training produces.

Yardstick (as in test_cuda_parity.py::test_standalone_posenc_matches_oracle): on the same fp32 inputs, the kernel's
distance from the fp64 oracle must be within C = 4 times the distance of the same oracle evaluated in fp32, plus a
floor.  Distances are relative: |loss - exact| / |exact| for the loss, and for d_w and d_t (fp64 autograd) the largest
over rays of max_i |x - exact| / max_i |exact| within a ray, so a ray with small weights is held to its own scale.

Floors, from the kernel's order of summation (u = 2^-24, the fp32 unit round-off):
  loss   (4 + 2 sqrt(R)) u.  The ratio already measures the rounding of each ray's own sum of positive terms; the
         mean over rays is R atomic additions in arrival order, each rounding a partial sum (<= the total) by at most
         u/2.  Independent rounding errors of standard deviation u / (2 sqrt 3) sum to at most sqrt(R / 12) u, and
         2 sqrt(R) u is ~7 of those standard deviations.  The 4 u covers the per-ray sums at R = 1.
  grads  (8 + 2 ceil((S - 1) / 32)) u.  A ray's prefix and suffix sums are warp trees of depth 5 chained over
         ceil((S - 1) / 32) chunks; summation of that depth errs by at most depth * u of the sum of |terms|, and
         d_w combines two such sums (u_i A_i - M_i and M_gt - u_i A_gt), d_t two others (A_i - A_gt).  After centring,
         sum |terms| is of the scale of the ray's largest gradient.

Ties: where three consecutive t are equal, two mid-points tie, and at a tie the kernel's A_i - A_gt and torch's abs
backward pick different subgradients (both valid).  d_t is gated only on rays without tied mid-points, exact or as the
fp32 form rounds them; d_w and the loss are continuous there and are gated on every ray.  (At t + 1000 with S = 4096
every ray has a tie: 4096 samples share 65 536 fp32 values in [1000.5, 1004.5].  d_t at t + 1000 is gated at S <= 64.)

Layouts: t uniform in [0.5, 4.5] with w = rand^3, and the same t + 100 and + 1000; 128 coarse samples in [0.5, 4.5]
plus S - 128 fine samples ~ N(3, spread) with Gaussian weights peaked at 3, at spread 0.05 and 0.005, increasing
(metric) and decreasing (inverse-depth) t; rays of zero weights, one-hot weights and runs of equal t; S in {2, 31,
32, 33, 64, 4096} (32 mid-points at S = 33: one warp chunk and one lane of the next) at R = 1 and, up to S = 64,
R = 4097 (a partial 4-ray block and 4097 atomic additions into the loss).  S = 4096 runs at R = 1 and 3, not 4097: the
oracle's pair matrix would hold 7e10 entries.

Measured on an H100 80GB HBM3 (700 W power limit): worst ratio kernel distance / bound per group of cases over two
runs (the loss's atomic sum makes it vary from run to run), for the kernel before it centred the mid-points on the
ray's weighted mean and after (each test prints its ratios with -s):

    layout                          before: loss   d_w    d_t      after: loss   d_w    d_t
    uniform                                 0.12   0.40   0.16            0.06   0.16   0.16
    uniform + 100                           0.47   2.43   0.18            0.20   0.03   0.18
    uniform + 1000                          3.42   3.25   0.20            0.04   0.005  0.20
    peaked, spread 0.05                     0.58   0.37   0.22            0.20   0.19   0.22
    peaked, spread 0.005                    1.33   0.34   0.20            0.08   0.13   0.20
    degenerate rays                         0.05   0.47   0.15            0.08   0.15   0.15
    R = 1 and S = 4096                      0.28   0.33   0.15            0.08   0.26   0.15
    R = 3, S = 4096, + 1000                 3.62   3.95   -               0.11   0.006  -
    R = 4097                                0.35   0.59   0.36            0.39   0.25   0.36
    R = 4097, + 1000                        0.27   2.93   0.36            0.33   0.13   0.36

Before, 10 of the 35 checks failed: every + 100 and + 1000 case but R = 4097 at S = 2 (one interval, no pair term), and
one peaked case (spread 0.005, S = 384, inverse).  The peaked layouts' loss error was 1.4e-6 ... 2.3e-6 at spread 0.005,
10 ... 55x the centred kernel's, yet mostly within the (4 + 2 sqrt(64)) u = 1.2e-6 floor plus 4x the fp32 form's
error; at + 1000 d_w erred by 2.2e-4 ... 3.1e-4 and now by < 5e-7.  Centring adds 0.4 ... 0.7 us to the call at
R = 4096 (tools/time_distortion.py, medians of three alternated runs, with d_t: 12.5 -> 13.2 us at S = 128 and
16.9 -> 17.3 us at S = 256).
"""
import math

import pytest
import torch

from oracle import sparf_oracle as O

pytestmark = pytest.mark.gpu

C = 4.0
ULP = 2.0 ** -24


def _loss_floor(R):
    return (4 + 2 * math.sqrt(R)) * ULP


def _grad_floor(S):
    return (8 + 2 * math.ceil((S - 1) / 32)) * ULP


def _ray_dist(x, exact, rows=None):
    """Largest over rays of max_i |x - exact| / max_i |exact| ([R, S] tensors; rays with exact == 0 use scale 1)."""
    x, exact = x.double(), exact.double()
    if rows is not None:
        x, exact = x[rows], exact[rows]
    if exact.numel() == 0:
        return 0.0
    scale = exact.abs().amax(dim=1)
    scale = torch.where(scale > 0, scale, torch.ones_like(scale))
    return ((x - exact).abs().amax(dim=1) / scale).max().item()


def _oracle(t, w, dtype):
    """Loss, d_w and d_t of the literal form at `dtype` on the fp32 inputs t, w [R, S]."""
    tt = t.to(dtype)[..., None].requires_grad_(True)
    ww = w.to(dtype)[..., None].requires_grad_(True)
    loss = O.distortion_loss(tt, ww)
    loss.backward()
    return loss.item(), ww.grad[..., 0], tt.grad[..., 0]


def _untied_rays(t):
    """Rays whose mid-points are pairwise distinct, both exactly (fp64 from the fp32 t) and as the fp32 oracle rounds
    them: mid-points a few ulps apart can round to one value, and the fp32 form then takes the tie's subgradient."""
    ok = torch.ones(t.shape[0], dtype=torch.bool, device=t.device)
    for x in (t.double(), t):
        u = (x[:, 1:] + x[:, :-1]) / 2
        ok &= (u[:, 1:] != u[:, :-1]).all(dim=1)
    return ok


def _check(name, t, w):
    """Gate loss, d_w and d_t of the kernel on t, w [R, S] (fp32, on the device)."""
    from sparf_b200 import ops
    R, S = t.shape
    tk, wk = t[..., None].clone().requires_grad_(True), w[..., None].clone().requires_grad_(True)
    loss = ops.distortion_loss(tk, wk)
    loss.backward()
    l64, dw64, dt64 = _oracle(t, w, torch.float64)
    l32, dw32, dt32 = _oracle(t, w, torch.float32)
    untied = _untied_rays(t)
    dists = [
        (abs(loss.item() - l64) / abs(l64), abs(l32 - l64) / abs(l64), _loss_floor(R)),
        (_ray_dist(wk.grad[..., 0], dw64), _ray_dist(dw32, dw64), _grad_floor(S)),
        (_ray_dist(tk.grad[..., 0], dt64, untied), _ray_dist(dt32, dt64, untied), _grad_floor(S)),
    ]
    ratios = [ek / (C * eo + floor) for ek, eo, floor in dists]
    print("%-28s R=%-5d S=%-5d ratio loss %.3f  d_w %.3f  d_t %.3f  (kernel %.1e %.1e %.1e, fp32 %.1e %.1e %.1e)" % (
        (name, R, S) + tuple(ratios) + tuple(d[0] for d in dists) + tuple(d[1] for d in dists)))
    for what, (ek, eo, floor) in zip(("loss", "d_w", "d_t"), dists):
        assert ek <= C * eo + floor, "%s %s: kernel %.2e vs fp32 oracle %.2e (bound %.2e)" % (
            name, what, ek, eo, C * eo + floor)


def _uniform(R, S, seed, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    t = torch.sort(torch.rand(R, S, generator=g, dtype=torch.float64) * 4 + 0.5, dim=1).values + shift
    w = torch.rand(R, S, generator=g) ** 3
    return t.float().cuda(), w.cuda()


def _peaked(R, S, spread, decreasing, seed):
    """128 coarse samples in [0.5, 4.5] plus S - 128 fine samples ~ N(3, spread), Gaussian weights peaked at t = 3."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(R, 128, generator=g, dtype=torch.float64) * 4 + 0.5
    fine = 3 + spread * torch.randn(R, S - 128, generator=g, dtype=torch.float64)
    t = torch.sort(torch.cat([coarse, fine], dim=1), dim=1, descending=decreasing).values
    w = torch.exp(-0.5 * ((t - 3) / spread) ** 2) * (0.5 + 0.5 * torch.rand(R, S, generator=g, dtype=torch.float64))
    return t.float().cuda(), w.float().cuda()


@pytest.mark.parametrize("shift", [0.0, 100.0, 1000.0])
@pytest.mark.parametrize("S", [128, 257])
def test_distortion_uniform_and_far(S, shift):
    """Uniform t, w = rand^3; + 100 and + 1000 put the weight mass far from t = 0 compared with its spread."""
    t, w = _uniform(64, S, seed=S + int(shift), shift=shift)
    _check("uniform +%g" % shift, t, w)


@pytest.mark.parametrize("decreasing", [False, True], ids=["metric", "inverse"])
@pytest.mark.parametrize("spread", [0.05, 0.005])
@pytest.mark.parametrize("S", [256, 384])
def test_distortion_peaked_at_a_surface(S, spread, decreasing):
    """A trained NeRF's fine pass: samples and weights concentrated at the surface, t = 3."""
    t, w = _peaked(64, S, spread, decreasing, seed=S)
    _check("peaked %g %s" % (spread, "inverse" if decreasing else "metric"), t, w)


@pytest.mark.parametrize("S", [5, 33, 257])
def test_distortion_degenerate_rays(S):
    """Ray 0: all-zero weights (the centre falls back to the first mid-point).  Ray 1: one-hot weight.  Ray 2: runs
    of three equal t (dt = 0, tied mid-points).  Ray 3: zero weights and equal t.  Ray 4: one-hot weight on a run of
    equal t.  Rays 5-8: uniform.  Ray 9: weight only on w_0, which never enters the loss."""
    t, w = _uniform(10, S, seed=7 * S)
    t, w = t.clone(), w.clone()
    w[0] = 0
    w[1] = 0
    w[1, S // 2] = 0.8
    for r in (2, 3, 4):
        for i in range(1, S - 2, 4):
            t[r, i + 1] = t[r, i + 2] = t[r, i]
    w[3] = 0
    w[4] = 0
    w[4, 2] = 0.6
    w[9] = 0
    w[9, 0] = 1
    assert not _untied_rays(t)[2:5].any()
    _check("degenerate", t, w)


@pytest.mark.parametrize("R,S", [(1, 2), (1, 31), (1, 32), (1, 33), (1, 64), (1, 4096), (3, 4096),
                                 (4097, 2), (4097, 31), (4097, 32), (4097, 33), (4097, 64)])
def test_distortion_shapes(R, S):
    """Partial and whole warp chunks, one long ray, and 4097 rays (a partial 4-ray block, 4097 atomic additions)."""
    t, w = _uniform(R, S, seed=R * 10000 + S)
    _check("shape", t, w)
    if R > 1:
        t, w = _uniform(R, S, seed=R * 10000 + S, shift=1000.0)
        _check("shape +1000", t, w)
