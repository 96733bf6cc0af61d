"""Early ray termination for inference renders: a ray stops being evaluated once the optical depth it has accumulated
shows it opaque (transmittance below eps), alone or on top of an occupancy grid (sparf_b200.occupancy).

    graph.set_early_termination(eps=1e-4, window=16)
    with torch.no_grad():
        ret = graph.render_by_slices(opt, pose, H, W, intr, depth_range, iter, mode="val")

A pass's samples are evaluated in windows of `window` samples per ray.  After each window every alive ray adds the
window's optical depth to its running tau, and it dies when tau > -ln(eps): its remaining samples are skipped, with
σ = 0 and rgb = 0, exactly as the grid's skipped samples are.  Every evaluated sample is evaluated exactly as the
dense render evaluates it (semantics in include/sparf_b200.h).  The composite then changes by less than eps in
opacity and rgb (2 eps with an opaque background) and by less than eps * max t in depth; the fine pass's samples
move with the coarse weights, so its error is not bounded.  Each window reads its sample count on the host, so a render
on this path cannot be captured into a CUDA graph.  Scenes whose rays mostly turn opaque gain; soft or small objects
gain little, and so does inverse-depth sampling alone, which crowds the samples in front of the surface.  A contracted
occupancy grid (sparf_b200.occupancy) skips those front samples, and termination on top of it skips the ones behind.

Training steps can terminate too (train_forward_samples, Graph.set_training_termination): the same kept set on the
pass's own σ (density noise included), with gradients, one tape and one backward per pass, and nothing read back on the
host, so that a step stays one CUDA graph.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops


def tau_max(eps: float) -> float:
    """The optical depth above which a ray dies: fp32(-ln eps); eps = 0 gives +inf (nothing dies)."""
    return float(np.float32(-math.log(eps))) if eps > 0 else math.inf


@torch.no_grad()
def forward_samples(nerf, grid, eps: float, window: int, center, ray, depth_samples) -> dict:
    """NeRF.forward_samples (no noise) with the samples of terminated rays, and those the occupancy grid (box or
    contracted; or None) skips, set to σ = 0, rgb = 0: center, ray [B,N,3]; depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3],
    density_samples [B,N,S]).  The evaluated samples go through ops.mlp_forward as one-sample rays (o, d, t)."""
    B, N, S = depth_samples.shape[:3]
    R = B * N
    dev = depth_samples.device
    o, d, t = center.reshape(R, 3), ray.reshape(R, 3), depth_samples.reshape(R, S)
    sigma = torch.zeros(R, S, device=dev)
    rgb = torch.zeros(R * S, 3, device=dev)
    alive = torch.ones(R, dtype=torch.uint8, device=dev)
    tau = torch.zeros(R, device=dev)
    limit = tau_max(eps)
    if grid is not None and grid.contraction is not None:
        compact = lambda k0, k1: ops.contracted_compact(o, d, t, k0, k1, alive, grid.bits, grid.res, *grid.contraction)
    else:
        grid_args = dict(bits=grid.bits, res=grid.res, range=grid.range) if grid is not None else {}
        compact = lambda k0, k1: ops.termination_compact(o, d, t, k0, k1, alive, **grid_args)
    for k0 in range(0, S, window):
        k1 = min(k0 + window, S)
        idx, o_k, d_k, t_k = compact(k0, k1)
        if idx.numel():            # an empty window (every ray dead, or the grid skips it all) may precede a full one
            sigma_k, rgb_k = ops.mlp_forward(nerf._spec(), o_k, d_k, t_k, nerf.kernel_params(), progress=nerf.progress)
            sigma.view(-1).index_copy_(0, idx, sigma_k.view(-1))
            rgb.index_copy_(0, idx, rgb_k.view(-1, 3))
        if k1 < S:
            ops.termination_update(sigma, t, d, k0, k1, limit, tau, alive)
    return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))


def train_forward_samples(nerf, grid, eps: float, window: int, opt, center, ray, depth_samples, mode) -> dict:
    """NeRF.forward_samples with gradients and early ray termination (ops.mlp_forward_terminated), on top of the
    training occupancy grid `grid` (box or contracted; or None): the samples behind an opaque point of the ray, and those
    the grid skips, get σ = 0, rgb = 0 and no gradient; the others the values of the dense pass, with its density noise
    (the same randn_like draw, taken at the kept samples).  A ray dies on this pass's own σ, noise included.  Nothing in
    it synchronises, so a training step that calls it can be captured into one CUDA graph.  center, ray [B,N,3];
    depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3], density_samples [B,N,S])."""
    B, N, S = depth_samples.shape[:3]
    t = depth_samples.reshape(B * N, S)
    noise = None
    if opt.nerf.density_noise_reg and mode == "train":
        noise = (torch.randn_like(depth_samples[..., 0]).to(t.device) * opt.nerf.density_noise_reg).reshape(B * N, S)
    sigma, rgb = ops.mlp_forward_terminated(nerf._spec(), center.reshape(B * N, 3), ray.reshape(B * N, 3), t, grid, eps,
                                            window, nerf.kernel_params(), noise=noise, progress=nerf.progress)
    return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))
