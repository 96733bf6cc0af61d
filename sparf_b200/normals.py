"""Normal maps of full-image renders (Graph.set_normals): per ray, the composite of the density normals at the samples
that contribute to the pixel,

    normal = sum over the samples k with w_k != 0, in increasing k, of w_k * n(x_k),   n = -g / |g| (0 where g = 0),

g = ops.density_gradient at x_k, the normal mesh.density_normals gives a vertex.  x_k = o + d * t_k is formed as the MLP
encoder forms it (an fp32 multiply, then an fp32 add, no FMA), so each normal is taken at the point whose density the
render composited.  The map is world-space and unnormalised: |normal| <= opacity, and a ray that hits nothing has a
short normal.  Samples an occupancy grid or early termination skipped have sigma = 0, hence w = 0, and are never
differentiated, so normals need no code of their own for either.
"""
from __future__ import annotations

import torch

from . import _lib, ops
from .mesh import _trunk, unit_normals


@torch.no_grad()
def sample_points(center: torch.Tensor, ray: torch.Tensor, t: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """x = o + d * t at the flat sample indices idx of a [R, S] batch: center, ray [R, 3], t [R, S] -> [len(idx), 3]"""
    S = t.shape[1]
    r = idx // S
    return center[r] + ray[r] * t.reshape(-1)[idx, None]


@ops._on_tensor_device
@torch.no_grad()
def composite_normals(nerf, center: torch.Tensor, ray: torch.Tensor, t: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """normal [B, N, 3] of one pass: center, ray [B, N, 3], t and weights [B, N, S, 1] (the pass's samples and composite
    weights), nerf the pass's network.  The count of samples with w != 0 is read back to the host."""
    B, N, S = t.shape[:3]
    R = B * N
    w = weights.reshape(R * S)
    idx = torch.nonzero(w != 0).reshape(-1)            # increasing: each ray's kept samples are consecutive
    K = idx.numel()
    if K == 0:
        return torch.zeros(B, N, 3, device=w.device, dtype=torch.float32)
    x = sample_points(center.reshape(R, 3).float(), ray.reshape(R, 3).float(), t.reshape(R, S).float(), idx)
    g = ops.density_gradient(nerf._spec(), x, _trunk(nerf), progress=nerf.progress.detach())
    src = (w[idx, None] * unit_normals(g)).contiguous()
    out = torch.empty(R, 3, device=w.device, dtype=torch.float32)
    k_dev = torch.tensor([K], device=w.device, dtype=torch.int64)
    _lib.check(_lib.lib().sparf_compact_ray_sum(R, S, K, ops._ptr(k_dev), ops._ptr(idx), 3, ops._ptr(src), ops._ptr(out),
                                                ops._stream()), "compact_ray_sum")
    return out.view(B, N, 3)
