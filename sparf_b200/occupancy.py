"""Empty-space skipping for inference renders: an occupancy grid over a box, built from the density lattice of
`opt.trimesh` (mesh.density_grid), and a forward pass that runs the MLP only on the samples the grid keeps.

    from sparf_b200 import occupancy
    graph.set_occupancy(occupancy.build_grid(opt, graph.nerf), occupancy.build_grid(opt, graph.nerf_fine))
    with torch.no_grad():
        ret = graph.render_by_slices(opt, pose, H, W, intr, depth_range, iter, mode="val")

A sample is skipped when it lies inside the box in a cell none of whose lattice points within one cell has σ >= thres;
its σ and rgb are then 0, and every other sample is evaluated exactly as the dense render evaluates it (semantics in
include/sparf_b200.h).  A grid is a snapshot of the network when it was built: rebuild it after the weights change.
Samples outside the box are always evaluated, so scenes whose samples mostly lie outside it (inverse-depth LLFF) gain
little.
"""
from __future__ import annotations

import torch

from . import mesh, ops

_POPCOUNT = [bin(i).count("1") for i in range(256)]


class OccupancyGrid:
    """bits [ceil(res^3 / 32)] (int32 storage of uint32 words; cell (i,j,k) is bit idx & 31 of word idx >> 5, idx =
    (i*res + j)*res + k) over the box [r0, r1]^3 split into res^3 cells, built at density threshold thres."""

    def __init__(self, bits: torch.Tensor, res: int, range, thres: float):
        assert bits.dtype == torch.int32 and bits.numel() == (res ** 3 + 31) // 32
        self.bits, self.res, self.thres = bits.contiguous(), int(res), float(thres)
        self.range = (float(range[0]), float(range[1]))

    def occupied_fraction(self) -> float:
        """occupied cells / res^3"""
        table = torch.tensor(_POPCOUNT, dtype=torch.int64, device=self.bits.device)
        return table[self.bits.view(torch.uint8).long()].sum().item() / self.res ** 3


@torch.no_grad()
def build_grid(opt, nerf, res=None, range=None, thres=0.01, engine=None) -> OccupancyGrid:
    """The occupancy grid of one network (graph.nerf or graph.nerf_fine) at its current weights and nerf.progress: σ on
    the lattice of opt.trimesh (res and range default to it, as in mesh.density_grid), then ops.occupancy_build at
    thres.  engine: None = the current ops engine."""
    res, rng, _ = mesh.trimesh_settings(opt, res, range)
    sigma = mesh.density_grid(opt, nerf, res=res, range=rng, engine=engine)
    return OccupancyGrid(ops.occupancy_build(sigma, thres), res, rng, thres)


@torch.no_grad()
def forward_samples(nerf, grid: OccupancyGrid, center, ray, depth_samples) -> dict:
    """NeRF.forward_samples (no noise) with the samples the grid skips set to σ = 0, rgb = 0: center, ray [B,N,3];
    depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3], density_samples [B,N,S]).  The kept samples go through
    ops.mlp_forward as one-sample rays (o, d, t), which evaluates each of them exactly as the dense call does."""
    B, N, S = depth_samples.shape[:3]
    M = B * N * S
    idx, o_k, d_k, t_k = ops.occupancy_compact(grid.bits, grid.res, grid.range, center.reshape(B * N, 3),
                                               ray.reshape(B * N, 3), depth_samples.reshape(B * N, S))
    sigma = torch.zeros(M, device=depth_samples.device)
    rgb = torch.zeros(M, 3, device=depth_samples.device)
    if idx.numel():
        sigma_k, rgb_k = ops.mlp_forward(nerf._spec(), o_k, d_k, t_k, nerf.kernel_params(), progress=nerf.progress)
        sigma.index_copy_(0, idx, sigma_k.view(-1))
        rgb.index_copy_(0, idx, rgb_k.view(-1, 3))
    return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))
