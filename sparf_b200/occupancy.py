"""Empty-space skipping for inference renders: an occupancy grid over a box, built from the density lattice of
`opt.trimesh` (mesh.density_grid), and a forward pass that runs the MLP only on the samples the grid keeps.

    from sparf_b200 import occupancy
    graph.set_occupancy(occupancy.build_grid(opt, graph.nerf), occupancy.build_grid(opt, graph.nerf_fine))
    with torch.no_grad():
        ret = graph.render_by_slices(opt, pose, H, W, intr, depth_range, iter, mode="val")

A sample is skipped when it lies inside the box in a cell none of whose lattice points within one cell has σ >= thres;
its σ and rgb are then 0, and every other sample is evaluated exactly as the dense render evaluates it (semantics in
include/sparf_b200.h).  A grid is a snapshot of the network when it was built: rebuild it after the weights change.
Samples outside the box are always evaluated.  For scenes whose samples mostly lie outside any box (inverse-depth LLFF,
rooms seen from the inside) build a contracted grid instead, which covers all of space:

    grid = occupancy.build_grid(opt, graph.nerf, contraction=(center, radius))

Its lookup maps a point x to y = (x - center) / radius and, where m = ||y||_inf > 1, on to y / m * (2 - 1 / m)
(mip-NeRF 360's contraction in the inf-norm), into the cube [-2, 2]^3; the grid's cells split that cube.  The cells are
uniform in the linear region ||y||_inf <= 1.  Beyond it they grow like m^2: they are uniform in 1 / m, which is how
inverse-depth sampling spaces its samples.

Choosing center and radius: put the cameras and the near bound inside the linear region.  The LLFF loader scales a
forward-facing scene so that its nearest bound is about 1.33, and the samples start at t = 1 from cameras near the
origin.  center = the mean camera centre and radius = 1.33 (or the cameras' spread, if that is larger) then put the
first quarter of every ray, where inverse depth crowds its samples, in the linear region, and space the cells beyond it
like the samples.  Indoors (Replica), center the grid on the room and pick radius so that the walls lie inside or just
past the linear region.  Lattice points at infinity (on the cube's faces) are never evaluated and count as occupied, so
the outer two-cell shell, beyond ||x - center||_inf = radius * res / 8, is always kept.  Conservativeness is weaker in
the stretched outer cells than in the linear region: there one cell spans a long stretch of world space between its
lattice points.

In training, a grid can be kept current on the device inside the captured step instead of being rebuilt between steps
(Instant-NGP's update).  Build it with a per-cell density, then call update_ after the optimiser step:

    grids = [occupancy.build_grid(opt, m, ema=True) for m in graph.get_network_components()]
    graph.set_training_occupancy(*grids)
    def step():
        ...; loss.backward(); adam.step()
        for g, m in zip(grids, graph.get_network_components()):
            occupancy.update_(g, m, 4096, 4096)

update_ re-samples a fixed budget of cells, half uniformly from all cells and half from the occupied ones, at a random
point in each, and sets each cell's density to max(decay * density, the σ sampled there), then re-thresholds the bits.
Its cost is set by the budget, not by res^3, nothing in it synchronises, and every size is fixed, so the next replay's
renders see the new bits without any host-side bookkeeping.  The draws come from torch.rand on the grid's device: ranks
of a distributed job whose CUDA generators are seeded alike keep identical grids; nothing else keeps them in step.  A
contracted grid's outer two-cell shell is never sampled and stays occupied.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import mesh, ops

_POPCOUNT = [bin(i).count("1") for i in range(256)]
FLT_MAX = float(np.finfo(np.float32).max)
CONTRACTED_RANGE = (-2.0, 2.0)      # the cube the contraction maps space into


class OccupancyGrid:
    """bits [ceil(res^3 / 32)] (int32 storage of uint32 words; cell (i,j,k) is bit idx & 31 of word idx >> 5, idx =
    (i*res + j)*res + k) over the box [r0, r1]^3 split into res^3 cells, built at density threshold thres.
    contraction: None (a box grid over world space), or (center (3 floats), radius) for a contracted grid, whose cells
    split the contracted cube: range is then CONTRACTED_RANGE.  center and radius are kept as fp32 values.
    density: None, or fp32 [res^3] per-cell densities (indexed like the bits) that update_ decays and raises."""

    def __init__(self, bits: torch.Tensor, res: int, range, thres: float, contraction=None, density=None):
        assert bits.dtype == torch.int32 and bits.numel() == (res ** 3 + 31) // 32
        assert density is None or (density.dtype == torch.float32 and density.numel() == res ** 3)
        self.bits, self.res, self.thres = bits.contiguous(), int(res), float(thres)
        self.density = None if density is None else density.contiguous().view(-1)
        self.range = (float(range[0]), float(range[1]))
        self.contraction = None
        if contraction is not None:
            assert self.range == CONTRACTED_RANGE, "a contracted grid covers the cube [-2, 2]^3"
            self.contraction = _as_contraction(contraction)

    def occupied_fraction(self) -> float:
        """occupied cells / res^3"""
        table = torch.tensor(_POPCOUNT, dtype=torch.int64, device=self.bits.device)
        return table[self.bits.view(torch.uint8).long()].sum().item() / self.res ** 3


def _as_contraction(contraction):
    """((cx, cy, cz), radius) as python floats holding fp32 values; finite, radius > 0"""
    center, radius = contraction
    c = tuple(float(np.float32(v)) for v in (center.tolist() if torch.is_tensor(center) else center))
    r = float(np.float32(radius))
    assert len(c) == 3 and all(math.isfinite(v) for v in c + (r,)) and r > 0, contraction
    return c, r


def contracted_warp(center, radius):
    """The lattice map of a contracted grid's build (mesh.lattice_density's warp).  A lattice point v of the contracted
    cube (fp32 [P, 3]) with n = ||v||_inf < 2 goes to the world point center + radius * y, where y = v for n <= 1 and
    y = v / (n (2 - n)) beyond, the inverse of the lookup's map.  This is computed in fp64 and rounded once to fp32.
    Points with n >= 2 lie at infinity: they are not evaluated, and their σ is NaN."""
    center, radius = _as_contraction((center, radius))

    def warp(v):
        v = v.double()
        n = v.abs().amax(-1, keepdim=True)
        far = n[:, 0] >= 2
        den = torch.where((n <= 1) | far[:, None], torch.ones_like(n), n * (2 - n))
        c = torch.tensor(center, dtype=torch.float64, device=v.device)
        x = torch.where(far[:, None], c, c + radius * (v / den))
        return x.float(), far

    return warp


@torch.no_grad()
def build_grid(opt, nerf, res=None, range=None, thres=0.01, engine=None, contraction=None, ema=False) -> OccupancyGrid:
    """The occupancy grid of one network (graph.nerf or graph.nerf_fine) at its current weights and nerf.progress: σ on
    the lattice of opt.trimesh (res and range default to it, as in mesh.density_grid), then ops.occupancy_build at
    thres.  contraction = (center, radius) builds a contracted grid over all of space instead (module docstring): σ at
    the world points (contracted_warp) of the lattice linspace(-2, 2, res + 1)^3, evaluated slab by slab as
    mesh.density_grid does, NaN at infinity, then the same ops.occupancy_build.  range must then be None.
    ema=True also gives the grid a density that update_ can keep current: each cell's max of σ at its 8 corners, NaN and
    +inf as FLT_MAX.  The bits are the same either way.  engine: None = the current ops engine."""
    if contraction is None:
        res, rng, _ = mesh.trimesh_settings(opt, res, range)
    else:
        assert range is None, "a contracted grid covers the cube [-2, 2]^3 of the contracted space"
        res, rng = mesh.trimesh_settings(opt, res)[0], CONTRACTED_RANGE
        contraction = _as_contraction(contraction)
    sigma = _lattice_sigma(opt, nerf, res, rng, contraction, engine)
    return OccupancyGrid(ops.occupancy_build(sigma, thres), res, rng, thres, contraction,
                         _corner_max(sigma) if ema else None)


def _lattice_sigma(opt, nerf, res, rng, contraction, engine):
    """σ on the lattice a grid is built from: mesh.density_grid over the box rng, or the contracted lattice"""
    if contraction is None:
        return mesh.density_grid(opt, nerf, res=res, range=rng, engine=engine)
    return mesh.lattice_density(nerf, mesh.lattice_axis(res, CONTRACTED_RANGE), engine=engine,
                                warp=contracted_warp(*contraction))


def _corner_max(sigma):
    """lattice σ [res+1]^3 -> the per-cell density [res^3]: the max over each cell's 8 corners, NaN and +inf as
    FLT_MAX (exact, so it does not depend on the order)"""
    s = torch.nan_to_num(sigma, nan=FLT_MAX, posinf=FLT_MAX)
    n = s.shape[0] - 1
    d = s[:n, :n, :n].clone()
    for a, b, c in ((0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)):
        torch.maximum(d, s[a:a + n, b:b + n, c:c + n], out=d)
    return d.reshape(-1)


@torch.no_grad()
def refresh_(grid: OccupancyGrid, opt, nerf, engine=None) -> OccupancyGrid:
    """Rebuild `grid` in place from the network's current weights and nerf.progress: the lattice and threshold of
    build_grid, written into the grid's existing `bits` tensor (and `density`, where the grid has one), so that a CUDA
    graph captured with the grid sees the new cells on its next replay.  A grid is a snapshot of the network when it was
    built or last refreshed: in training (Graph.set_training_occupancy) the samples it skips get no gradient until the
    next refresh, so refresh it every few steps, between steps (outside any captured graph), or keep it current inside
    the step with update_."""
    sigma = _lattice_sigma(opt, nerf, grid.res, grid.range, grid.contraction, engine)
    grid.bits.copy_(ops.occupancy_build(sigma, grid.thres))
    if grid.density is not None:
        grid.density.copy_(_corner_max(sigma))
    return grid


@torch.no_grad()
def update_(grid: OccupancyGrid, nerf, n_uniform: int, n_occupied: int, decay: float = 0.95, draws=None,
            engine=None) -> OccupancyGrid:
    """Keep a grid built with ema=True current, in place on grid.density and grid.bits (module docstring): re-sample
    n_uniform interior cells drawn uniformly and n_occupied drawn from the occupied interior cells
    (ops.occupancy_sample), query σ = softplus(raw) at a random point in each (ops.density_forward, no noise, the BARF
    mask at nerf.progress), then density = max(decay * density, σ sampled in the cell) for every interior cell and
    bits = !(density < grid.thres) (ops.occupancy_ema_).  draws: None draws (u_cell [N], u_jit [N,3]) with torch.rand on
    the grid's device, N = n_uniform + n_occupied; or those two tensors.  Nothing synchronises and every size is fixed:
    call it after the optimiser step of a captured training step, so that the next replay's renders see the new bits.
    Raises before any work on a grid without density, decay outside (0, 1], a negative budget, draws of the wrong shape,
    or a contracted grid with res < 8.  engine: None = the current ops engine."""
    if grid.density is None:
        raise ValueError("update_: the grid has no density; build it with build_grid(..., ema=True)")
    if not 0.0 < float(decay) <= 1.0:
        raise ValueError("update_: decay %r outside (0, 1]" % (decay,))
    if int(n_uniform) < 0 or int(n_occupied) < 0:
        raise ValueError("update_: negative budget (%d, %d)" % (n_uniform, n_occupied))
    if grid.contraction is not None and grid.res < 8:
        raise ValueError("update_: a contracted grid needs res >= 8 (res %d)" % grid.res)
    n = int(n_uniform) + int(n_occupied)
    if draws is None:
        u_cell = torch.rand(n, device=grid.bits.device)
        u_jit = torch.rand(n, 3, device=grid.bits.device)
    else:
        u_cell, u_jit = draws
        if tuple(u_cell.shape) != (n,) or tuple(u_jit.shape) != (n, 3):
            raise ValueError("update_: draws of shapes %s, %s; expected (%d,), (%d, 3)"
                             % (tuple(u_cell.shape), tuple(u_jit.shape), n, n))
    if n == 0:
        cells = torch.empty(0, dtype=torch.int64, device=grid.bits.device)
        sigma = torch.empty(0, device=grid.bits.device)
    else:
        cells, points = ops.occupancy_sample(grid.bits, grid.res, grid.range, grid.contraction, n_uniform, n_occupied,
                                             u_cell, u_jit)
        raw, _ = ops.density_forward(nerf._spec(), points, mesh._trunk(nerf), progress=nerf.progress.detach(),
                                     engine=mesh._engine(engine), features=False)
        sigma = F.softplus(raw)
    ops.occupancy_ema_(grid.density, grid.bits, grid.res, grid.contraction is not None, cells, sigma, decay, grid.thres)
    return grid


def train_forward_samples(nerf, grid: OccupancyGrid, opt, center, ray, depth_samples, mode) -> dict:
    """NeRF.forward_samples with gradients over the samples the grid keeps (ops.mlp_forward_grid): the skipped samples
    get σ = 0, rgb = 0 and no gradient; the kept ones the values of the dense pass, with its density noise (the same
    randn_like draw, taken at the kept samples).  Nothing in it synchronises, so a training step that calls it can be
    captured into one CUDA graph.  center, ray [B,N,3]; depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3],
    density_samples [B,N,S])."""
    B, N, S = depth_samples.shape[:3]
    t = depth_samples.reshape(B * N, S)
    noise = None
    if opt.nerf.density_noise_reg and mode == "train":
        noise = (torch.randn_like(depth_samples[..., 0]).to(t.device) * opt.nerf.density_noise_reg).reshape(B * N, S)
    sigma, rgb = ops.mlp_forward_grid(nerf._spec(), center.reshape(B * N, 3), ray.reshape(B * N, 3), t, grid,
                                      nerf.kernel_params(), noise=noise, progress=nerf.progress)
    return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))


@torch.no_grad()
def forward_samples(nerf, grid: OccupancyGrid, center, ray, depth_samples) -> dict:
    """NeRF.forward_samples (no noise) with the samples the grid skips set to σ = 0, rgb = 0: center, ray [B,N,3];
    depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3], density_samples [B,N,S]).  The kept samples (by the box or
    the contracted lookup, after the grid's kind) go through ops.mlp_forward as one-sample rays (o, d, t), which
    evaluates each of them exactly as the dense call does."""
    B, N, S = depth_samples.shape[:3]
    M = B * N * S
    o, d, t = center.reshape(B * N, 3), ray.reshape(B * N, 3), depth_samples.reshape(B * N, S)
    if grid.contraction is None:
        idx, o_k, d_k, t_k = ops.occupancy_compact(grid.bits, grid.res, grid.range, o, d, t)
    else:
        idx, o_k, d_k, t_k = ops.contracted_compact(o, d, t, 0, S, None, grid.bits, grid.res, *grid.contraction)
    sigma = torch.zeros(M, device=depth_samples.device)
    rgb = torch.zeros(M, 3, device=depth_samples.device)
    if idx.numel():
        sigma_k, rgb_k = ops.mlp_forward(nerf._spec(), o_k, d_k, t_k, nerf.kernel_params(), progress=nerf.progress)
        sigma.index_copy_(0, idx, sigma_k.view(-1))
        rgb.index_copy_(0, idx, rgb_k.view(-1, 3))
    return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))
