"""Coloured meshes by TSDF fusion: depth and colour maps rendered from a set of cameras are integrated into a truncated
signed distance volume on BARF's lattice (csrc/tsdf.cu), and marching cubes extracts its zero level from the observed
points only (ops.marching_cubes_masked).  Unlike mesh.extract_mesh this needs no density threshold, and it keeps only
the surfaces the cameras see.

    from sparf_b200 import mesh, tsdf
    vol = tsdf.TSDFVolume(res=256)
    tsdf.fuse_renders(opt, graph, vol, pose_w2c, intr, H, W, depth_range)
    m = tsdf.extract_mesh(vol)
    mesh.write_ply("scene.ply", m["vertices"], m["faces"], colors=m["colors"])

The rules (projection, update, masking) are specified in include/sparf_b200.h.
"""
from __future__ import annotations

import torch

from . import _lib, mesh, ops
from .utils.edict import edict

# default truncation in voxels ((r1 - r0) / res): wide enough that the lattice points next to a surface are observed on
# both sides of it by the views that see it, narrow enough that the far side of a thin object stays separate
TRUNC_VOXELS = 4.0
# pixels rendered and integrated per batch of views in fuse_renders (each batch's maps: 17 B per pixel)
BATCH_PIXELS = 1 << 21


class TSDFVolume:
    """The state of a TSDF volume on the lattice mesh.lattice_axis(res, range) (n = res + 1 points per axis, axis 0 =
    x): tsdf [n, n, n] (initially 1), weight [n, n, n] (initially 0) and color [n, n, n, 3] (initially 0), fp32 on
    `device`.  res and range default as in mesh.trimesh_settings (TRIMESH_DEFAULTS); trunc (world units) defaults to
    TRUNC_VOXELS voxels."""

    def __init__(self, res=None, range=None, trunc=None, device="cuda"):
        self.res, self.range, _ = mesh.trimesh_settings({}, res, range)
        if self.res < 1:
            raise ValueError("TSDFVolume: res %d (>= 1)" % self.res)
        self.trunc = float(trunc) if trunc is not None else TRUNC_VOXELS * (self.range[1] - self.range[0]) / self.res
        if not self.trunc > 0 or self.trunc == float("inf"):
            raise ValueError("TSDFVolume: trunc %r (finite, > 0)" % (trunc,))
        n = self.res + 1
        self.device = torch.device(device)
        self.axis = mesh.lattice_axis(self.res, self.range).to(self.device)
        self.tsdf = torch.empty(n, n, n, device=self.device, dtype=torch.float32)
        self.weight = torch.empty_like(self.tsdf)
        self.color = torch.empty(n, n, n, 3, device=self.device, dtype=torch.float32)
        self.reset_()

    @property
    def n(self) -> int:
        return self.res + 1

    def reset_(self) -> "TSDFVolume":
        """restore the initial state (tsdf 1, weight 0, color 0), in place"""
        self.tsdf.fill_(1.0)
        self.weight.zero_()
        self.color.zero_()
        return self


def _check_tensor(name, t, shape, dtypes, device):
    if not torch.is_tensor(t):
        raise ValueError("integrate_: %s must be a tensor, got %s" % (name, type(t).__name__))
    if t.dim() != len(shape) or any(s is not None and a != s for a, s in zip(t.shape, shape)):
        want = "[%s]" % ", ".join("*" if s is None else str(s) for s in shape)
        raise ValueError("integrate_: %s must be %s, got %s" % (name, want, list(t.shape)))
    if t.dtype not in dtypes:
        raise ValueError("integrate_: %s must be %s, got %s" % (name, " or ".join(map(str, dtypes)), t.dtype))
    if t.device != device:
        raise ValueError("integrate_: %s is on %s, the volume on %s" % (name, t.device, device))


def integrate_(vol: TSDFVolume, depth, pose_w2c, intr, rgb=None, valid=None) -> TSDFVolume:
    """Integrate B views into vol in place (sparf_tsdf_integrate): depth [B, H, W] camera z-depth, pose_w2c [B, 3, 4],
    intr [B, 3, 3] or [3, 3] (shared), rgb [B, H, W, 3] or None, valid [B, H, W] bool / uint8 or None (all valid); fp32
    tensors on the volume's device.  The views are taken in order; integrating them in several calls gives the same
    volume as one call.  ValueError for a bad shape, dtype or device."""
    f32 = (torch.float32,)
    dev = vol.tsdf.device
    if not torch.is_tensor(depth) or depth.dim() != 3:
        raise ValueError("integrate_: depth must be a tensor [B, H, W], got %s"
                         % ((list(depth.shape),) if torch.is_tensor(depth) else type(depth).__name__))
    B, H, W = depth.shape
    if B < 1 or H < 1 or W < 1:
        raise ValueError("integrate_: depth [B, H, W] must not be empty, got %s" % list(depth.shape))
    _check_tensor("depth", depth, (B, H, W), f32, dev)
    _check_tensor("pose_w2c", pose_w2c, (B, 3, 4), f32, dev)
    if torch.is_tensor(intr) and intr.dim() == 2:
        _check_tensor("intr", intr, (3, 3), f32, dev)
        intr = intr.expand(B, 3, 3)
    _check_tensor("intr", intr, (B, 3, 3), f32, dev)
    if rgb is not None:
        _check_tensor("rgb", rgb, (B, H, W, 3), f32, dev)
    if valid is not None:
        _check_tensor("valid", valid, (B, H, W), (torch.bool, torch.uint8), dev)
    if dev.type != "cuda":
        raise ValueError("integrate_: the volume must be on a CUDA device, it is on %s" % dev)
    return _integrate(vol, depth.contiguous(), pose_w2c.contiguous(), intr.contiguous(),
                      None if rgb is None else rgb.contiguous(), None if valid is None else valid.contiguous())


@ops._on_tensor_device
def _integrate(vol, depth, pose, intr, rgb, valid):
    B, H, W = depth.shape
    vp = None if valid is None else (valid if valid.dtype == torch.uint8 else valid.view(torch.uint8))
    _lib.check(_lib.lib().sparf_tsdf_integrate(
        ops._ptr(vol.axis), vol.n, vol.trunc, B, H, W, ops._ptr(pose), ops._ptr(intr), ops._ptr(depth), ops._ptr(rgb),
        ops._ptr(vp), ops._ptr(vol.tsdf), ops._ptr(vol.weight), ops._ptr(vol.color), ops._stream()), "tsdf_integrate")
    return vol


def render_maps(pred, fine=True, min_opacity=0.5):
    """(depth, rgb, valid) of one val render [B, H*W, ...]: the fine pass's outputs where it exists and fine is set,
    depth / opacity (the expected termination depth given a hit), rgb as rendered, valid = opacity >= min_opacity"""
    sfx = "_fine" if fine and pred.get("depth_fine") is not None else ""
    opacity = pred["opacity" + sfx][..., 0]
    return pred["depth" + sfx][..., 0] / opacity, pred["rgb" + sfx], opacity >= min_opacity


@torch.no_grad()
def render_batches(opt, graph, pose_w2c, intr, H: int, W: int, depth_range, min_opacity=0.5, fine=True, device=None):
    """Render the views pose_w2c [B, 3, 4] (intr [B, 3, 3] or [3, 3]) of H x W pixels with
    graph.render_image_at_specific_pose_and_rays(..., mode="val"), in batches of about BATCH_PIXELS pixels, and yield
    each batch's integrate_ arguments (depth [b, H, W], pose_w2c, intr, rgb [b, H, W, 3], valid [b, H, W]) from
    render_maps.  depth_range [2] = (near, far) of a metric-depth scene (an inverse-depth opt reads
    opt.nerf.depth.range).  Whatever occupancy grid or early termination the graph has attached is used."""
    dev = torch.device(device) if device is not None else pose_w2c.device
    pose_w2c = pose_w2c.to(dev, torch.float32)
    B = pose_w2c.shape[0]
    intr = intr.to(dev, torch.float32)
    intr = intr.expand(B, 3, 3) if intr.dim() == 2 else intr
    data = edict(depth_range=torch.as_tensor(depth_range, dtype=torch.float32).reshape(1, 2).to(dev))
    per = max(1, BATCH_PIXELS // (H * W))
    for b0 in range(0, B, per):
        pose, K = pose_w2c[b0:b0 + per].contiguous(), intr[b0:b0 + per].contiguous()
        pred = graph.render_image_at_specific_pose_and_rays(opt, data, pose, K, H, W, iter=None, mode="val")
        depth, rgb, valid = render_maps(pred, fine, min_opacity)
        nb = pose.shape[0]
        yield (depth.reshape(nb, H, W).contiguous(), pose, K, rgb.reshape(nb, H, W, 3).contiguous(),
               valid.reshape(nb, H, W).contiguous())


def fuse_renders(opt, graph, vol: TSDFVolume, pose_w2c, intr, H: int, W: int, depth_range, min_opacity=0.5,
                 fine=True) -> TSDFVolume:
    """Render the views (render_batches: val mode, no gradients) and integrate them into vol, batch by batch: depth /
    opacity of the fine pass (of the coarse one without a fine pass or with fine=False), its rgb, valid where opacity >=
    min_opacity.  The renders' outputs are integrated as they are, with whatever occupancy grid or early termination
    the graph has attached."""
    for depth, pose, K, rgb, valid in render_batches(opt, graph, pose_w2c, intr, H, W, depth_range, min_opacity, fine,
                                                     device=vol.tsdf.device):
        integrate_(vol, depth, pose, K, rgb=rgb, valid=valid)
    return vol


@torch.no_grad()
def vertex_colors(vol: TSDFVolume, verts: torch.Tensor) -> torch.Tensor:
    """colors [V, 3] of index-space vertices on lattice edges: the colour at the edge's lower end p plus the vertex's
    fraction s along the edge times the difference to the upper end, c(p) + s (c(p + e_a) - c(p)), in fp32, clamped to
    [0, 1].  s = the vertex's coordinate along a minus p_a, exact in fp32; a vertex at a lattice point takes its
    colour."""
    if verts.shape[0] == 0:
        return torch.zeros(0, 3, device=verts.device, dtype=torch.float32)
    base = verts.floor()
    frac = verts - base
    s, a = frac.max(dim=1)
    p = base.long()
    q = p.clone()
    q[torch.arange(p.shape[0], device=p.device), a] += (s > 0).long()
    n = vol.n
    c = vol.color.view(-1, 3)
    c0 = c[(p[:, 0] * n + p[:, 1]) * n + p[:, 2]]
    c1 = c[(q[:, 0] * n + q[:, 1]) * n + q[:, 2]]
    return (c0 + s[:, None] * (c1 - c0)).clamp_(0.0, 1.0)


@torch.no_grad()
def extract_mesh(vol: TSDFVolume) -> dict:
    """The zero level of the volume: ops.marching_cubes_masked of -tsdf, NaN where weight == 0, at iso 0, so the inside
    is tsdf <= 0 and the faces point outward, and no surface appears where observed space meets unobserved space.
    -> dict(vertices [V, 3] fp32 world (mesh.to_world), faces [F, 3] int64, colors [V, 3] fp32 in [0, 1]
    (vertex_colors)) on the volume's device."""
    field = torch.where(vol.weight > 0, -vol.tsdf, torch.full_like(vol.tsdf, float("nan")))
    verts, faces = ops.marching_cubes_masked(field, 0.0)
    del field
    return dict(vertices=mesh.to_world(verts, vol.res, vol.range), faces=faces, colors=vertex_colors(vol, verts))
