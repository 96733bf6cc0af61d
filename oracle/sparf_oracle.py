"""CPU ORACLE for the SPARF ray-marching hot path.  TEST INFRASTRUCTURE ONLY.

This file is a from-scratch restatement, in plain torch tensor algebra (fp32 by default, fp64 on
request), of the algorithm the reference implements in

    source/models/renderer.py        (ray batch orchestration, depth sampling, PDF resampling)
    source/models/frequency_nerf.py  (positional encoding, 8x256 MLP + colour head, compositing)
    source/utils/camera.py           (pixel -> ray, pose inversion)
    source/models/poses_models/two_columns.py (9-D pose embedding -> [R|t])
    source/training/core/base_losses.py       (photometric Huber loss, DS-NeRF sparse-depth loss)

Only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of
`bench.py` may import it; the product (`sparf_b200/`) never does.  Gradients come from torch
autograd over this restatement, exactly as the reference obtains them.

PARITY PINNING: the reference has no tests for this path (SURVEY.md §4), so the oracle is pinned
against outputs of the reference itself: tests/golden/*.npz, produced by tests/golden/make_golden.py
which imports the unmodified reference from /root/reference in the build container.
tests/test_oracle_vs_golden.py checks every stored output and gradient.

All functions are functional (no nn.Module) and take the MLP as a dict with the reference's
state_dict keys (`mlp_feat.{i}.weight` ... `mlp_rgb.{i}.bias`, `progress`).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# ----------------------------------------------------------------------------------------------
# camera / rays                                                     (source/utils/camera.py)
# ----------------------------------------------------------------------------------------------
def invert_pose(pose: Tensor) -> Tensor:
    """[...,3,4] rigid inverse: R' = R^T, t' = -R^T t.   camera.py:92-98 (Pose.invert)."""
    R, t = pose[..., :3], pose[..., 3:]
    Rt = R.transpose(-1, -2)
    return torch.cat([Rt, -(Rt @ t)], dim=-1)


def rays_from_pixels(pose_w2c: Tensor, intr: Tensor, uv: Tensor) -> Tuple[Tensor, Tensor]:
    """uv [B,N,2] image coordinates -> (center, ray) [B,N,3] in world space, ray un-normalised.

    camera.py:318-334 (img2cam / cam2world), :372-379 and :407-416: p = K^-1 [u,v,1];
    both p and the zero point are pushed through the FULL c2w pose and subtracted, i.e.
    ray = (Rc p + tc) - tc with Rc = R^T, tc = -R^T t."""
    B = pose_w2c.shape[0]
    ones = torch.ones_like(uv[..., :1])
    hom = torch.cat([uv, ones], dim=-1)                                  # [B,N,3]
    cam = hom @ torch.linalg.inv(intr).transpose(-1, -2)                 # K^-1 applied to rows
    c2w = invert_pose(pose_w2c)                                          # [B,3,4]
    cam_h = torch.cat([cam, ones], dim=-1)                               # [B,N,4]
    zero_h = torch.cat([torch.zeros_like(cam), ones], dim=-1)
    world = cam_h @ c2w.transpose(-1, -2)
    center = zero_h @ c2w.transpose(-1, -2)
    return center, world - center


def pixel_grid(H: int, W: int, device=None, dtype=torch.float32) -> Tensor:
    """Row-major pixel centres (x+0.5, y+0.5), index = y*W + x.   camera.py:363-368."""
    ys = torch.arange(H, device=device, dtype=dtype) + 0.5
    xs = torch.arange(W, device=device, dtype=dtype) + 0.5
    Y, X = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([X, Y], dim=-1).reshape(-1, 2)


def rays_from_ray_idx(pose_w2c: Tensor, intr: Tensor, H: int, W: int, ray_idx: Optional[Tensor]):
    """renderer.py:273-291: the reference builds the rays of the FULL H*W grid and then indexes them
    with shared (n,) indices or per-image (B,n) indices; the oracle does the same so that even the
    BLAS blocking of the tiny 3x3 products is identical."""
    B = pose_w2c.shape[0]
    grid = pixel_grid(H, W, device=pose_w2c.device, dtype=pose_w2c.dtype)  # [HW,2]
    center, ray = rays_from_pixels(pose_w2c, intr, grid[None].repeat(B, 1, 1))
    if ray_idx is None:
        return center, ray
    if ray_idx.dim() == 2 and ray_idx.shape[0] == B:
        gi = ray_idx.long()[..., None].expand(-1, -1, 3)
        return center.gather(1, gi), ray.gather(1, gi)
    return center[:, ray_idx.long()], ray[:, ray_idx.long()]


def rays_at_pixels(pose_w2c: Tensor, intr: Tensor, pixels: Tensor):
    """Float pixel locations used as given (NO +0.5).   camera.py:384-416."""
    B = pose_w2c.shape[0]
    uv = pixels[None].expand(B, -1, -1) if pixels.dim() == 2 else pixels
    return rays_from_pixels(pose_w2c, intr, uv)


# ----------------------------------------------------------------------------------------------
# pose parametrisation                           (source/models/poses_models/two_columns.py)
# ----------------------------------------------------------------------------------------------
def pose_to_d9(pose: Tensor) -> Tensor:
    """[N,3,4] -> [N,9] = (t, first two ROWS of R).   two_columns.py:23-39."""
    return torch.cat([pose[:, :3, 3], pose[:, :2, :3].reshape(pose.shape[0], 6)], dim=-1)


def d9_to_pose(d9: Tensor) -> Tensor:
    """Gram-Schmidt on the two rows, third = cross.   two_columns.py:42-62, :166-193."""
    t, a1, a2 = d9[:, :3], d9[:, 3:6], d9[:, 6:9]
    b1 = F.normalize(a1, dim=-1)
    b2 = F.normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    R = torch.stack([b1, b2, b3], dim=-2)
    return torch.cat([R, t[..., None]], dim=-1)


def _taylor(theta: Tensor, first: int, nth: int = 10) -> Tensor:
    """sum_i (-1)^i theta^(2i) / d_i, d_i = running product of consecutive integer pairs starting at `first`
    (camera.py:180-205: A = sin x / x uses pairs (2i)(2i+1) for i > 0; B = (1 - cos x)/x^2 pairs (2i+1)(2i+2);
    C = (x - sin x)/x^3 pairs (2i+2)(2i+3))."""
    ans = torch.zeros_like(theta)
    denom = 1.0
    for i in range(nth + 1):
        if first == 0:
            if i > 0:
                denom *= (2 * i) * (2 * i + 1)
        else:
            denom *= (2 * i + first) * (2 * i + first + 1)
        ans = ans + (-1) ** i * theta ** (2 * i) / denom
    return ans


def se3_to_SE3(wu: Tensor) -> Tensor:
    """[...,6] (rotation vector w, translation generator u) -> [...,3,4] = [exp(w^) | V(w) u].   camera.py:142-157."""
    w, u = wu[..., :3], wu[..., 3:]
    O = torch.zeros_like(w[..., 0])
    wx = torch.stack([torch.stack([O, -w[..., 2], w[..., 1]], dim=-1),
                      torch.stack([w[..., 2], O, -w[..., 0]], dim=-1),
                      torch.stack([-w[..., 1], w[..., 0], O], dim=-1)], dim=-2)
    theta = w.norm(dim=-1)[..., None, None]
    I = torch.eye(3, device=w.device, dtype=wu.dtype)
    A, B, C = _taylor(theta, 0), _taylor(theta, 1), _taylor(theta, 2)
    R = I + A * wx + B * wx @ wx
    V = I + B * wx + C * wx @ wx
    return torch.cat([R, V @ u[..., None]], dim=-1)


def compose_pair(pose_a: Tensor, pose_b: Tensor) -> Tensor:
    """pose_b o pose_a on [...,3,4].   camera.py:108-115."""
    Ra, ta, Rb, tb = pose_a[..., :3], pose_a[..., 3:], pose_b[..., :3], pose_b[..., 3:]
    return torch.cat([Rb @ Ra, Rb @ ta + tb], dim=-1)


# ----------------------------------------------------------------------------------------------
# depth sampling                                             (source/models/renderer.py)
# ----------------------------------------------------------------------------------------------
def sample_depth(B: int, R: int, S: int, depth_range, *, param: str = "metric",
                 rand: Optional[Tensor] = None, device=None, dtype=torch.float32) -> Tensor:
    """t_k = ((u_k + k)/S)(far-near)+near, u = rand or 0.5; inverse: 1/(t+1e-8).  renderer.py:401-419.
    depth_range is a (2,) tensor for metric depth (data_dict.depth_range[0], so far-near is an fp32
    subtraction) or the python list opt.nerf.depth.range for inverse depth.  Returns [B,R,S]."""
    near, far = depth_range[0], depth_range[1]
    if torch.is_tensor(near):
        near, far = near.to(dtype), far.to(dtype)
    u = rand.reshape(B, R, S).to(dtype) if rand is not None else torch.full((B, R, S), 0.5, device=device, dtype=dtype)
    k = torch.arange(S, device=u.device, dtype=dtype)
    t = (u + k) / S * (far - near) + near
    if param == "inverse":
        t = 1 / (t + 1e-8)
    return t


def sample_depth_to_max(depth_max: Tensor, S: int, near: float) -> Tensor:
    """Per-ray far bound, no jitter: t_k = ((1+k)/S)(far_r - near)+near.   renderer.py:616-621."""
    if torch.is_tensor(near):
        near = near.to(depth_max.dtype)
    k = torch.arange(S, device=depth_max.device, dtype=depth_max.dtype)
    return (1 + k) / S * (depth_max[..., None] - near) + near


def sample_pdf(weights: Tensor, S: int, S_fine: int, depth_range: Sequence[float],
               grid: Optional[Tensor] = None, u: Optional[Tensor] = None) -> Tensor:
    """Inverse-transform sampling of the coarse weights.   renderer.py:421-456.
    weights [B,R,S]; grid = the ONE shared (S_fine+1,) grid (linspace when deterministic, or the
    recorded torch.rand(S_fine+1) draw); u = the (S_fine,) sample positions themselves, in place of the
    grid's mid-points.  Returns [B,R,S_fine]."""
    near, far = depth_range[0], depth_range[1]   # torch.linspace takes the 0-dim tensors as they are
    dt = weights.dtype
    pdf = weights / (weights.sum(-1, keepdim=True) + 1e-6)
    cdf = torch.cat([torch.zeros_like(pdf[..., :1]), pdf.cumsum(-1)], dim=-1)      # [B,R,S+1]
    if u is None:
        if grid is None:
            grid = torch.linspace(0, 1, S_fine + 1, device=weights.device, dtype=dt)
        grid = grid.to(dt)
        u = 0.5 * (grid[:-1] + grid[1:])
    u = u.to(dt).expand(*cdf.shape[:-1], S_fine).contiguous()
    idx = torch.searchsorted(cdf, u, right=True)
    lo = (idx - 1).clamp(min=0)
    hi = idx.clamp(max=S)
    bins = torch.linspace(near, far, S + 1, device=weights.device, dtype=dt).expand(*cdf.shape[:-1], S + 1)
    c_lo, c_hi = cdf.gather(-1, lo), cdf.gather(-1, hi)
    b_lo, b_hi = bins.gather(-1, lo), bins.gather(-1, hi)
    frac = (u - c_lo) / (c_hi - c_lo + 1e-8)
    return b_lo + frac * (b_hi - b_lo)


# ----------------------------------------------------------------------------------------------
# positional encoding + MLP                               (source/models/frequency_nerf.py)
# ----------------------------------------------------------------------------------------------
def c2f_weights(L: int, progress: float, barf_c2f, device=None, dtype=torch.float32) -> Optional[Tensor]:
    """BARF mask w_j = (1 - cos(pi * clamp(alpha - j, 0, 1))) / 2.   frequency_nerf.py:248-253."""
    if barf_c2f is None:
        return None
    start, end = barf_c2f
    # the reference evaluates alpha in fp32 from the fp32 `progress` parameter
    alpha = (torch.tensor(progress, dtype=torch.float32) - start) / (end - start) * L
    k = torch.arange(L, dtype=torch.float32)
    w = (1 - ((alpha - k).clamp(min=0, max=1) * math.pi).cos()) / 2
    return w.to(device=device, dtype=dtype)


def posenc(x: Tensor, L: int, mask: Optional[Tensor]) -> Tensor:
    """[...,C] -> [...,2CL]: per coordinate, L sines then L cosines, f_j = 2^j*pi (fp32 product of the
    fp32 power of two and float(pi)); optional c2f mask per frequency.   frequency_nerf.py:47-69, :256."""
    freq = (2.0 ** torch.arange(L, dtype=torch.float32, device=x.device) * math.pi).to(x.dtype)
    spec = x[..., None] * freq                                           # [...,3,L]
    s, c = spec.sin(), spec.cos()
    if mask is not None:
        s, c = s * mask, c * mask
    return torch.stack([s, c], dim=-2).reshape(*x.shape[:-1], 2 * x.shape[-1] * L)


def mlp_forward(params: Dict[str, Tensor], pts: Tensor, ray: Tensor, *, L_3D: int = 10, L_view: int = 4,
                skip: Sequence[int] = (4,), barf_c2f=None, noise: Optional[Tensor] = None
                ) -> Tuple[Tensor, Tensor]:
    """pts [B,R,S,3], ray [B,R,3] (un-normalised) -> (density [B,R,S], rgb [B,R,S,3]).

    frequency_nerf.py:149-227: trunk with the encoded input re-concatenated AFTER the features at
    the skip layer; last trunk layer emits (raw_sigma | 256 features); softplus density (+ optional
    additive noise on the raw value); head on [relu(features) | unit-direction encoding]; sigmoid."""
    dt = pts.dtype
    prog = float(params["progress"])
    m3 = c2f_weights(L_3D, prog, barf_c2f, pts.device, dt)
    mv = c2f_weights(L_view, prog, barf_c2f, pts.device, dt)
    enc = torch.cat([pts, posenc(pts, L_3D, m3)], dim=-1)
    n_feat = len([k for k in params if k.startswith("mlp_feat.") and k.endswith(".weight")])
    h = enc
    for li in range(n_feat):
        if li in skip:
            h = torch.cat([h, enc], dim=-1)
        h = F.linear(h, params["mlp_feat.%d.weight" % li].to(dt), params["mlp_feat.%d.bias" % li].to(dt))
        if li == n_feat - 1:
            raw, h = h[..., 0], h[..., 1:]
        h = F.relu(h)
    if noise is not None:
        raw = raw + noise.reshape(raw.shape).to(dt)
    density = F.softplus(raw)
    unit = F.normalize(ray, dim=-1)[..., None, :].expand_as(pts)
    denc = torch.cat([unit, posenc(unit, L_view, mv)], dim=-1)
    h = torch.cat([h, denc], dim=-1)
    n_rgb = len([k for k in params if k.startswith("mlp_rgb.") and k.endswith(".weight")])
    for li in range(n_rgb):
        h = F.linear(h, params["mlp_rgb.%d.weight" % li].to(dt), params["mlp_rgb.%d.bias" % li].to(dt))
        if li != n_rgb - 1:
            h = F.relu(h)
    return density, torch.sigmoid(h)


def composite(ray: Tensor, density: Tensor, rgb_s: Tensor, t: Tensor, *, white_bg: bool = False) -> Dict[str, Tensor]:
    """Quadrature of the volume rendering integral.   frequency_nerf.py:283-343.
    ray [B,R,3], density [B,R,S], rgb_s [B,R,S,3], t [B,R,S]."""
    length = ray.norm(dim=-1, keepdim=True)                               # [B,R,1]
    gaps = torch.cat([t[..., 1:] - t[..., :-1], torch.full_like(t[..., :1], 1e10)], dim=-1) * length
    sd = density * gaps
    alpha = 1 - torch.exp(-sd)
    excl = torch.cat([torch.zeros_like(sd[..., :1]), sd[..., :-1]], dim=-1).cumsum(-1)
    T = torch.exp(-excl)
    w = T * alpha                                                         # [B,R,S]
    depth = (w * t).sum(-1, keepdim=True)
    depth_var = (w * (t - depth) ** 2).sum(-1, keepdim=True)
    rgb = (w[..., None] * rgb_s).sum(-2)
    rgb_var = ((rgb_s - rgb[..., None, :]).sum(-1) * w).sum(-1, keepdim=True)   # (sic) signed, not squared
    opacity = w.sum(-1, keepdim=True)
    if white_bg:
        rgb = rgb + (1 - opacity)
    return dict(rgb=rgb, rgb_var=rgb_var, depth=depth, depth_var=depth_var, opacity=opacity,
                weights=w[..., None], all_cumulated=T[..., -2], rgb_samples=rgb_s, density_samples=density,
                t=t[..., None])


# ----------------------------------------------------------------------------------------------
# render orchestration                                  (source/models/renderer.py:250-345, 504-593)
# ----------------------------------------------------------------------------------------------
def render(opt, params: Dict[str, Tensor], params_fine: Optional[Dict[str, Tensor]], center: Tensor, ray: Tensor,
           depth_range, *, mode: str = "train", rand: Optional[Tensor] = None, noise: Optional[Tensor] = None,
           noise_fine: Optional[Tensor] = None, grid_fine: Optional[Tensor] = None, iteration: Optional[int] = None,
           depth_max: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Coarse pass, optional hierarchical fine pass.  center/ray [B,R,3].

    depth_max given => the render_to_max variant (renderer.py:504-593): per-ray far bound and the
    fine network evaluated on the SAME samples, no resampling."""
    B, R = ray.shape[:2]
    S, Sf = opt.nerf.sample_intvs, opt.nerf.sample_intvs_fine
    kw = dict(L_3D=opt.arch.posenc.L_3D, L_view=opt.arch.posenc.L_view, skip=tuple(opt.arch.skip),
              barf_c2f=opt.barf_c2f)
    bg = bool(opt.nerf.setbg_opaque or opt.mask_img)
    stratified = bool(opt.nerf.sample_stratified) and mode not in ("val", "eval", "test")
    use_noise = bool(opt.nerf.density_noise_reg) and mode == "train"

    if depth_max is not None:
        t = sample_depth_to_max(depth_max, S, depth_range[0])
    else:
        t = sample_depth(B, R, S, depth_range, param=opt.nerf.depth.param,
                         rand=rand if stratified else None, device=ray.device, dtype=ray.dtype)
    pts = center[:, :, None] + ray[:, :, None] * t[..., None]
    dens, rgb_s = mlp_forward(params, pts, ray, noise=noise if use_noise else None, **kw)
    out = dict(origins=center, viewdirs=ray)
    out.update(composite(ray, dens, rgb_s, t, white_bg=bg))

    fine_on = bool(opt.nerf.fine_sampling)
    ratio = getattr(opt.nerf, "ratio_start_fine_sampling_at_x", None) if hasattr(opt.nerf, "ratio_start_fine_sampling_at_x") else None
    if fine_on and ratio is not None and iteration is not None and iteration < opt.max_iter * ratio:
        fine_on = False
    if fine_on:
        if depth_max is not None:
            t_all = t
        else:
            with torch.no_grad():
                det = mode not in ("train", "test-optim") or not opt.nerf.sample_stratified
                t_f = sample_pdf(out["weights"][..., 0], S, Sf, depth_range, None if det else grid_fine)
            t_all = torch.cat([t, t_f], dim=-1).sort(dim=-1).values
        pts = center[:, :, None] + ray[:, :, None] * t_all[..., None]
        dens, rgb_s = mlp_forward(params_fine, pts, ray, noise=noise_fine if use_noise else None, **kw)
        fine = composite(ray, dens, rgb_s, t_all, white_bg=bg)
        out.update({k + "_fine": v for k, v in fine.items()})
    return out


# ----------------------------------------------------------------------------------------------
# photometric loss                                   (source/training/core/base_losses.py)
# ----------------------------------------------------------------------------------------------
def huber2(pred: Tensor, target: Tensor) -> Tensor:
    """2 * mean Huber(delta=0.5).   base_losses.py:155-156."""
    return F.huber_loss(pred, target, reduction="mean", delta=0.5) * 2.0


def gather_gt(image: Tensor, ray_idx: Tensor) -> Tensor:
    """image [B,3,H,W] -> colours at ray_idx: [B,n,3].   base_losses.py:274-300."""
    B = image.shape[0]
    flat = image.reshape(B, 3, -1).permute(0, 2, 1)
    if ray_idx.dim() == 2 and ray_idx.shape[0] == B:
        return torch.gather(flat, 1, ray_idx.long()[..., None].expand(-1, -1, 3))
    return flat[:, ray_idx.long()]


def photometric_loss(out: Dict[str, Tensor], image: Tensor, ray_idx: Tensor) -> Tensor:
    """base_losses.py:302-307: Huber on coarse rgb, plus the same on rgb_fine when present."""
    gt = gather_gt(image, ray_idx)
    loss = huber2(out["rgb"].reshape(gt.shape), gt)
    if "rgb_fine" in out:
        loss = loss + huber2(out["rgb_fine"].reshape(gt.shape), gt)
    return loss


def colmap_depth_loss(depth_maps: Sequence[Dict[str, Tensor]], colmap_depth_at_ray: Sequence[Tensor],
                      colmap_weight_at_ray: Sequence[Tensor], batch_size: int) -> Tensor:
    """DS-NeRF sparse-depth term (base_losses.py:385-401): per image with triangulated points,
    mean(w (d_colmap - d_rendered)^2) for the coarse (+ fine) depth; 0.1 * sum / batch_size."""
    loss = 0.0
    for out, d, w in zip(depth_maps, colmap_depth_at_ray, colmap_weight_at_ray):
        loss = loss + torch.mean(((d - out["depth"].reshape(-1)) ** 2) * w)
        if "depth_fine" in out:
            loss = loss + torch.mean(((d - out["depth_fine"].reshape(-1)) ** 2) * w)
    return 0.1 * loss / batch_size


# ----------------------------------------------------------------------------------------------
# default-off regularisers                 (source/training/core/regularization_losses.py)
# ----------------------------------------------------------------------------------------------
def distortion_loss(t: Tensor, w: Tensor) -> Tensor:
    """mip-NeRF-360 distortion loss, literal O(S^2) form.   regularization_losses.py:20-48 (normalize=False).
    t, w: [..., S, 1] (the renderer's `t` and `weights`)."""
    w, t = w[..., 0], t[..., 0]
    ut = (t[..., 1:] + t[..., :-1]) / 2
    w = w[..., 1:]
    dut = torch.abs(ut[..., :, None] - ut[..., None, :])
    inter = torch.sum(w * torch.sum(w[..., None, :] * dut, dim=-1), dim=-1)
    intra = torch.sum(w ** 2 * torch.diff(t), dim=-1) / 3
    return (inter + intra).mean()


def depth_patch_loss(depths: Tensor, patch_size: int, charbonnier_padding: float = 0.001) -> Tensor:
    """Charbonnier smoothness over depth patches.   regularization_losses.py:51-66."""
    B = depths.shape[0]
    d = depths.reshape(B, -1, patch_size ** 2)
    resid_sq = (d[..., None] - d[..., None, :]) ** 2
    return torch.sqrt(resid_sq + charbonnier_padding ** 2).mean()


def regularization_losses(out: Dict[str, Tensor], distortion: bool, depth_patch: bool, patch_size: int = 2) -> Dict[str, Tensor]:
    """base_losses.py:162-194: strengths 2e-3 (distortion) and 2e-2 (depth patch), coarse + fine summed."""
    loss = {}
    if distortion:
        v = 2e-3 * distortion_loss(out["t"], out["weights"])
        if "weights_fine" in out:
            v = v + 2e-3 * distortion_loss(out["t_fine"], out["weights_fine"])
        loss["distortion"] = v
    if depth_patch:
        v = 2e-2 * depth_patch_loss(out["depth"], patch_size)
        if "depth_fine" in out:
            v = v + 2e-2 * depth_patch_loss(out["depth_fine"], patch_size)
        loss["depth_patch"] = v
    return loss
