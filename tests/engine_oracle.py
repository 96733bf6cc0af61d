"""fp64 restatement of the MLP and of the density queries that starts from the engines' own fp32 encoding: the checker
of tests/test_engine_precision.py.  TEST INFRASTRUCTURE ONLY.

oracle.sparf_oracle.mlp_forward in fp64 answers "how far is the engine from exact arithmetic on exact inputs"; on these
nets most of that distance is the fp32 rounding of x = o + t d and of x 2^j pi, amplified by the top band (one ulp of x
is ~1e-3 rad there), so its bounds have to be loose.  Here the inputs are rounded exactly as the encoders round them
(csrc/mlp.cu, encode_xyz_kernel / encode_dir_kernel):

    x32   = o + d * t                  two fp32 ops      == add_rn(o, mul_rn(d, t))
    arg32 = x32 * (2^j * float32(pi))  one fp32 product  == mul_rn(x, band_freq(j))
    u32   = d / |d|                    fp32 ops          (the kernel's sqrtf of a contracted sum may differ by one ulp)

and everything after the rounding -- sin / cos, the c2f weights, the layers, softplus, sigmoid -- runs in fp64, in the
oracle's layer order.  The rounding is straight-through (value of the fp32 result, derivative of the fp64 formula), so
autograd gives the gradients w.r.t. origins, directions, points and every parameter at the point the kernels evaluate.
What remains between an engine and this reference is the engine's arithmetic after the encoding.

Every ReLU pre-activation is returned, so that a test can leave out the samples whose ReLU branch rounding can flip
(margin_mask): the mask depends on the reference alone.

Parameters are in the engines' order (ops.MLPSpec.fill): [trunk_w0, trunk_b0, ..., head_w0, head_b0, head_w1, head_b1].
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import sparf_oracle as O

Tensor = torch.Tensor

PI32 = float(torch.tensor(math.pi, dtype=torch.float32))     # float32(pi) as a python double, exactly


def band_freqs(L: int, device=None) -> Tensor:
    """f_j = 2^j * float32(pi) for j < L, fp32 (exact: scaling by a power of two)"""
    return (2.0 ** torch.arange(L, dtype=torch.float32, device=device)) * PI32


def _straight_through(exact: Tensor, rounded: Tensor) -> Tensor:
    """the value of `rounded` with the derivative of `exact`"""
    return exact + (rounded.to(exact.dtype) - exact).detach()


def _encode(x: Tensor, x32: Optional[Tensor], L: int, w: Optional[Tensor]):
    """[..., 3] -> ([..., 3 + 6L] in the engines' layout: x, then per coordinate L sines and L cosines, times the c2f
    weight w [L] (fp32 values); the band arguments [..., 3, L]).  x32 given: x carries its value, and the arguments are
    rounded to fp32 products of x32."""
    f = band_freqs(L, x.device)
    arg = x[..., None] * f.to(x.dtype)
    if x32 is not None:
        arg = _straight_through(arg, x32[..., None] * f)
    s, c = arg.sin(), arg.cos()
    if w is not None:
        s, c = s * w.to(x.dtype), c * w.to(x.dtype)
    return torch.cat([x, torch.stack([s, c], dim=-2).reshape(*x.shape[:-1], 6 * L)], dim=-1), arg


def _c2f(spec, L: int, progress, device) -> Optional[Tensor]:
    if spec.barf_c2f is None:
        return None
    return O.c2f_weights(L, float(progress), spec.barf_c2f, device, torch.float32)


def _trunk(spec, params: Sequence[Tensor], enc: Tensor, pre: List[Tensor]):
    """trunk layers 0 .. n_trunk-1 -> (raw [...], relu(features) [..., width]); appends every ReLU pre-activation"""
    h = enc
    raw = None
    for li in range(spec.n_trunk):
        if li == spec.skip_layer:
            h = torch.cat([h, enc], dim=-1)
        z = F.linear(h, params[2 * li], params[2 * li + 1])
        if li == spec.n_trunk - 1:
            raw, z = z[..., 0], z[..., 1:]
        pre.append(z)
        h = F.relu(z)
    return raw, h


def mlp_reference(spec, params: Sequence[Tensor], origins: Tensor, dirs: Tensor, t: Tensor, *,
                  noise: Optional[Tensor] = None, progress=None, rounded: bool = True) -> Dict[str, object]:
    """origins, dirs [R, 3], t [R, S], noise [R, S], params: fp64 tensors holding fp32 values (leaves, if gradients are
    wanted) -> dict(sigma [R, S], rgb [R, S, 3], raw [R, S] (before the noise), pre: the ReLU pre-activations
    [R, S, n] of the trunk layers and of the head's hidden layer, x [R, S, 3], arg [R, S, 3, L_xyz], u [R, 3],
    arg_view [R, 3, L_view]).  rounded=False: the fp64 graph of oracle.sparf_oracle.mlp_forward (no fp32 rounding
    anywhere)."""
    dt = torch.float64
    o, d, tt = origins.to(dt), dirs.to(dt), t.to(dt)
    x = o[:, None, :] + d[:, None, :] * tt[..., None]
    x32 = None
    if rounded:
        x32 = origins.float()[:, None, :] + dirs.float()[:, None, :] * t.float()[..., None]
        x = _straight_through(x, x32)
    pre: List[Tensor] = []
    enc, arg = _encode(x, x32, spec.L_xyz, _c2f(spec, spec.L_xyz, progress, x.device))
    raw, h = _trunk(spec, params, enc, pre)
    sigma = F.softplus(raw + noise.to(dt) if noise is not None else raw)
    u = F.normalize(d, dim=-1)
    u32 = None
    if rounded:
        d32 = dirs.float()
        n32 = (d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1] + d32[:, 2] * d32[:, 2]).sqrt().clamp_min(1e-12)
        u32 = d32 / n32[:, None]
        u = _straight_through(u, u32)
    denc, arg_view = _encode(u, u32, spec.L_view, _c2f(spec, spec.L_view, progress, u.device))
    S = t.shape[1]
    hh = torch.cat([h, denc[:, None, :].expand(-1, S, -1)], dim=-1)
    o2 = 2 * spec.n_trunk
    z = F.linear(hh, params[o2], params[o2 + 1])
    pre.append(z)
    rgb = torch.sigmoid(F.linear(F.relu(z), params[o2 + 2], params[o2 + 3]))
    return dict(sigma=sigma, rgb=rgb, raw=raw, pre=pre, x=x, arg=arg, u=u, arg_view=arg_view)


def density_reference(spec, params: Sequence[Tensor], points: Tensor, *, progress=None,
                      rounded: bool = True) -> Dict[str, object]:
    """points [M, 3] (fp32 values), the trunk's 2 n_trunk fp64 parameters -> dict(raw [M], feat [M, width],
    pre: the trunk's ReLU pre-activations, arg [M, 3, L_xyz]).  The points are the engines' x as they are; rounded:
    the band arguments are fp32 products."""
    x = points.to(torch.float64)
    x32 = points.float() if rounded else None
    pre: List[Tensor] = []
    enc, arg = _encode(x, x32, spec.L_xyz, _c2f(spec, spec.L_xyz, progress, x.device))
    raw, feat = _trunk(spec, params, enc, pre)
    return dict(raw=raw, feat=feat, pre=pre, arg=arg)


def margin_mask(pre: Sequence[Tensor], mu: float) -> Tensor:
    """Samples (all leading dimensions of the pre-activations) with any ReLU pre-activation closer to 0 than mu times
    the root mean square of its layer: there, rounding may take the other ReLU branch.  -> bool [leading dims]."""
    flag = None
    for z in pre:
        z = z.detach()
        rms = z.pow(2).mean().sqrt()
        f = (z.abs() < mu * rms).any(dim=-1)
        flag = f if flag is None else flag | f
    return flag


# ----------------------------------------------------------------------------------------------
# networks
# ----------------------------------------------------------------------------------------------
def make_params(spec, seed: int) -> List[Tensor]:
    """fp32 CPU parameters of the network `spec` in the engines' order: tests/golden/common.det_weights (uniform with
    the ReLU gain, non-zero biases, peaky: a density row x3 with bias -3 and a colour layer x2, so that density and
    colour vary along a ray)."""
    import common
    opt = common.make_opt(width=spec.width, depth_layers=spec.n_trunk, L_3D=spec.L_xyz, L_view=spec.L_view)
    opt.arch.skip = [spec.skip_layer] if spec.skip_layer >= 0 else []
    opt.arch.layers_rgb = [None, spec.head_width, 3]
    sd = common.det_weights(opt, seed, peaky=True, sigma_bias=-3.0)
    return [sd[k] for k in param_keys(spec)]


def param_keys(spec) -> List[str]:
    """oracle.sparf_oracle's state-dict keys in the engines' order"""
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(spec.n_trunk)], [])
    return keys + ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]


def ray_inputs(R: int, S: int, seed: int):
    """fp32 CPU origins [R, 3] (~0.5 randn), directions [R, 3] (length 1 ... 1.2), sorted depths t [R, S] in
    [1.2, 5.2] (the default metric range) and density noise [R, S] (0.5 randn)"""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g) * 0.5
    d = torch.randn(R, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True) * (1 + 0.2 * torch.rand(R, 1, generator=g))
    t = torch.sort(torch.rand(R, S, generator=g) * 4 + 1.2, dim=1).values
    noise = torch.randn(R, S, generator=g) * 0.5
    return o, d, t, noise
