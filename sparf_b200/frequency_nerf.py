"""Host-side mirror of source/models/frequency_nerf.py (`NeRF`, `FrequencyEmbedder`).

Same module tree and state_dict keys as the reference (`mlp_feat.{i}.{weight,bias}`,
`mlp_rgb.{i}.{weight,bias}`, `progress`), same constructor and method signatures, so optimisers,
checkpoints and the trainers' `progress.data.fill_` keep working; the arithmetic of
`forward_samples` / `composite` runs in the CUDA kernels behind include/sparf_b200.h.
"""
from __future__ import annotations

from typing import Any, Dict

import torch
import torch.nn as nn

from . import ops


class FrequencyEmbedder:
    """Kept for API compatibility (renderer.Graph builds two of them and hands them to
    `forward_samples`, frequency_nerf.py:42-69).  The encoding itself is fused into the MLP kernels:
    f_j = 2^j*pi, per coordinate L sines then L cosines."""

    def __init__(self, opt: Dict[str, Any]):
        self.opt = opt
        pe = opt.arch.posenc
        if not (pe.log_sampling and pe.include_pi_in_posenc):
            raise NotImplementedError("sparf_b200 kernels implement the log-sampled, pi-scaled encoding "
                                      "(arch.posenc.log_sampling=True, include_pi_in_posenc=True) only")

    def __call__(self, opt, input, L):
        """[..., C] -> [..., 2*C*L] (frequency_nerf.py:47-69).  The render path never calls this (the MLP kernels
        fuse the encoding); it is the stand-alone tensor op for other callers."""
        return ops.posenc(input, L)


def _layer_dims(layers):
    return list(zip(layers[:-1], layers[1:]))


class NeRF(nn.Module):
    """8x256 trunk (skip at layer 4, last layer = density + 256 features) and 283->128->3 colour head.
    Construction mirrors frequency_nerf.py:72-147 (Xavier-uniform with ReLU gain, zero biases)."""

    def __init__(self, opt: Dict[str, Any], is_fine_network: bool = False):
        super().__init__()
        self.opt = opt
        self.define_network(opt, is_fine_network=is_fine_network)
        # a Parameter so that the coarse-to-fine state is checkpointed (frequency_nerf.py:79-85)
        self.progress = nn.Parameter(torch.tensor(1.0 if opt.barf_c2f is None else 0.0))

    # -------------------------------------------------------------------------------- construction
    def define_network(self, opt, is_fine_network: bool = False):
        pe = opt.arch.posenc
        if not (pe.add_raw_3D_points and pe.add_raw_rays and opt.nerf.view_dep and pe.L_3D > 0 and pe.L_view > 0):
            raise NotImplementedError("sparf_b200 kernels cover the reference's default input layout: raw xyz + "
                                      "encoding, view-dependent colour with raw direction + encoding")
        if opt.arch.density_activ != "softplus":
            raise NotImplementedError("density_activ=%r: only softplus is implemented" % opt.arch.density_activ)
        in_xyz = 3 + 6 * pe.L_3D
        in_view = 3 + 6 * pe.L_view
        feat_layers = opt.arch.layers_feat_fine if (is_fine_network and opt.arch.layers_feat_fine is not None) \
            else opt.arch.layers_feat
        dims = _layer_dims(feat_layers)
        widths = {k_out for _, k_out in dims}
        if len(widths) != 1 or len(opt.arch.skip) > 1:
            raise NotImplementedError("uniform trunk width and at most one skip layer are supported")
        self.mlp_feat = nn.ModuleList()
        for li, (k_in, k_out) in enumerate(dims):
            if li == 0:
                k_in = in_xyz
            if li in opt.arch.skip:
                k_in += in_xyz
            if li == len(dims) - 1:
                k_out += 1
            lin = nn.Linear(k_in, k_out)
            if opt.arch.tf_init:
                self.tensorflow_init_weights(opt, lin, out="first" if li == len(dims) - 1 else None)
            self.mlp_feat.append(lin)
        self.mlp_rgb = nn.ModuleList()
        rgb_dims = _layer_dims(opt.arch.layers_rgb)
        if len(rgb_dims) != 2 or rgb_dims[-1][1] != 3:
            raise NotImplementedError("colour head must be [feat+view -> hidden -> 3]")
        for li, (k_in, k_out) in enumerate(rgb_dims):
            if li == 0:
                k_in = feat_layers[-1] + in_view
            lin = nn.Linear(k_in, k_out)
            if opt.arch.tf_init:
                self.tensorflow_init_weights(opt, lin, out="all" if li == len(rgb_dims) - 1 else None)
            self.mlp_rgb.append(lin)
        self.spec = ops.MLPSpec(n_trunk=len(dims), width=feat_layers[-1], head_width=rgb_dims[0][1],
                                skip_layer=(opt.arch.skip[0] if len(opt.arch.skip) else -1),
                                L_xyz=pe.L_3D, L_view=pe.L_view, barf_c2f=opt.barf_c2f)

    def initialize(self):
        for m in self.modules():
            if isinstance(m, nn.Linear):
                self.tensorflow_init_weights(self.opt, m)

    def choose_activation(self, opt):
        return nn.ReLU(True)

    def tensorflow_init_weights(self, opt, linear: nn.Linear, out: str = None):
        gain = nn.init.calculate_gain("relu")
        if out == "all":
            nn.init.xavier_uniform_(linear.weight)
        elif out == "first":  # density row without the ReLU gain, features with it
            nn.init.xavier_uniform_(linear.weight[:1])
            nn.init.xavier_uniform_(linear.weight[1:], gain=gain)
        else:
            nn.init.xavier_uniform_(linear.weight, gain=gain)
        nn.init.zeros_(linear.bias)

    # -------------------------------------------------------------------------------- kernels
    def kernel_params(self):
        """Parameter tensors in the order the C ABI expects."""
        ps = []
        for lin in self.mlp_feat:
            ps += [lin.weight, lin.bias]
        for lin in self.mlp_rgb:
            ps += [lin.weight, lin.bias]
        return ps

    def _spec(self):
        # barf_c2f can be switched off/on by the trainers between stages (opt is shared, mutable)
        self.spec.barf_c2f = tuple(self.opt.barf_c2f) if self.opt.barf_c2f is not None else None
        return self.spec

    def forward_samples(self, opt, center: torch.Tensor, ray: torch.Tensor, depth_samples: torch.Tensor,
                        embedder_pts=None, embedder_view=None, mode: str = None) -> Dict[str, Any]:
        """center, ray [B,N,3]; depth_samples [B,N,S,1] -> dict(rgb_samples [B,N,S,3], density_samples [B,N,S]).
        Mirrors frequency_nerf.py:260-281 (+ :172-227)."""
        B, N, S = depth_samples.shape[:3]
        t = depth_samples.reshape(B * N, S)
        noise = None
        if opt.nerf.density_noise_reg and mode == "train":
            # same draw as the reference (randn_like of the [B,N,S] raw density, frequency_nerf.py:191-192)
            noise = (torch.randn_like(depth_samples[..., 0]).to(t.device) * opt.nerf.density_noise_reg).reshape(B * N, S)
        sigma, rgb = ops.mlp_forward(self._spec(), center.reshape(B * N, 3), ray.reshape(B * N, 3), t,
                                     self.kernel_params(), noise=noise, progress=self.progress)
        return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))

    def forward(self, opt, points_3D_samples: torch.Tensor, ray: torch.Tensor, embedder_pts=None,
                embedder_view=None, mode: str = None) -> Dict[str, Any]:
        """Arbitrary 3-D points [B,N,S,3] with per-ray directions [B,N,3] (frequency_nerf.py:172-227):
        evaluated as one-sample rays (x = p + 0*d)."""
        B, N, S = points_3D_samples.shape[:3]
        pts = points_3D_samples.reshape(-1, 3)
        dirs = ray[:, :, None, :].expand(B, N, S, 3).reshape(-1, 3)
        t = torch.zeros(pts.shape[0], 1, device=pts.device)
        noise = None
        if opt.nerf.density_noise_reg and mode == "train":
            noise = (torch.randn_like(points_3D_samples[..., 0]).to(pts.device) * opt.nerf.density_noise_reg).reshape(-1, 1)
        sigma, rgb = ops.mlp_forward(self._spec(), pts, dirs, t, self.kernel_params(), noise=noise,
                                     progress=self.progress)
        return dict(rgb_samples=rgb.view(B, N, S, 3), density_samples=sigma.view(B, N, S))

    def positional_encoding(self, opt, input, embedder_fn, L):
        """Encoding with the BARF coarse-to-fine mask (frequency_nerf.py:229-258) as a stand-alone tensor op; `embedder_fn`
        is accepted for signature compatibility (the kernel implements the log-sampled, pi-scaled embedder)."""
        return ops.posenc(input, L, barf_c2f=opt.barf_c2f, progress=self.progress)

    def compute_raw_density(self, opt, points_3D_samples: torch.Tensor, embedder_pts=None):
        """The trunk alone at points [..., 3] (frequency_nerf.py:149-170) -> (raw_density [...] before the softplus, no noise;
        feat [..., width] after the ReLU).  Differentiable w.r.t. the points (normals = -grad of the density) and the
        trunk's parameters.  `embedder_pts` is accepted for signature compatibility (the kernel implements the
        log-sampled, pi-scaled embedder).  For density grids without the features: ops.density_forward(..., features=False)."""
        shape = points_3D_samples.shape[:-1]
        raw, feat = ops.density_forward(self._spec(), points_3D_samples, self.kernel_params()[:2 * len(self.mlp_feat)],
                                        progress=self.progress)
        return raw.view(shape), feat.view(*shape, feat.shape[-1])

    def composite(self, opt, ray: torch.Tensor, pred_dict: Dict[str, Any], depth_samples: torch.Tensor) -> Dict[str, Any]:
        """Volume-rendering quadrature (frequency_nerf.py:283-343) on the kernel; adds rgb, rgb_var, depth,
        depth_var, opacity [B,N,k], weights [B,N,S,1], all_cumulated [B,N] to pred_dict."""
        B, N, S = depth_samples.shape[:3]
        white = bool(opt.nerf.setbg_opaque or opt.mask_img)
        rgb, depth, opacity, weights, depth_var, rgb_var, all_cum = ops.composite(
            pred_dict["density_samples"].reshape(B * N, S), pred_dict["rgb_samples"].reshape(B * N, S, 3),
            depth_samples.reshape(B * N, S), ray.reshape(B * N, 3), white)
        pred_dict.update(rgb=rgb.view(B, N, 3), rgb_var=rgb_var.view(B, N, 1), depth=depth.view(B, N, 1),
                         depth_var=depth_var.view(B, N, 1), opacity=opacity.view(B, N, 1),
                         weights=weights.view(B, N, S, 1), all_cumulated=all_cum.view(B, N))
        return pred_dict
