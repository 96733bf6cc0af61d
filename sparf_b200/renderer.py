"""Host-side mirror of source/models/renderer.py (`Graph`): same constructor, attributes, public
methods, argument meaning and output-dict keys, so the reference's trainers and loss modules can
use it unchanged (INTEGRATION.md).  Every tensor is produced by the kernels behind
include/sparf_b200.h; this file only routes arguments.

Differences from the reference that are deliberate:
  * rays are generated only for the requested pixels (the reference builds the full H*W grid and
    then indexes it, renderer.py:273-291 / camera.py:363-379);
  * the NaN retry loop (renderer.py:274-275) and the unreachable NDC branch (renderer.py:293-295, a
    TypeError in the reference) are not reproduced;
  * `origins` / `viewdirs` / `rgb_samples` / `density_samples` are still returned (cheap).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Union

import numpy as np
import torch

from . import ops
from .frequency_nerf import FrequencyEmbedder, NeRF
from .utils.edict import edict


def _invert_pose(pose: torch.Tensor) -> torch.Tensor:
    R, t = pose[..., :3], pose[..., 3:]
    Rt = R.transpose(-1, -2)
    return torch.cat([Rt, -(Rt @ t)], dim=-1)


class Graph(torch.nn.Module):
    """NeRF model: MLP prediction + volume rendering (renderer.py:28)."""

    def __init__(self, opt: Dict[str, Any], device: torch.device):
        super().__init__()
        self.opt = opt
        self.device = device
        self.define_renderer(opt)

    def define_renderer(self, opt):
        if opt.camera.ndc:
            raise NotImplementedError("camera.ndc=True is unreachable in the reference (TypeError, renderer.py:295)")
        self.nerf = NeRF(opt).to(self.device)
        if opt.nerf.fine_sampling:
            self.nerf_fine = NeRF(opt, is_fine_network=True).to(self.device)
        self.embedder_pts = FrequencyEmbedder(self.opt)
        self.embedder_view = FrequencyEmbedder(self.opt)

    def re_initialize(self):
        self.nerf.initialize()
        if self.opt.nerf.fine_sampling:
            self.nerf_fine.initialize()

    def get_network_components(self):
        return [self.nerf] + ([self.nerf_fine] if self.opt.nerf.fine_sampling else [])

    def L1_loss(self, pred, label):
        return (pred.contiguous() - label).abs().mean()

    def MSE_loss(self, pred, label, mask=None):
        loss = (pred.contiguous() - label) ** 2
        if mask is not None:
            loss = loss[mask]
        return loss.mean()

    # ---------------------------------------------------------------------------- poses (overridable)
    def get_w2c_pose(self, opt, data_dict, mode=None):
        return data_dict.pose  # fixed GT poses; the joint trainers override this (joint_pose_nerf_trainer.py:718)

    def get_pose(self, opt, data_dict, mode=None):
        return self.get_w2c_pose(opt, data_dict, mode)

    def get_c2w_pose(self, opt, data_dict, mode=None):
        return _invert_pose(self.get_w2c_pose(opt, data_dict, mode))

    # ---------------------------------------------------------------------------- helpers
    @staticmethod
    def _depth_range(opt, data_dict):
        # renderer.py:104-108: python list for inverse depth, dataset tensor otherwise
        return opt.nerf.depth.range if opt.nerf.depth.param == "inverse" else data_dict.depth_range[0]

    @staticmethod
    def _range_floats(depth_range):
        """(near, far, far - near) as python floats carrying the reference's fp32 arithmetic: for metric depth the
        range is a device tensor (data_dict.depth_range[0]) and `far - near` an fp32 subtraction; for inverse depth
        a python list.  Device tensors are read back ONCE (cached): no per-step synchronisation."""
        lo, hi = depth_range[0], depth_range[1]
        if torch.is_tensor(lo):
            def read(t):
                v = t.detach().float().cpu()
                return float(v[0]), float(v[1]), float(v[1] - v[0])
            base = depth_range if torch.is_tensor(depth_range) else torch.stack([lo, hi])
            return ops.cached("range", base, read)
        near = float(torch.tensor(float(lo), dtype=torch.float32))
        far = float(torch.tensor(float(hi), dtype=torch.float32))
        return near, far, float(torch.tensor(float(hi - lo), dtype=torch.float32))

    @staticmethod
    def _fine_disabled(opt, iter, also_absolute=False):
        """True while the schedule keeps the fine network off (renderer.py:317-320, 576-581)."""
        if hasattr(opt.nerf, "ratio_start_fine_sampling_at_x") and opt.nerf.ratio_start_fine_sampling_at_x is not None \
                and iter is not None and iter < opt.max_iter * opt.nerf.ratio_start_fine_sampling_at_x:
            return True
        if also_absolute and hasattr(opt.nerf, "start_fine_sampling_at_x") and opt.nerf.start_fine_sampling_at_x is not None \
                and iter is not None and iter < opt.nerf.start_fine_sampling_at_x:
            return True
        return False

    def _rays(self, pose, intr, H, W, pixels, ray_idx):
        if pixels is not None:
            return ops.raygen(pose, intr, W, pixels=pixels.to(self.device))
        if ray_idx is None:
            ray_idx = torch.arange(H * W, device=self.device)
        return ops.raygen(pose, intr, W, ray_idx=ray_idx.to(self.device))

    # ---------------------------------------------------------------------------- public entry points
    def _full_or_selected(self, opt, pose, intr, H, W, depth_range, iter, mode, pixels=None, ray_idx=None):
        """The dispatch the three public entry points share: explicit pixels / ray indices -> one `render` call,
        otherwise the whole image, sliced when opt.nerf.rand_rays is set (renderer.py:181-187, 236-244)."""
        kw = dict(H=H, W=W, intr=intr, depth_range=depth_range, iter=iter, mode=mode)
        if pixels is not None or ray_idx is not None:
            ret = self.render(opt, pose, pixels=pixels, ray_idx=ray_idx, **kw)
            ret.ray_idx = ray_idx
            return ret
        return self.render_by_slices(opt, pose, **kw) if opt.nerf.rand_rays else self.render(opt, pose, **kw)

    def _train_subset(self, opt, H, W, mode, n_images):
        """Random pixel subset shared by all rendered images in train / test-optim mode (renderer.py:114, 124), else None."""
        if opt.nerf.rand_rays and mode in ("train", "test-optim"):
            return torch.randperm(H * W, device=self.device)[:opt.nerf.rand_rays // n_images]
        return None

    def forward(self, opt, data_dict, iter, img_idx=None, mode=None):
        """Render a random subset of pixels (train / test-optim) or all pixels of every image
        (renderer.py:77-140)."""
        H, W = data_dict.image.shape[-2:]
        if img_idx is not None:
            # (the reference passes img_idx into the `iter` slot here, renderer.py:117; no caller uses it)
            ray_idx = self._train_subset(opt, H, W, mode, len(img_idx) if isinstance(img_idx, list) else 1)
            ret = self.render_image_at_specific_rays(opt, data_dict, iter, img_idx=img_idx, ray_idx=ray_idx, mode=mode)
            if ray_idx is not None:
                ret.ray_idx = ray_idx
            ret.idx_img_rendered = img_idx
            return ret
        n_images = len(data_dict.idx)
        ray_idx = self._train_subset(opt, H, W, mode, n_images)
        ret = self._full_or_selected(opt, self.get_w2c_pose(opt, data_dict, mode=mode), data_dict.intr, H, W,
                                     self._depth_range(opt, data_dict), iter, mode, ray_idx=ray_idx)
        ret.idx_img_rendered = self._arange(n_images)
        return ret

    def render_image_at_specific_pose_and_rays(self, opt, data_dict, pose, intr, H, W, iter, pixels=None,
                                               ray_idx=None, mode="train"):
        """Render given pixels (or the full image) at given w2c pose(s) (renderer.py:142-190)."""
        pose = pose.unsqueeze(0) if pose.dim() == 2 else pose
        intr = intr.unsqueeze(0) if intr.dim() == 2 else intr
        return self._full_or_selected(opt, pose, intr, H, W, self._depth_range(opt, data_dict), iter, mode,
                                      pixels=pixels, ray_idx=ray_idx)

    def render_image_at_specific_rays(self, opt, data_dict, iter, img_idx=None, pixels=None, ray_idx=None,
                                      mode="train"):
        """Render given pixels for all (or a subset `img_idx`) of the scene's images (renderer.py:192-248)."""
        pose, intr = self.get_w2c_pose(opt, data_dict, mode=mode), data_dict.intr
        n_images = pose.shape[0]
        if img_idx is not None:
            if not isinstance(img_idx, (tuple, list)):
                img_idx = [img_idx]
            pose, intr = pose[img_idx].view(-1, 3, 4), intr[img_idx].view(-1, 3, 3)
        H, W = data_dict.image.shape[-2:]
        ret = self._full_or_selected(opt, pose, intr, H, W, self._depth_range(opt, data_dict), iter, mode,
                                     pixels=pixels, ray_idx=ray_idx)
        ret.idx_img_rendered = torch.from_numpy(np.array(img_idx)).to(self.device) if img_idx is not None else \
            self._arange(n_images)
        return ret

    def _arange(self, n):
        """arange(n) on the device, built once per n (the reference rebuilds it on every call, renderer.py:246)."""
        cache = self.__dict__.setdefault("_arange_cache", {})
        if n not in cache:
            cache[n] = torch.arange(start=0, end=n, device=self.device)
        return cache[n]

    # ---------------------------------------------------------------------------- occupancy grids
    def set_occupancy(self, grid, grid_fine=None):
        """Attach occupancy grids (sparf_b200.occupancy.OccupancyGrid) to the coarse and the fine network; None detaches.
        `render` then skips the samples a network's grid marks empty, but only in val / eval / test mode with gradients
        off: every other call renders densely.  Without a fine grid the fine pass stays dense."""
        self._occupancy = (grid, grid_fine)

    def set_training_occupancy(self, grid, grid_fine=None):
        """Attach occupancy grids for training: `render` in train and test-optim mode, with or without gradients, then
        evaluates only the samples a network's grid keeps (occupancy.train_forward_samples); the others get σ = 0,
        rgb = 0 and no gradient.  None detaches; without a fine grid the fine pass stays dense.  A grid is a snapshot:
        refresh it between steps with occupancy.refresh_, which writes into the same tensor, so that a captured step
        sees it.  Tensor-core engines only.  set_occupancy (inference) and render_to_max are unaffected."""
        self._train_occupancy = (grid, grid_fine)

    def set_early_termination(self, eps=1e-4, window=16):
        """Stop evaluating a ray once its transmittance is below eps (sparf_b200.termination), checked every `window`
        samples, in the coarse and the fine pass and on top of any occupancy grid; None detaches.  Like the grids it
        applies only in val / eval / test mode with gradients off."""
        if eps is None:
            self._termination = None
            return
        assert 0 <= eps < 1 and int(window) == window >= 1, (eps, window)
        self._termination = (float(eps), int(window))

    def set_training_termination(self, eps=1e-4, window=16):
        """Stop evaluating a ray in training once its transmittance is below eps, checked every `window` samples
        (termination.train_forward_samples): `render` in train and test-optim mode, with or without gradients, in the
        coarse and the fine pass, on top of the training grid a pass has (set_training_occupancy) or alone.  The samples
        skipped get σ = 0, rgb = 0 and no gradient; a step stays one CUDA graph.  None detaches.  Tensor-core engines
        only.  set_early_termination (inference) and render_to_max are unaffected."""
        if eps is None:
            self._train_termination = None
            return
        if isinstance(eps, bool) or not isinstance(eps, (int, float)) or not 0 <= eps < 1:
            raise ValueError("set_training_termination: eps %r (a number, 0 <= eps < 1)" % (eps,))
        if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or window < 1:
            raise ValueError("set_training_termination: window %r (an integer >= 1)" % (window,))
        self._train_termination = (float(eps), int(window))

    def set_normals(self, enabled=True):
        """Add normal maps to renders (sparf_b200.normals): `render` in val / eval / test mode with gradients off then also
        returns `normal` [B,N,3] (and `normal_fine` from the fine pass), the composite weight-sum of the density normals
        -grad(raw) / |grad(raw)| over the samples with w != 0: world-space and unnormalised (|normal| <= opacity).  Every
        other output is unchanged; train and test-optim renders, render_to_max and renders with gradients return no normal.
        False detaches."""
        if not isinstance(enabled, bool):
            raise ValueError("set_normals: enabled %r (True or False)" % (enabled,))
        self._normals = enabled

    def _add_normals(self, nerf, pred, center, ray, depth_samples, mode):
        if getattr(self, "_normals", False) and mode in ("val", "eval", "test") and not torch.is_grad_enabled():
            from . import normals
            pred["normal"] = normals.composite_normals(nerf, center, ray, depth_samples, pred["weights"])
        return pred

    def _forward_samples(self, nerf, which, opt, center, ray, depth_samples, mode):
        """nerf.forward_samples, or in val / eval / test mode without gradients termination.forward_samples when early
        termination is set, occupancy.forward_samples when only grid `which` (0 coarse, 1 fine) is attached; in train and
        test-optim mode termination.train_forward_samples (with training grid `which`, if any) when training termination
        is set, else occupancy.train_forward_samples when training grid `which` is attached"""
        train_grid = getattr(self, "_train_occupancy", (None, None))[which]
        train_term = getattr(self, "_train_termination", None)
        if train_term is not None and mode in ("train", "test-optim"):
            from . import termination
            return termination.train_forward_samples(nerf, train_grid, *train_term, opt, center, ray, depth_samples, mode)
        if train_grid is not None and mode in ("train", "test-optim"):
            from . import occupancy
            return occupancy.train_forward_samples(nerf, train_grid, opt, center, ray, depth_samples, mode)
        grid = getattr(self, "_occupancy", (None, None))[which]
        term = getattr(self, "_termination", None)
        if (grid is not None or term is not None) and mode in ("val", "eval", "test") and not torch.is_grad_enabled():
            if term is not None:
                from . import termination
                return termination.forward_samples(nerf, grid, *term, center, ray, depth_samples)
            from . import occupancy
            return occupancy.forward_samples(nerf, grid, center, ray, depth_samples)
        return nerf.forward_samples(opt, center, ray, depth_samples, embedder_pts=self.embedder_pts,
                                    embedder_view=self.embedder_view, mode=mode)

    # ---------------------------------------------------------------------------- core
    def render(self, opt, pose, H, W, intr, pixels=None, ray_idx=None, depth_range=None, iter=None, mode=None):
        """Coarse pass + optional hierarchical fine pass (renderer.py:250-345).  With an occupancy grid attached
        (set_occupancy), val / eval / test renders without gradients skip the samples it marks empty; with early
        termination set (set_early_termination), they also skip the samples behind an opaque point of the ray."""
        batch_size = len(pose)
        center, ray = self._rays(pose, intr, H, W, pixels, ray_idx)          # [B,N,3]
        pred = edict(origins=center, viewdirs=ray)
        depth_samples = self.sample_depth(opt, batch_size, num_rays=ray.shape[1], n_samples=opt.nerf.sample_intvs,
                                          H=H, W=W, depth_range=depth_range, mode=mode)   # [B,N,S,1]
        pred_coarse = self._forward_samples(self.nerf, 0, opt, center, ray, depth_samples, mode)
        pred_coarse["t"] = depth_samples
        pred_coarse = self._add_normals(self.nerf, self.nerf.composite(opt, ray, pred_coarse, depth_samples), center, ray,
                                        depth_samples, mode)
        pred.update(pred_coarse)
        if opt.nerf.fine_sampling and not self._fine_disabled(opt, iter):
            with torch.no_grad():
                det = mode not in ["train", "test-optim"] or (not opt.nerf.sample_stratified)
                depth_all = self._resample_and_merge(opt, pred_coarse["weights"][..., 0], depth_samples[..., 0],
                                                     depth_range, det)           # [B,N,S+Sf,1]
            pred_fine = self._forward_samples(self.nerf_fine, 1, opt, center, ray, depth_all, mode)
            pred_fine["t"] = depth_all
            pred_fine = self._add_normals(self.nerf_fine, self.nerf_fine.composite(opt, ray, pred_fine, depth_all), center,
                                          ray, depth_all, mode)
            pred.update({k + "_fine": v for k, v in pred_fine.items()})
        return pred

    def render_by_slices(self, opt, pose, H, W, intr, depth_range, iter, mode=None):
        """Full-image rendering in slices of opt.nerf.rand_rays pixels (renderer.py:347-381)."""
        keys = ["rgb", "rgb_var", "depth", "depth_var", "opacity", "normal", "all_cumulated"]
        if opt.nerf.fine_sampling and not self._fine_disabled(opt, iter):
            keys += [k + "_fine" for k in keys]
        ret_all = edict({k: [] for k in keys})
        step = opt.nerf.rand_rays
        if mode in ["val", "eval", "test"] or not (opt.nerf.sample_stratified or opt.nerf.density_noise_reg):
            # Nothing random is drawn in these modes (renderer.py:326, 404; frequency_nerf.py:191) and rays do not
            # interact, so the slice size does not change any output: use slices as large as comfortably fit, i.e. one
            # persistent forward-only kernel launch over (up to) 131072 rays instead of H*W / rand_rays small ones.
            step = max(step, self.full_image_rays_per_launch // max(1, len(pose)))
        for c in range(0, H * W, step):
            ray_idx = torch.arange(c, min(c + step, H * W), device=self.device)
            ret = self.render(opt, pose, H=H, W=W, intr=intr, ray_idx=ray_idx, depth_range=depth_range, iter=iter, mode=mode)
            for k in ret_all:
                if k in ret.keys():
                    ret_all[k].append(ret[k])
        for k in ret_all:
            ret_all[k] = torch.cat(ret_all[k], dim=1) if len(ret_all[k]) > 0 else None
        return ret_all

    # ---------------------------------------------------------------------------- sampling
    def sample_depth(self, opt, batch_size, n_samples, H, W, depth_range, num_rays=None, mode=None):
        """Stratified / mid-point depth samples, same range for every ray (renderer.py:383-419)."""
        depth_min, depth_max = depth_range
        num_rays = num_rays or H * W
        rand = None
        if opt.nerf.sample_stratified and mode not in ["val", "eval", "test"]:
            rand = torch.rand(batch_size, num_rays, n_samples, 1, device=self.device).to(self.device)
        near, _, rng = self._range_floats(depth_range)
        t = ops.sample_depth(batch_size * num_rays, n_samples, near, rng,
                             inverse=(opt.nerf.depth.param == "inverse"), rand=rand, device=self.device)
        return t.view(batch_size, num_rays, n_samples, 1)

    # renderer.py:439 draws the shared fine-sampling grid on the CPU generator and copies it over (a host->device
    # copy per step).  device_side_rng = True -- and always while a CUDA graph is being captured, where a pageable
    # host copy cannot be recorded -- draws the same U[0,1) grid with the device generator instead.
    device_side_rng = False
    # render_by_slices in the deterministic modes: rays (over all views) per forward launch
    full_image_rays_per_launch = 131072

    def _shared_grid_midpoints(self, n_samples_fine, det):
        # renderer.py:435-442: one grid for all rays
        if det:
            grid = torch.linspace(0, 1, n_samples_fine + 1, device=self.device)
        elif self.device_side_rng or torch.cuda.is_current_stream_capturing():
            grid = torch.rand(n_samples_fine + 1, device=self.device)
        else:
            grid = torch.rand(n_samples_fine + 1).to(self.device)
        return 0.5 * (grid[:-1] + grid[1:])

    def _resample_and_merge(self, opt, weights, t_coarse, depth_range, det):
        B, N, S = weights.shape
        near, far, _ = self._range_floats(depth_range)
        u = self._shared_grid_midpoints(opt.nerf.sample_intvs_fine, det)
        _, t_all = ops.sample_pdf_merge(weights.reshape(B * N, S), t_coarse.reshape(B * N, S), u, near, far)
        return t_all.view(B, N, -1, 1)

    def sample_depth_from_pdf(self, opt, weights, n_samples_coarse, n_samples_fine, depth_range, det):
        """Inverse-transform sampling of the coarse weights [B,N,S] -> [B,N,S_fine,1] (renderer.py:421-456)."""
        B, N, S = weights.shape
        near, far, _ = self._range_floats(depth_range)
        u = self._shared_grid_midpoints(n_samples_fine, det)
        dummy = torch.zeros(B * N, S, device=self.device)
        t_fine, _ = ops.sample_pdf_merge(weights.reshape(B * N, S), dummy, u, near, far)
        return t_fine.view(B, N, n_samples_fine, 1)

    # ---------------------------------------------------------------------------- per-ray far bound
    def render_up_to_maxdepth_at_specific_pose_and_rays(self, opt, data_dict, pose, intr, H, W, depth_max, iter,
                                                        pixels=None, ray_idx=None, mode="train"):
        """renderer.py:460-502."""
        if pose.dim() == 2:
            pose = pose.unsqueeze(0)
        if intr.dim() == 2:
            intr = intr.unsqueeze(0)
        depth_range = self._depth_range(opt, data_dict)
        ret = self.render_to_max(opt, pose, intr=intr, pixels=pixels, ray_idx=ray_idx, mode=mode, H=H, W=W,
                                 depth_min=self._range_floats(depth_range)[0], depth_max=depth_max, iter=iter)
        ret.ray_idx = ray_idx
        return ret

    def render_to_max(self, opt, pose, H, W, intr, pixels=None, ray_idx=None, depth_max=None, depth_min=None,
                      iter=None, mode=None):
        """Per-ray far bound; the fine network sees the SAME samples (renderer.py:504-593)."""
        batch_size = len(pose)
        center, ray = self._rays(pose, intr, H, W, pixels, ray_idx)
        pred = edict(origins=center, viewdirs=ray)
        depth_samples = self.sample_depth_diff_max_range_per_ray(opt, batch_size, num_rays=ray.shape[1],
                                                                 n_samples=opt.nerf.sample_intvs, H=H, W=W,
                                                                 depth_max=depth_max, depth_min=depth_min, mode=mode)
        pred_coarse = self.nerf.forward_samples(opt, center, ray, depth_samples, embedder_pts=self.embedder_pts,
                                                embedder_view=self.embedder_view, mode=mode)
        pred_coarse["t"] = depth_samples
        pred_coarse = self.nerf.composite(opt, ray, pred_coarse, depth_samples)
        pred.update(pred_coarse)
        if opt.nerf.fine_sampling and not self._fine_disabled(opt, iter, also_absolute=True):
            pred_fine = self.nerf_fine.forward_samples(opt, center, ray, depth_samples, embedder_pts=self.embedder_pts,
                                                       embedder_view=self.embedder_view, mode=mode)
            pred_fine["t"] = depth_samples
            pred_fine = self.nerf_fine.composite(opt, ray, pred_fine, depth_samples)
            pred.update({k + "_fine": v for k, v in pred_fine.items()})
        return pred

    def sample_depth_diff_max_range_per_ray(self, opt, batch_size, n_samples, H, W, depth_min, depth_max,
                                            num_rays=None, mode=None):
        """t_k = ((1+k)/S)(far_r - near) + near with a far bound per ray [B,N] (renderer.py:595-624)."""
        num_rays = num_rays or H * W
        t = ops.sample_depth(batch_size * num_rays, n_samples, float(depth_min), 0.0,
                             far_per_ray=depth_max.to(self.device).reshape(-1), device=self.device)
        return t.view(batch_size, num_rays, n_samples, 1)
