"""Ray-batch data parallelism for the hot path (SURVEY.md §8e).

The reference is single-GPU (`distributed = False`, base_trainer.py:104).  Rays are independent, so
the natural multi-GPU scheme is: one process per GPU, identical replicas of the MLPs and poses, every
rank renders its shard of the step's ray batch, and the only exchange is ONE all-reduce (sum) of a flat
fp32 gradient buffer `[d theta_coarse | d theta_fine | d pose]` per step.  Loss means are taken over the
global batch, so each rank scales its local mean by (local rays / global rays) before backward; clip
and Adam then run replicated on the reduced buffer and stay in lock-step.
"""
from __future__ import annotations

from typing import Iterable, List, Optional

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int):
    """Contiguous shard [lo, hi) of n items for `rank` (sizes differ by at most one)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_rays(ray_idx: torch.Tensor, rank: Optional[int] = None, world: Optional[int] = None) -> torch.Tensor:
    """Rank's slice of a shared (n,) or per-image (B,n) ray-index tensor: the union over ranks is the
    single-GPU batch (same seeded randperm on every rank)."""
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    lo, hi = shard_range(ray_idx.shape[-1], rank, world)
    return ray_idx[..., lo:hi]


class FlatGradients:
    """Points every parameter's `.grad` at a view of one flat fp32 buffer so that zeroing, the global-norm
    clip and the all-reduce are single operations.

    Contract with the optimiser loop: zero gradients with `fg.zero_()` (or `optimizer.zero_grad(set_to_none=False)`),
    NOT with the default `zero_grad()`, which sets `.grad = None` and thereby detaches the parameters from the flat
    buffer.  `all_reduce` / `clip_grad_norm_` / `has_nonfinite` verify the aliasing first: a detached `.grad = None` is
    re-attached, a `.grad` that points at other storage raises (its contents would silently miss the collective).
    The `progress` scalar of the NeRF modules (written via `.data.fill_`, never differentiated) is left out."""

    def __init__(self, modules: Iterable[torch.nn.Module], skip_names=("progress",)):
        self.params: List[torch.nn.Parameter] = []
        seen = set()
        for m in modules:
            for name, p in m.named_parameters():
                if p.requires_grad and id(p) not in seen and name.split(".")[-1] not in skip_names:
                    seen.add(id(p))
                    self.params.append(p)
        dev = self.params[0].device
        self.flat = torch.zeros(sum(p.numel() for p in self.params), device=dev, dtype=torch.float32)
        self._views = []
        o = 0
        for p in self.params:
            v = self.flat[o:o + p.numel()].view_as(p)
            self._views.append(v)
            p.grad = v
            # this parameter has persistent, contiguous fp32 .grad storage: the MLP backward kernels may accumulate
            # into it directly (every MLP and density pass of ops takes that route when all the parameters of its call
            # carry the mark: ops._inplace_refs)
            p._sparf_inplace_grad = True
            o += p.numel()

    def check_attached(self):
        for p, v in zip(self.params, self._views):
            if p.grad is None:
                p.grad = v                      # optimizer.zero_grad(set_to_none=True): re-attach (the view is zeroed by zero_())
            elif p.grad.data_ptr() != v.data_ptr():
                raise RuntimeError("FlatGradients: a parameter's .grad no longer aliases the flat buffer (use fg.zero_() "
                                   "or zero_grad(set_to_none=False)); its gradient would miss the all-reduce")

    def zero_(self):
        self.check_attached()
        self.flat.zero_()

    def all_reduce(self, group=None):
        """Sum over ranks (one collective per step).  No-op in a single process."""
        self.check_attached()
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)

    def clip_grad_norm_(self, max_norm: float) -> torch.Tensor:
        """Global-norm clip on the (already reduced) flat buffer; same semantics as
        torch.nn.utils.clip_grad_norm_ over all parameters (base.py:96-97, iter_based_trainer.py:144-146)."""
        self.check_attached()
        total = self.flat.norm(2)
        coef = (max_norm / (total + 1e-6)).clamp(max=1.0)
        self.flat.mul_(coef)
        return total

    def has_nonfinite(self) -> torch.Tensor:
        """Decision for the NaN/Inf 'skip step' guard, taken on the reduced buffer so ranks agree."""
        self.check_attached()
        return ~torch.isfinite(self.flat).all()


def global_mean_scale(n_local: int, n_global: int) -> float:
    """Factor turning a local mean over n_local rays into this rank's share of the global mean."""
    return float(n_local) / float(n_global)
