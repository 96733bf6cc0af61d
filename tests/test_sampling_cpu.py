"""RaySamplingStrategy / sample_rays mirrors (sparf_b200/sampling_strategies.py) against the reference's own classes:
same pools, same torch.randperm draws in the same order => identical rays under one seed.  The reference's draws are
stored in tests/golden/ref_ray_sampling.npz (tests/golden/make_module_golden.py)."""
import os

import numpy as np
import pytest
import torch

import common

CASES = [dict(), dict(sampled_fraction_in_center=0.25), dict(depth_patch=0), dict(depth_patch=0, sampled_fraction_in_center=0.5)]
SAMPLE_RAYS_KW = [dict(nbr=50), dict(nbr=64, fraction_in_center=0.25), dict()]


def _opt(**kw):
    opt = common.make_opt(rand_rays=96)
    opt.sample_fraction_in_fg_mask = 0.0
    opt.sampled_fraction_in_center = 0.0
    opt.depth_regu_patch_size = 2
    for k, v in kw.items():
        if k == "depth_patch":
            opt.loss_weight.depth_patch = v
        else:
            opt[k] = v
    return opt


def _gold():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ray_sampling.npz"))


@pytest.mark.parametrize("case", CASES)
def test_ray_sampling_strategy_matches_reference(case):
    from sparf_b200.sampling_strategies import RaySamplingStrategy, sample_rays
    gold = _gold()
    i = CASES.index(case)
    ours = RaySamplingStrategy(_opt(**case), common.make_scene(3, 3, 24, 32), torch.device("cpu"))
    for center in (False, True):
        torch.manual_seed(5)
        a = ours(96, sample_in_center=center)
        b = torch.from_numpy(gold["case%d_center%d" % (i, center)])
        assert a.shape == b.shape and torch.equal(a, b)
    for j, kw in enumerate(SAMPLE_RAYS_KW):
        torch.manual_seed(9)
        pa, ra = sample_rays(24, 32, **kw)
        assert torch.equal(pa, torch.from_numpy(gold["sample_rays%d_pixels" % j]))
        assert torch.equal(ra, torch.from_numpy(gold["sample_rays%d_idx" % j]))
