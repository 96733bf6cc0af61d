"""Pose-parameter modules vs the reference's own modules.  The reference module's outputs on the same inputs are
stored in tests/golden/ref_pose_quaternion.npz (tests/golden/make_module_golden.py)."""
import os

import numpy as np
import pytest
import torch

import common
from sparf_b200.poses_models import QuaternionsPoseParameters
from sparf_b200.utils.edict import edict

REF_CASES = [(False, False, True, True), (True, True, True, True), (True, False, False, True), (False, True, True, False)]


def _opt(c2w, rel, rot=True, trans=True):
    opt = edict()
    opt.camera = edict(optimize_c2w=c2w, optimize_trans=trans, optimize_rot=rot, optimize_relative_poses=rel,
                       n_first_fixed_poses=1)
    return opt


def _poses(seed, n=4):
    data = common.make_scene(seed, n, 24, 32)
    return common.perturb_poses(data.pose, seed)


@pytest.mark.parametrize("c2w", [False, True])
@pytest.mark.parametrize("rel", [False, True])
def test_quaternion_pose_model_round_trip_and_gradients(c2w, rel):
    w2c = _poses(3)
    m = QuaternionsPoseParameters(_opt(c2w, rel), 4, w2c, torch.device("cpu"))
    assert torch.allclose(m.get_w2c_poses(), w2c, atol=2e-6)
    assert m.rot_embedding.shape == (4 - (1 if rel else 0), 4)
    loss = (m.get_w2c_poses() * torch.linspace(-1, 1, 48).view(4, 3, 4)).sum()
    loss.backward()
    assert m.rot_embedding.grad.abs().sum() > 0 and m.trans_embedding.grad.abs().sum() > 0


def _move(m, rot, trans):
    """move a pose model off its initial value (same way for ours and the reference's)"""
    with torch.no_grad():
        if rot:
            m.rot_embedding += 0.05 * torch.arange(m.rot_embedding.numel()).view_as(m.rot_embedding).float().cos()
        if trans:
            m.trans_embedding += 0.1


@pytest.mark.parametrize("c2w,rel,rot,trans", REF_CASES)
def test_quaternion_pose_model_matches_reference_module(c2w, rel, rot, trans):
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pose_quaternion.npz"))
    i = REF_CASES.index((c2w, rel, rot, trans))
    w2c = torch.from_numpy(gold["pose%d_input_w2c" % i])     # the poses the reference module was built from
    ours = QuaternionsPoseParameters(_opt(c2w, rel, rot, trans), 4, w2c, torch.device("cpu"))
    assert torch.allclose(torch.as_tensor(ours.rot_embedding), torch.from_numpy(gold["pose%d_rot_init" % i]), atol=1e-6)
    _move(ours, rot, trans)
    assert torch.allclose(ours.get_w2c_poses(), torch.from_numpy(gold["pose%d_w2c" % i]), atol=1e-6)
    assert torch.allclose(ours.get_c2w_poses(), torch.from_numpy(gold["pose%d_c2w" % i]), atol=1e-6)
