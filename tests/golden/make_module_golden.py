#!/usr/bin/env python
"""Fixtures of tests/test_pose_models_cpu.py and tests/test_sampling_cpu.py: outputs of the reference's own
QuaternionsPoseParameters, RaySamplingStrategy and sample_rays on the inputs those tests build.

    python tests/golden/make_module_golden.py      (needs the reference, see oracle/ref_loader.py)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import common  # noqa: E402
import test_pose_models_cpu as P  # noqa: E402
import test_sampling_cpu as T  # noqa: E402


def main():
    from oracle import ref_loader
    S = ref_loader.load("trainer").sampling
    from source.models.poses_models.quaternion import QuaternionsPoseParameters as Ref

    out = {}
    for i, (c2w, rel, rot, trans) in enumerate(P.REF_CASES):
        w2c = P._poses(5)
        out["pose%d_input_w2c" % i] = w2c.numpy().copy()
        ref = Ref(P._opt(c2w, rel, rot, trans), 4, w2c, torch.device("cpu"))
        out["pose%d_rot_init" % i] = torch.as_tensor(ref.rot_embedding).detach().numpy().copy()
        P._move(ref, rot, trans)
        out["pose%d_w2c" % i] = ref.get_w2c_poses().detach().numpy()
        out["pose%d_c2w" % i] = ref.get_c2w_poses().detach().numpy()
    np.savez_compressed(os.path.join(HERE, "ref_pose_quaternion.npz"), **out)

    out = {}
    for i, case in enumerate(T.CASES):
        theirs = S.RaySamplingStrategy(T._opt(**case), data_dict=common.make_scene(3, 3, 24, 32), device=torch.device("cpu"))
        for center in (False, True):
            torch.manual_seed(5)
            out["case%d_center%d" % (i, center)] = theirs(96, sample_in_center=center).numpy()
    for j, kw in enumerate(T.SAMPLE_RAYS_KW):
        torch.manual_seed(9)
        pb, rb = S.sample_rays(24, 32, **kw)
        out["sample_rays%d_pixels" % j], out["sample_rays%d_idx" % j] = pb.numpy(), rb.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_ray_sampling.npz"), **out)


if __name__ == "__main__":
    main()
