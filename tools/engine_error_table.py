#!/usr/bin/env python
"""Error of every MLP engine against the fp64 oracle at the headline shape (3 views 300x400, 3 x 341 rays x 128 samples,
photometric loss, gradients of the 20 MLP tensors and of the 9-D pose embedding), next to the error of the reference's
own fp32 arithmetic (the oracle run in fp32 on the same GPU, TF32 off), and the time of one forward + backward.

    python tools/engine_error_table.py [--out FILE.md]

Columns: max-normalised error  max|x - exact| / max|exact|  and relative L2 error  ||x - exact|| / ||exact||, the worst
tensor of each group.  (Test infrastructure: imports oracle/ through tests/test_headline_parity.py.)
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import numpy as np
import torch

import common
from test_headline_parity import _oracle_step

GROUPS = (("trunk weights", lambda k: k.startswith("mlp_feat") and k.endswith("weight")),
          ("trunk biases", lambda k: k.startswith("mlp_feat") and k.endswith("bias")),
          ("colour-head weights", lambda k: k.startswith("mlp_rgb") and k.endswith("weight")),
          ("colour-head biases", lambda k: k.startswith("mlp_rgb") and k.endswith("bias")),
          ("pose embedding", lambda k: k == "pose_embedding"))


def errs(x, ex):
    x, ex = x.double().reshape(-1), ex.double().reshape(-1)
    return (float((x - ex).abs().max() / ex.abs().max().clamp_min(1e-300)),
            float((x - ex).norm() / ex.norm().clamp_min(1e-300)))


def run_ours(engine, opt, sd, data_dev, init_w2c, ray_idx, dev, reps=5):
    import sparf_b200
    from sparf_b200.losses import BasePhotoandReguLoss
    from sparf_b200.poses_models import FirstTwoColunmnsPoseParameters
    from sparf_b200.renderer import Graph

    sparf_b200.set_engine(engine)
    B = data_dev.image.shape[0]
    pose_net = FirstTwoColunmnsPoseParameters(opt, nbr_poses=B, initial_poses_w2c=init_w2c.to(dev), device=dev).to(dev)

    class PoseGraph(Graph):
        def get_w2c_pose(self, opt, data_dict, mode=None):
            return pose_net.get_w2c_poses()

    net = PoseGraph(opt, dev)
    net.nerf.load_state_dict(sd)
    net.to(dev).train()
    loss_mod = BasePhotoandReguLoss(opt, net, train_data=None, device=dev)
    times = []
    for r in range(reps):
        for p in list(net.parameters()) + list(pose_net.parameters()):
            p.grad = None
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = net.render_image_at_specific_rays(opt, data_dev, iter=10, ray_idx=ray_idx.to(dev), mode="train")
        loss = loss_mod.compute_loss(opt, data_dev, out, iteration=10, mode="train")[0].render
        loss.backward()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    outs = {k: out[k].detach().double().cpu() for k in ("rgb", "depth", "opacity")}
    grads = {k: p.grad.detach().double().cpu() for k, p in net.nerf.named_parameters() if k != "progress"}
    grads["pose_embedding"] = pose_net.pose_embedding.grad.detach().double().cpu()
    return outs, float(loss), grads, min(times)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--engines", nargs="*", default=["simt_fp32", "tc_3x", "tc_3x_w1", "tc_1x"])
    args = ap.parse_args(argv)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    B, H, W, n, S = 3, 300, 400, 341, 128
    opt = common.make_opt(S=S, rand_rays=1024, barf_c2f=(0.1, 0.5))
    sd = common.det_weights(opt, 21, peaky=True, sigma_bias=-3.0, progress=0.35)
    data = common.make_scene(21, B, H, W, focal=400.0)
    data.depth_range = torch.tensor([[1.2, 5.2]] * B)
    init_w2c = common.perturb_poses(data.pose, 21, sigma=0.02)
    ray_idx = torch.from_numpy(np.random.default_rng(21).permutation(H * W)[:n].astype(np.int64))

    exact = _oracle_step(opt, sd, data, init_w2c, ray_idx, torch.float64, dev)
    rows = [("reference arithmetic (oracle, fp32 torch)",) + _oracle_step(opt, sd, data, init_w2c, ray_idx, torch.float32, dev) + (None,)]
    data_dev = data
    for k in ("image", "intr", "pose", "depth_range", "idx"):
        data_dev[k] = data_dev[k].to(dev)
    for eng in args.engines:
        rows.append(("sparf_b200 `%s`" % eng,) + run_ours(eng, opt, sd, data_dev, init_w2c, ray_idx, dev))

    lines = ["# Engine error against the fp64 oracle, headline shape (1023 rays x 128 samples, loss + all gradients)", "",
             "`python tools/engine_error_table.py` on one H100.  Each cell: max-normalised error / relative L2 error of the worst",
             "tensor of the group; ms = best of 5 eager forward + backward passes through the public API (no CUDA graph).", "",
             "| arithmetic | rgb | depth | loss (rel) | " + " | ".join(g for g, _ in GROUPS) + " | ms |",
             "|---|---|---|---|" + "---|" * len(GROUPS) + "---:|"]
    for name, outs, loss, grads, ms in rows:
        cells = ["%.1e / %.1e" % errs(outs[k].reshape(exact[0][k].shape), exact[0][k]) for k in ("rgb", "depth")]
        cells.append("%.1e" % (abs(loss - exact[1]) / abs(exact[1])))
        for _, sel in GROUPS:
            e = [errs(grads[k], exact[2][k]) for k in exact[2] if sel(k)]
            cells.append("%.1e / %.1e" % (max(x[0] for x in e), max(x[1] for x in e)))
        lines.append("| %s | %s | %s |" % (name, " | ".join(cells), "-" if ms is None else "%.2f" % ms))
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
