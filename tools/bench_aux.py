#!/usr/bin/env python
"""Secondary measurements (not the bench line): full-image inference through
Graph.render_by_slices (SURVEY 8f.3) and the hierarchical (coarse + fine network) training step, DTU-shaped."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch

import common
from sparf_b200 import ops
from sparf_b200.renderer import Graph


def ev_time(fn, n, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    dev = torch.device("cuda")
    B, H, W = 3, 300, 400
    data = common.make_scene(0, B, H, W, focal=400.0)
    data.depth_range = torch.tensor([[1.2, 5.2]] * B)
    for k in ("image", "intr", "pose", "depth_range", "idx"):
        data[k] = data[k].to(dev)

    # ---- full-image inference, one view, slices of 8192 rays, coarse 128 (+ fine 128 + 128)
    for fine in (False, True):
        opt = common.make_opt(S=128, S_fine=128, fine=fine, rand_rays=8192, stratified=False, noise=False)
        net = Graph(opt, dev).eval()
        pose, intr = data.pose[:1], data.intr[:1]

        def infer():
            with torch.no_grad():
                net.render_by_slices(opt, pose, H, W, intr, data.depth_range[0], iter=10 ** 9, mode="val")
        ms = ev_time(infer, 3)
        samples = H * W * (128 + (256 if fine else 0))
        print("inference %dx%d, %s: %.1f ms / image, %.1f M rays/s, %.0f M sample-evaluations/s" %
              (H, W, "coarse 128 + fine 256" if fine else "coarse 128", ms, H * W / ms / 1e3, samples / ms / 1e3))

    # ---- hierarchical training step (BASELINE config 2 with fine_sampling=True): 1023 rays, 128 + 256 samples
    opt = common.make_opt(S=128, S_fine=128, fine=True, rand_rays=1024, stratified=True, noise=False)
    net = Graph(opt, dev).train()
    from sparf_b200.distributed import FlatGradients
    fg = FlatGradients([net])
    image_flat = data.image.reshape(B, 3, -1).permute(0, 2, 1).contiguous()
    idx = torch.randperm(H * W, device=dev)[:341]

    def step():
        fg.zero_()
        out = net.render_image_at_specific_rays(opt, data, iter=10 ** 9, ray_idx=idx, mode="train")
        gt = image_flat[:, idx]
        loss = ops.huber2(out.rgb, gt) + ops.huber2(out.rgb_fine, gt)
        loss.backward()
    ms = ev_time(step, 20, warm=3)
    print("hierarchical training step (eager): %.2f ms, %.0f k rays/s (1023 rays, 128 coarse + 256 fine samples)" %
          (ms, 1023 / ms))


if __name__ == "__main__":
    main()
