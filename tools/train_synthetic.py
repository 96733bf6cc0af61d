#!/usr/bin/env python
"""End-to-end training loop on the CUDA path, reference-shaped: `RaySamplingStrategy` -> `Graph.render...` ->
`define_loss(...).compute_loss` -> `backward()` -> fused clip + Adam + ExponentialLR, the WHOLE iteration captured once
as a CUDA graph and replayed (source/training/nerf_trainer.py:207-275 `train_iteration` + iter_based_trainer.py:128-147).

The scene is synthetic (no datasets in this image): a "teacher" NeRF with fixed random weights renders the training views
(full-image inference through `render_by_slices`); a freshly initialised "student" of the same architecture is trained on
them.  Prints the photometric loss as it goes; `main()` returns (first_losses, last_losses) for the convergence test.

    python tools/train_synthetic.py [--steps 400] [--views 3] [--size 48 64] [--rays 1024] [--fine 0] [--grid RES]

--grid RES trains with occupancy grids of RES^3 cells (Graph.set_training_occupancy), rebuilt from the student's weights
every --grid-every steps between graph replays (occupancy.refresh_); `main()` then also returns the fraction of the
training samples the grids keep at the end.  --grid-update N keeps the grids current on the device instead: every
--grid-every steps a CUDA graph of its own, captured once, replays occupancy.update_(grid, net, N, N) on each network
(N cells drawn uniformly and N from the occupied ones, per-cell density decay 0.95), with no host-side rebuild.  --term EPS adds early ray termination to the training steps
(Graph.set_training_termination(EPS, --term-window)), alone or on top of the grids; the kept fraction is then returned
as well.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch

import common


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--views", type=int, default=3)
    ap.add_argument("--size", type=int, nargs=2, default=[48, 64])
    ap.add_argument("--rays", type=int, default=1024)
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--fine", type=int, default=0)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--poses", type=int, default=0, help="1: joint pose-NeRF training from perturbed poses (BARF c2f mask)")
    ap.add_argument("--pose-noise", type=float, default=0.03)
    ap.add_argument("--lr-pose", type=float, default=2e-3)
    ap.add_argument("--engine", default="auto", help="MLP engine (auto | tc_3x | tc_3x_w1 | simt_fp32)")
    ap.add_argument("--grid", type=int, default=0, help="occupancy grids of RES^3 cells in the training steps (0: dense)")
    ap.add_argument("--grid-every", type=int, default=16, help="steps between grid refreshes or updates")
    ap.add_argument("--grid-update", type=int, default=0, help="N: update the grids on the device (occupancy.update_ "
                    "with N uniform and N occupied cells, in a graph of its own) instead of rebuilding them (0: refresh_)")
    ap.add_argument("--grid-thres", type=float, default=0.01, help="density threshold of the grids")
    ap.add_argument("--term", type=float, default=None, help="early ray termination at transmittance EPS in the training "
                    "steps (default: off)")
    ap.add_argument("--term-window", type=int, default=16, help="samples per termination window")
    ap.add_argument("--quiet", action="store_true")
    args = ap.parse_args(argv)

    import sparf_b200
    from sparf_b200.graphs import GraphedStep
    from sparf_b200.losses import define_loss
    from sparf_b200.optim import FlatParameters, FusedAdam
    from sparf_b200.renderer import Graph
    from sparf_b200.sampling_strategies import RaySamplingStrategy

    sparf_b200.set_engine(args.engine)
    dev = torch.device("cuda")
    B, (H, W) = args.views, args.size
    opt = common.make_opt(S=args.samples, S_fine=args.samples, fine=bool(args.fine), rand_rays=args.rays, stratified=True,
                          depth_range=(1.2, 5.2), barf_c2f=(0.1, 0.5) if args.poses else None)
    opt.sample_fraction_in_fg_mask = 0.0
    opt.sampled_fraction_in_center = 0.0
    data = common.make_scene(0, B, H, W)
    data.depth_range = torch.tensor([[1.2, 5.2]] * B)
    for k in ("image", "intr", "pose", "depth_range", "idx"):
        data[k] = data[k].to(dev)

    # ---- teacher: fixed "peaky" weights, renders the ground-truth views (val mode: deterministic, full image)
    teacher = Graph(opt, dev)
    teacher.nerf.load_state_dict(common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0, progress=1.0))
    if args.fine:
        teacher.nerf_fine.load_state_dict(common.det_weights(opt, 82, peaky=True, sigma_bias=-2.0, progress=1.0))
    teacher.eval()
    with torch.no_grad():
        full = teacher.forward(opt, data, iter=10 ** 9, mode="val")
        rgb = full["rgb_fine"] if args.fine else full["rgb"]
    data.image = rgb.reshape(B, H, W, 3).permute(0, 3, 1, 2).contiguous()

    # ---- student + the reference-shaped training objects
    torch.manual_seed(0)
    pose_net = None
    if args.poses:      # joint pose-NeRF training (joint_pose_nerf_trainer.py): perturbed initial poses, 9-D embedding
        from sparf_b200.poses_models import FirstTwoColunmnsPoseParameters
        init = common.perturb_poses(data.pose.cpu(), 0, sigma=args.pose_noise).to(dev)
        pose_net = FirstTwoColunmnsPoseParameters(opt, nbr_poses=B, initial_poses_w2c=init, device=dev).to(dev)

        class PoseGraph(Graph):
            def get_w2c_pose(self, opt, data_dict, mode=None):
                return pose_net.get_w2c_poses()

        net = PoseGraph(opt, dev)
    else:
        net = Graph(opt, dev)
    net.train()
    net.device_side_rng = True

    def pose_error():
        """mean rotation angle (deg) and camera-centre distance between the current estimates and the true poses, WITHOUT
        the similarity alignment the reference's evaluation applies first (a jointly optimised scene is only defined up to
        a global similarity, so this number need not shrink; it is printed for orientation only)"""
        est, gt = pose_net.get_w2c_poses().detach(), data.pose
        R = est[:, :, :3] @ gt[:, :, :3].transpose(1, 2)
        ang = torch.acos(((R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2] - 1) / 2).clamp(-1, 1)) * 180 / 3.14159265
        c_est = -(est[:, :, :3].transpose(1, 2) @ est[:, :, 3:])[..., 0]
        c_gt = -(gt[:, :, :3].transpose(1, 2) @ gt[:, :, 3:])[..., 0]
        return ang.mean().item(), (c_est - c_gt).norm(dim=-1).mean().item()

    class TrainData:
        all = data

        def __len__(self):
            return B

    loss_module = define_loss("photometric", opt, net, TrainData(), dev)
    loss_module.check_finite = False
    sampler = RaySamplingStrategy(opt, data_dict=data, device=dev)
    flat = FlatParameters(net.get_network_components())
    adam = FusedAdam(flat, lr=args.lr, gamma=(1e-4 / args.lr) ** (1.0 / max(args.steps, 1)), max_norm=0.1)
    flat_pose = adam_pose = None
    if pose_net is not None:      # second optimiser group: poses, unclipped (default_config.py:43), own learning rate
        flat_pose = FlatParameters([pose_net])
        adam_pose = FusedAdam(flat_pose, lr=args.lr_pose, gamma=(1e-5 / args.lr_pose) ** (1.0 / max(args.steps, 1)))
    progress_step = torch.full((), 1.0 / max(args.steps, 1), device=dev)

    def iteration():
        flat.zero_grad()
        if flat_pose is not None:
            flat_pose.zero_grad()
            for m in net.get_network_components():           # BARF schedule: progress = iteration / max_iter, on the device
                m.progress.data.add_(progress_step).clamp_(max=1.0)
        rays = sampler(opt.nerf.rand_rays)                       # device-side torch.randperm: fresh rays every replay
        out = net.render_image_at_specific_rays(opt, data, iter=0, ray_idx=rays, mode="train")
        loss = loss_module.compute_loss(opt, data, out, iteration=0, mode="train")[0]["all"]
        loss.backward()
        adam.step()
        if adam_pose is not None:
            adam_pose.step()
        return loss.detach()

    err0 = pose_error() if pose_net is not None else None

    grids = []
    if args.grid:     # built before the capture: the graph reads the grids' bits, which refresh_ rewrites in place
        from sparf_b200 import occupancy
        grids = [occupancy.build_grid(opt, m, res=args.grid, thres=args.grid_thres, ema=bool(args.grid_update))
                 for m in net.get_network_components()]
        net.set_training_occupancy(*grids)
    grid_step = None
    if grids and args.grid_update:

        def grid_update():
            for g, m in zip(grids, net.get_network_components()):
                occupancy.update_(g, m, args.grid_update, args.grid_update)
        grid_step = GraphedStep(grid_update, (), warmup=1)
    if args.term is not None:
        net.set_training_termination(args.term, args.term_window)

    step = GraphedStep(iteration, (), warmup=2)
    losses = []
    for it in range(args.steps):
        if grid_step is not None and it % args.grid_every == 0 and it > 0:
            grid_step()
        elif grids and grid_step is None and it % args.grid_every == 0:
            for g, m in zip(grids, net.get_network_components()):
                occupancy.refresh_(g, opt, m)
        losses.append(step().clone())     # (the graph's output tensor is static: keep a copy of its value)
        if not args.quiet and (it % 50 == 0 or it == args.steps - 1):
            print("iter %4d  photometric loss %.5f" % (it, float(losses[-1])))
    torch.cuda.synchronize()
    vals = torch.stack(losses).float().cpu()
    k = max(1, args.steps // 10)
    extra = ()
    if grids or args.term is not None:     # kept fraction of the coarse samples of a training batch (skipped: σ = 0 exactly)
        with torch.no_grad():
            out = net.render_image_at_specific_rays(opt, data, iter=0, ray_idx=sampler(opt.nerf.rand_rays), mode="train")
        extra = ((out["density_samples"] != 0).float().mean().item(),)
        if not args.quiet:
            print("kept fraction of the coarse samples: %.3f" % extra[0])
    if pose_net is not None:
        err1 = pose_error()
        if not args.quiet:
            print("unaligned pose offset (rotation deg, camera centre): initial %.3f / %.4f -> final %.3f / %.4f" % (err0 + err1))
        return (vals[:k].mean().item(), vals[-k:].mean().item(), err0, err1) + extra
    return (vals[:k].mean().item(), vals[-k:].mean().item()) + extra


if __name__ == "__main__":
    res = main()
    first, last = res[0], res[1]
    print("mean loss of the first 10%% of the iterations: %.5f   of the last 10%%: %.5f" % (first, last))
