"""Loss layer (sparf_b200/losses.py): CPU checks of the host-side geometry / aggregation, and the full
SPARF step (photometric + correspondence + depth-consistency, 6 render calls) on the GPU against the
golden produced by the reference's own loss modules (tests/golden/make_golden.py: run_loss_case)."""
import numpy as np
import pytest
import torch

import common
from helpers import RandomReplayer, check_grads, load_golden


def test_geometry_roundtrip_cpu():
    from sparf_b200 import losses as L
    g = torch.Generator().manual_seed(0)
    K = torch.tensor([[40.0, 0, 16], [0, 40.0, 12], [0, 0, 1]])
    T = torch.eye(4)
    T[:3, 3] = torch.tensor([0.1, -0.2, 0.3])
    px = torch.rand(50, 2, generator=g) * 20 + 2
    d = torch.rand(50, generator=g) * 3 + 1
    X = L.batch_backproject_to_3d(px, d, K, L.pose_inverse_4x4(T))     # camera -> world
    uv, z = L.batch_project(X, T, K, return_depth=True)                 # world -> same camera
    assert torch.allclose(uv, px, atol=2e-4) and torch.allclose(z, d, atol=1e-5)
    uv2 = L.batch_project_to_other_img(px, d, K, K, torch.eye(4))
    assert torch.allclose(uv2, px, atol=2e-4)
    M = torch.eye(4)
    M[:3, :3] = torch.linalg.qr(torch.randn(3, 3, generator=g))[0]
    M[:3, 3] = torch.randn(3, generator=g)
    assert torch.allclose(L.pose_inverse_4x4(M) @ M, torch.eye(4), atol=1e-5)


def test_loss_aggregation_cpu():
    from sparf_b200 import losses as L
    opt = common.make_opt()
    opt.loss_weight.corres = -3.0

    class Fixed:
        def __init__(self, d):
            self.d = d

        def compute_loss(self, *a, **k):
            return {k: torch.tensor(v) for k, v in self.d.items()}, {}, {}

    agg = L.Loss([Fixed({"render": 0.5}), Fixed({"corres": 20.0})])
    out, _, _ = agg.compute_loss(opt, None, None, iteration=0, mode="train")
    assert abs(float(out["all"]) - (0.5 + 20.0 * 1e-3)) < 1e-6
    assert abs(float(out["corres_after_w"]) - 0.02) < 1e-7


def test_sample_rays_and_nearest_pose_cpu():
    from sparf_b200 import losses as L
    torch.manual_seed(0)
    px, flat = L.sample_rays(24, 32, nbr=100)
    assert px.shape == (100, 2) and px[:, 0].max() <= 30 and px[:, 1].max() <= 22
    assert torch.equal(flat, (px[:, 1] * 32 + px[:, 0]).long())
    poses = np.stack([np.eye(4)] * 3)
    poses[0, :3, 3] = [0, 0, -3]
    poses[1, :3, 3] = [0.3, 0, -3]
    poses[2, :3, 3] = [3, 0, 0]
    assert L.get_nearest_pose_ids(poses[0], poses, tar_id=0) == 1


def _loss_case_setup(name, dev):
    gold = load_golden(name)
    c, opt, data, ray_idx, sd, sd_fine, init_w2c = common.loss_case_inputs(name)
    for k in ("image", "intr", "pose", "depth_range", "idx", "colmap_depth", "colmap_conf"):
        if k in data:
            data[k] = data[k].to(dev)
    return gold, c, opt, data, ray_idx.to(dev), sd, sd_fine, init_w2c.to(dev)


class _TrainData:
    def __init__(self, d, n):
        self.all, self.n = d, n

    def __len__(self):
        return self.n


def _run_and_check(name, engine, gold, c, opt, data, ray_idx, net, loss_module, pose_embedding, gtol, gnorm="max"):
    with RandomReplayer(gold):
        data["iter"] = c["iteration"]
        out = net.render_image_at_specific_rays(opt, data, iter=c["iteration"], ray_idx=ray_idx, mode="train")
        data.poses_w2c = net.get_w2c_pose(opt, data, mode="train")
        loss_dict, stats, _ = loss_module.compute_loss(opt, data, out, iteration=c["iteration"], mode="train")
    loss_dict["all"].backward()
    torch.cuda.synchronize()
    rep = {}
    for k in [k[5:] for k in gold if k.startswith("loss_") and not k.endswith("_after_w")]:
        ref = float(gold["loss_" + k])
        got = float(loss_dict[k])
        rep[k] = abs(got - ref) / max(abs(ref), 1e-6)
        # correspondence / depth-consistency / sparse-depth terms sit behind hierarchical resampling and data-dependent
        # point selection (visibility >= 0.2); inverse depth adds its conditioning (test_oracle_vs_golden.py):
        # 2e-3; the photometric term and the total: 2e-4 (metric depth)
        loose = k in ("corres", "depth_cons", "colmap_depth") or c.get("depth_param") == "inverse"
        assert rep[k] < (2e-3 if loose else 2e-4), (name, k, got, ref)
    grads = {}
    for tag, m in [("nerf", net.nerf)] + ([("nerf_fine", net.nerf_fine)] if c["fine"] else []):
        for pname, p in m.named_parameters():
            if pname != "progress" and ("grad_%s.%s" % (tag, pname) in gold or "grad_%s.%s.sub" % (tag, pname) in gold):
                grads["grad_%s.%s" % (tag, pname)] = p.grad
    grads["grad_pose_embedding"] = pose_embedding.grad
    worst = check_grads(grads, gold, tol=gtol, norm=gnorm)
    print(name, engine, {k: "%.1e" % v for k, v in rep.items()}, "worst grad (%s) %.1e" % (gnorm, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("name", list(common.LOSS_CASES))
def test_full_sparf_step_vs_reference(name, engine):
    """photometric + corres + depth-cons (+ the DS-NeRF sparse-depth case) on our Graph / loss mirrors vs the reference's
    modules on its Graph (goldens: tests/golden/make_golden.py run_loss_case).  The depth-consistency term
    back-propagates through the float pixel locations of its second render (raygen d_pixels)."""
    import sparf_b200
    from sparf_b200.losses import define_loss
    from sparf_b200.poses_models import FirstTwoColunmnsPoseParameters
    from sparf_b200.renderer import Graph

    sparf_b200.set_engine(engine)
    dev = torch.device("cuda")
    gold, c, opt, data, ray_idx, sd, sd_fine, init_w2c = _loss_case_setup(name, dev)
    pose_net = FirstTwoColunmnsPoseParameters(opt, nbr_poses=c["B"], initial_poses_w2c=init_w2c, device=dev).to(dev)

    class PoseGraph(Graph):
        def __init__(self, opt, device, pose_net):
            super().__init__(opt, device)
            self.pose_net = pose_net

        def get_w2c_pose(self, opt, data_dict, mode=None):
            return self.pose_net.get_w2c_poses()

    net = PoseGraph(opt, dev, pose_net)
    net.nerf.load_state_dict(sd)
    if c["fine"]:
        net.nerf_fine.load_state_dict(sd_fine)
    net.to(dev).train()
    flow = common.FakeFlowNet(c["B"], c["H"], c["W"])
    np.random.seed(c["seed"])
    loss_module = define_loss(opt.loss_type, opt, net, _TrainData(data, c["B"]), dev, flow_net=flow)
    # gradient bound: the reference's own fp32 gradients sit ~3e-2 from the exact ones on these nets (conditioning,
    # test_tc_engine.py); inverse depth (samples out to t = 256, arguments ~1e5 rad in the top encoding bands, plus the
    # hard visibility / validity thresholds of the SPARF losses): the reference's fp32 gradients are themselves 7e-2 from
    # exact on the photometric-only case c4 (test_inverse_depth_conditioning_c4) and single entries behave like phase
    # noise (max-norm measured 0.2 .. 0.41, relative L2 0.2 (fp32 engine) .. 0.36 (tensor-core engine) per tensor): the gate is the relative L2 distance per tensor
    inv = c.get("depth_param") == "inverse"
    _run_and_check(name, engine, gold, c, opt, data, ray_idx, net, loss_module, pose_net.pose_embedding,
                   gtol=0.5 if inv else 6e-2, gnorm="l2" if inv else "max")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c7_sparf_losses", "c9_colmap_depth"])
def test_reference_trainer_graph_and_losses_on_our_renderer(name):
    """THE DROP-IN PROOF.  The reference's OWN `joint_pose_nerf_trainer.Graph` subclass (:710-749), its own pose model
    and its own `loss_factory.define_loss` modules run UNCHANGED with `source.models.renderer` resolved to
    `sparf_b200.renderer` (oracle/ref_loader.py shadow_renderer=True): every render they trigger goes through the CUDA
    kernels, and the losses / gradients must match the goldens the unmodified reference produced on its own renderer."""
    from oracle import ref_loader
    if not ref_loader.ref_root():
        pytest.skip("oracle/_ref not built (python oracle/build_ref.py in the build container)")
    import sparf_b200
    import sparf_b200.renderer as our_renderer

    sparf_b200.set_engine("auto")
    ref = ref_loader.load("trainer", shadow_renderer=True)
    try:
        assert issubclass(ref.joint.Graph, our_renderer.Graph) and ref.joint.Graph is not our_renderer.Graph
        dev = torch.device("cuda")
        gold, c, opt, data, ray_idx, sd, sd_fine, init_w2c = _loss_case_setup(name, dev)
        pose_net = ref.two_columns.FirstTwoColunmnsPoseParameters(opt, nbr_poses=c["B"], initial_poses_w2c=init_w2c, device=dev)
        net = ref.joint.Graph(opt, dev, pose_net)
        net.nerf.load_state_dict(sd)
        if c["fine"]:
            net.nerf_fine.load_state_dict(sd_fine)
        net.to(dev).train()
        flow = common.FakeFlowNet(c["B"], c["H"], c["W"])
        np.random.seed(c["seed"])
        loss_module = ref.loss_factory.define_loss(opt.loss_type, opt, net, _TrainData(data, c["B"]), dev, flow_net=flow)
        assert type(loss_module).__module__.startswith("source.training.core")
        _run_and_check(name, "reference trainer Graph + reference losses over sparf_b200 (auto engine)", gold, c, opt, data,
                       ray_idx, net, loss_module, pose_net.pose_embedding, gtol=6e-2)
    finally:
        ref_loader._purge()


def _sparf_problem(dev, stratified):
    import sparf_b200
    from sparf_b200.poses_models import FirstTwoColunmnsPoseParameters
    from sparf_b200.renderer import Graph
    sparf_b200.set_engine("auto")
    gold, c, opt, data, ray_idx, sd, sd_fine, init_w2c = _loss_case_setup("c7_sparf_losses", dev)
    opt.nerf.sample_stratified = stratified
    pose_net = FirstTwoColunmnsPoseParameters(opt, nbr_poses=c["B"], initial_poses_w2c=init_w2c, device=dev).to(dev)

    class PoseGraph(Graph):
        def get_w2c_pose(self, opt, data_dict, mode=None):
            return pose_net.get_w2c_poses()

    net = PoseGraph(opt, dev)
    net.nerf.load_state_dict(sd)
    net.nerf_fine.load_state_dict(sd_fine)
    net.to(dev).train()
    return c, opt, data, ray_idx, net, pose_net


def _sparf_step(c, opt, data, ray_idx, net, loss_module):
    data["iter"] = c["iteration"]
    out = net.render_image_at_specific_rays(opt, data, iter=c["iteration"], ray_idx=ray_idx, mode="train")
    data.poses_w2c = net.get_w2c_pose(opt, data, mode="train")
    loss_dict, stats, _ = loss_module.compute_loss(opt, data, out, iteration=c["iteration"], mode="train")
    loss_dict["all"].backward()
    data.pop("poses_w2c", None)
    return loss_dict


@pytest.mark.gpu
def test_device_side_losses_match_host_mode():
    """SURVEY 8f.2: the sync-free fixed-capacity mode of the correspondence / depth-consistency losses computes the same
    losses and gradients as the reference-faithful mode when both are given the same random choices (deterministic depth
    sampling so that padding rays do not shift any random stream)."""
    from sparf_b200.losses import define_loss
    dev = torch.device("cuda")
    rec = {"randint": [], "rand": [], "perm": []}
    results = {}
    for mode in ("host", "device"):
        c, opt, data, ray_idx, net, pose_net = _sparf_problem(dev, stratified=False)
        flow = common.FakeFlowNet(c["B"], c["H"], c["W"])
        loss_module = define_loss(opt.loss_type, opt, net, _TrainData(data, c["B"]), dev, flow_net=flow, device_side=(mode == "device"))
        corres_mod, dc_mod = loss_module.loss_modules[1], loss_module.loss_modules[2]
        if mode == "host":      # spy on the reference-order draws
            o_randint, o_rand, o_perm = np.random.randint, np.random.rand, torch.randperm
            np.random.seed(11)
            torch.manual_seed(11)

            def spy_randint(*a, **k):
                v = o_randint(*a, **k); rec["randint"].append(int(v)); return v

            def spy_rand(*a, **k):
                v = o_rand(*a, **k); rec["rand"].append(float(v)); return v

            def spy_perm(*a, **k):
                v = o_perm(*a, **k); rec["perm"].append(v.detach().cpu().clone()); return v

            np.random.randint, np.random.rand, torch.randperm = spy_randint, spy_rand, spy_perm
            try:
                losses = _sparf_step(c, opt, data, ray_idx, net, loss_module)
            finally:
                np.random.randint, np.random.rand, torch.randperm = o_randint, o_rand, o_perm
            assert len(rec["randint"]) == 2 and len(rec["rand"]) == 1 and len(rec["perm"]) == 2
        else:                   # replay them through the device-side hooks
            k_pair, id_self = rec["randint"]
            perm_corres, perm_px = rec["perm"]
            H, W = c["H"], c["W"]
            half = opt.nerf.rand_rays // 2
            i_map = corres_mod.filtered_flow_pairs[k_pair][0]
            valid_idx = corres_mod.mask_valid_corr[i_map, 0].reshape(-1).nonzero()[:, 0]
            keys = torch.full((H * W,), 1.0, device=dev)
            sel = valid_idx[perm_corres[:half].to(dev)]
            keys[sel] = torch.arange(len(sel), device=dev, dtype=torch.float32) / (2.0 * len(sel))
            corres_mod._rand_pair = lambda: torch.tensor([k_pair], device=dev)
            corres_mod._rand_keys = lambda n: keys
            from sparf_b200.sampling_strategies import sample_rays
            ys, xs = torch.meshgrid(torch.arange(H - 1), torch.arange(W - 1), indexing="ij")
            grid = torch.stack([xs.reshape(-1), ys.reshape(-1)], -1)
            px = grid[perm_px[: max(1024, opt.nerf.rand_rays)]].float().to(dev)
            dc_mod._rand_image = lambda B: torch.tensor([id_self], device=dev)
            dc_mod._rand_weight = lambda: torch.tensor(rec["rand"][0], device=dev, dtype=torch.float32)
            dc_mod._rand_pixels = lambda H_, W_, n: px
            losses = _sparf_step(c, opt, data, ray_idx, net, loss_module)
        torch.cuda.synchronize()
        grads = [p.grad.detach().clone() for p in list(net.nerf.parameters()) + list(net.nerf_fine.parameters()) if p.grad is not None]
        grads.append(pose_net.pose_embedding.grad.detach().clone())
        results[mode] = ({k: float(v) for k, v in losses.items() if torch.is_tensor(v) and v.dim() == 0}, grads)
    lh, gh = results["host"]
    ld, gd = results["device"]
    for k in ("render", "corres", "depth_cons", "all"):
        assert abs(lh[k] - ld[k]) <= 2e-5 * max(abs(lh[k]), 1e-6), (k, lh[k], ld[k])
    for a, b in zip(gh, gd):
        assert (a - b).abs().max().item() <= 2e-4 * max(a.abs().max().item(), 1e-12)
    print("device-side == host mode:", {k: "%.3e/%.3e" % (lh[k], ld[k]) for k in ("corres", "depth_cons")})


@pytest.mark.gpu
def test_sparf_step_is_sync_free_and_graph_capturable():
    """A full SPARF step (photometric + correspondence + depth-consistency: 6 render calls, gradients to both networks
    and the poses) in device-side mode performs NO host synchronisation (torch.cuda.set_sync_debug_mode('error')) and
    replays as ONE CUDA graph."""
    from sparf_b200.distributed import FlatGradients
    from sparf_b200.graphs import GraphedStep
    from sparf_b200.losses import define_loss
    dev = torch.device("cuda")
    c, opt, data, ray_idx, net, pose_net = _sparf_problem(dev, stratified=True)
    net.device_side_rng = True
    flow = common.FakeFlowNet(c["B"], c["H"], c["W"])
    loss_module = define_loss(opt.loss_type, opt, net, _TrainData(data, c["B"]), dev, flow_net=flow, device_side=True)
    fg = FlatGradients([net, pose_net])

    def step(idx):
        fg.zero_()
        return _sparf_step(c, opt, data, idx, net, loss_module)["all"].detach()

    step(ray_idx)                       # lazy initialisation (tables, workspaces, host caches) may synchronise
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        l1 = step(ray_idx)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert torch.isfinite(l1) and fg.flat.abs().sum() > 0
    graphed = GraphedStep(step, (ray_idx.clone(),), warmup=2)
    vals = []
    for _ in range(3):
        vals.append(float(graphed(ray_idx)))
        assert torch.isfinite(fg.flat).all() and fg.flat.abs().sum() > 0
    assert all(np.isfinite(v) for v in vals) and len(set(vals)) > 1     # fresh device-side random draws every replay
    print("SPARF step as one CUDA graph:", vals)
