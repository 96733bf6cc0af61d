"""Parity of the CUDA path (through the C ABI) against the reference's golden vectors and the oracle.

Tolerances (stated once, used below):
  * STAGE tests feed the reference's own intermediate tensors (origins / viewdirs / t from the golden)
    to one kernel stage, so the only differences are fp32 accumulation order inside the kernels:
    outputs <= 2e-5 rel (max|a-b| / max|b|), bit-exact for the sampling arithmetic.
  * END-TO-END tests run Graph exactly as make_golden.py ran the reference.  The 2^9*pi encoding band
    amplifies the 1-ulp differences of our per-pixel ray generation ~1e3x (the reference's own fp32
    result sits 1e-4..1e-3 from exact arithmetic on these nets, test_oracle_vs_golden.py), so the
    north-star bound applies: rgb / depth / opacity <= 1e-4 rel for the coarse pass; quantities behind
    the resampling (t_fine, *_fine) and gradients get the looser bounds written at each assert.
"""
import numpy as np
import pytest
import torch

import common
from helpers import check_grads, load_golden, rel_err, replay_graph

pytestmark = pytest.mark.gpu

ENGINES = ["simt_fp32", "tc_3x"]   # fp32 CUDA-core engine and the wgmma split-precision engine
# stage tests need the reference's intermediate tensors (origins / viewdirs / t), which render_by_slices drops
STAGE_CASES = [n for n in common.CASES if not common.CASES[n].get("full_image")]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


# ------------------------------------------------------------------------------------------------ stages
@pytest.mark.parametrize("name", STAGE_CASES)
def test_raygen_matches_reference(name):
    from sparf_b200 import ops
    from oracle import sparf_oracle as O
    c, opt, data, ray_idx, pixels, sd, sd_fine, init_w2c, depth_max = common.case_inputs(name)
    gold = load_golden(name)
    if init_w2c is not None:
        pose = O.d9_to_pose(O.pose_to_d9(init_w2c))
    elif c.get("test_optim"):
        pose = O.compose_pair(O.se3_to_SE3(c["se3_refine"]), data.pose)
        ray_idx = torch.from_numpy(gold["randperm_0"])[: opt.nerf.rand_rays // c["B"]]
    else:
        pose = data.pose
    if pixels is not None:
        o, d = ops.raygen(pose.cuda(), data.intr.cuda(), c["W"], pixels=pixels.cuda())
    else:
        o, d = ops.raygen(pose.cuda(), data.intr.cuda(), c["W"], ray_idx=ray_idx.cuda())
    assert rel_err(o, gold["out_origins"]) < 1e-6
    assert rel_err(d, gold["out_viewdirs"]) < 1e-6


@pytest.mark.parametrize("name", STAGE_CASES)
def test_sample_depth_bit_exact(name):
    from sparf_b200.renderer import Graph
    from helpers import build_graph, RandomReplayer
    gold = load_golden(name)
    net, c, opt, data, ray_idx, pixels, depth_max = build_graph(name)
    B, n, S = c["B"], gold["out_t"].shape[1], c["S"]
    with RandomReplayer({k: v for k, v in gold.items() if not k.startswith("randperm_")}):
        if c.get("to_max"):
            t = net.sample_depth_diff_max_range_per_ray(opt, B, S, c["H"], c["W"], depth_min=data.depth_range[0][0],
                                                        depth_max=depth_max, num_rays=n)
        else:
            t = net.sample_depth(opt, B, S, c["H"], c["W"], depth_range=Graph._depth_range(opt, data), num_rays=n,
                                 mode=c["mode"])
    ref = gold["out_t"]
    assert np.array_equal(t.cpu().numpy().reshape(ref.shape), ref), np.abs(t.cpu().numpy().reshape(ref.shape) - ref).max()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", STAGE_CASES)
def test_mlp_and_composite_stage(name, engine):
    """Reference rays + reference samples in -> per-sample and composited outputs out."""
    import sparf_b200
    from helpers import build_graph
    sparf_b200.set_engine(engine)
    gold = load_golden(name)
    net, c, opt, data, ray_idx, pixels, depth_max = build_graph(name)
    for suf, nerf in (("", net.nerf),) + ((("_fine", net.nerf_fine),) if c["fine"] else ()):
        center, ray = _dev(gold["out_origins"]), _dev(gold["out_viewdirs"])
        t = _dev(gold["out_t" + suf])
        noise_key = "randn_0" if suf == "" else "randn_1"
        pred = None
        if noise_key in gold:
            import helpers
            with helpers.RandomReplayer({noise_key: gold[noise_key]}):
                pred = nerf.forward_samples(opt, center, ray, t, mode=c["mode"])
        else:
            pred = nerf.forward_samples(opt, center, ray, t, mode=c["mode"])
        pred = nerf.composite(opt, ray, pred, t)
        # fp32 engine: the reference's op order, 2e-5; tensor-core 3-pass fp16 split: fp32-level products in a different
        # summation order, measured <= 3e-5 against the fp32 engine (tests/test_tc_engine.py)
        tol = 2e-5 if engine == "simt_fp32" else 3e-5
        if common.CASES[name].get("depth_param", "metric") == "inverse":
            # inverse depth reaches t ~ 256: the top encoding bands see arguments ~1e5 where one fp32 ulp
            # is ~1e-2 rad, so ANY difference in accumulation order is amplified to ~1e-3 downstream
            tol = 2e-3
        for k in ("density_samples", "rgb_samples", "rgb", "depth", "opacity", "weights", "depth_var", "all_cumulated"):
            ref = gold["out_" + k + suf]
            got = pred[k].detach().cpu().numpy().reshape(ref.shape)
            # depth_var = sum w (t - depth)^2 is a small difference of O(depth^2) terms: fp32-conditioned
            # at ~1e-3 when the density is peaked (visualisation-only output, base.py:644-648)
            bound = 2e-3 if k == "depth_var" else tol
            assert rel_err(got, ref) < bound, (k + suf, rel_err(got, ref))
        ref = gold["out_rgb_var" + suf]
        assert np.abs(pred["rgb_var"].detach().cpu().numpy().reshape(ref.shape) - ref).max() < max(1e-5, tol)


@pytest.mark.parametrize("name", ["c2_hier", "c5_hier_pose_bg"])
def test_sample_pdf_matches_reference(name):
    """Reference coarse weights in -> fine samples + merged sorted samples out."""
    from helpers import build_graph
    from sparf_b200.renderer import Graph
    gold = load_golden(name)
    net, c, opt, data, ray_idx, pixels, depth_max = build_graph(name)
    w = _dev(gold["out_weights"][..., 0])
    t_c = _dev(gold["out_t"])
    t_all = net._resample_and_merge(opt, w, t_c[..., 0], Graph._depth_range(opt, data), det=True)
    ref = gold["out_t_fine"]
    # cdf accumulation order differs (warp scan vs sequential): ~1e-6 relative on the sample positions
    assert rel_err(t_all.cpu().numpy().reshape(ref.shape), ref) < 5e-6
    t_f = net.sample_depth_from_pdf(opt, w, c["S"], c["S_fine"], Graph._depth_range(opt, data), det=True)
    merged = torch.cat([t_c, t_f], dim=2).sort(dim=2).values
    assert torch.equal(merged, t_all)


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(common.CASES))
def test_graph_end_to_end_vs_reference(name, engine):
    out, loss, grads, gold = replay_graph(name, engine)
    report = {}
    for k in ("rgb", "depth", "opacity"):
        ref = gold["out_" + k]
        e = rel_err(out[k].detach().cpu().numpy().reshape(ref.shape), ref)
        report[k] = e
        # north-star bound; inverse-depth rays reach |x| ~ 1e2 where the top band is pure rounding noise
        bound = 1e-4 if common.CASES[name].get("depth_param", "metric") == "metric" else 2e-3
        assert e < bound, (name, k, e)
    for k in ("rgb_fine", "depth_fine", "opacity_fine"):
        if "out_" + k in gold:
            ref = gold["out_" + k]
            e = rel_err(out[k].detach().cpu().numpy().reshape(ref.shape), ref)
            report[k] = e
            assert e < 1e-3, (name, k, e)   # sits behind the (discontinuous) inverse-CDF resampling
    if loss is None:     # forward-only cases (val / eval full image through render_by_slices)
        for k in ("depth_var", "all_cumulated", "depth_var_fine", "all_cumulated_fine"):
            if "out_" + k in gold:
                ref = gold["out_" + k]
                assert rel_err(out[k].detach().cpu().numpy().reshape(ref.shape), ref) < 2e-3, (name, k)
        print(name, engine, {k: "%.1e" % v for k, v in report.items()})
        return
    ltol = 2e-4 if common.CASES[name].get("depth_param", "metric") == "metric" else 2e-3
    assert abs(loss.item() - float(gold["loss"])) < ltol * max(1.0, abs(float(gold["loss"])))
    # gradients: fp32 accumulation over ~1e4 rows in a different order + the input-side noise above
    # The reference's own fp32 gradient sits ~3e-2 from the exact (fp64) gradient on these random nets
    # (tests/test_tc_engine.py::test_tc_backward_matches_simt measures both engines against fp64): the SIMT
    # engine shares the reference's op order and lands closer to IT; the tensor-core engine is equally close to
    # the truth but not to the reference's particular rounding.
    # (c8: with the Charbonnier / distortion terms the reference's fp32 gradient is itself 1.2e-1 from the fp64 one)
    # (c13: near plane 0.1, nine views: the fine network's gradients sit behind resampled positions close to the cameras
    #  and move ~1e-2 with the last bit of the coarse weights)
    gtol = 0.25 if "inverse" in name else (6e-2 if (engine != "simt_fp32" or common.CASES[name].get("regularisers")) else
                                           (3e-2 if name.startswith("c13") else 5e-3))
    worst = check_grads(grads, gold, tol=gtol)
    print(name, engine, {k: "%.1e" % v for k, v in report.items()}, "worst grad %.1e" % worst)


def _error_vs_fp64(name, engine, out_factor, grad_factor, grad_floor):
    """Our distance from the exact (fp64-oracle) result of a golden case, gated against the REFERENCE's own fp32 distance
    from it (the golden holds the reference's outputs and gradients): outputs max-norm, gradient tensors relative L2."""
    from helpers import replay_oracle
    exact_out, _, exact_grads, gold = replay_oracle(name, torch.float64)
    out, loss, grads, _ = replay_graph(name, engine)
    rep = {}
    for k in ("rgb", "depth", "opacity"):
        ex = exact_out[k].detach().numpy()
        ours = rel_err(out[k].detach().cpu().numpy().reshape(ex.shape), ex)
        ref = rel_err(gold["out_" + k].reshape(ex.shape), ex)
        rep[k] = (ours, ref)
        assert ours <= max(out_factor * ref, 1e-4), (name, k, ours, ref)
    for k, g in grads.items():
        ex = exact_grads[k].detach().numpy()
        mine = g.detach().cpu().double().numpy()
        if k in gold:
            ref_g = gold[k]
        else:
            ref_g, ex, mine = gold[k + ".sub"], common.subsample(ex), common.subsample(mine)
        scale = max(np.sqrt((ex ** 2).sum()), 1e-30)
        ours, ref = np.sqrt(((mine - ex) ** 2).sum()) / scale, np.sqrt(((ref_g - ex) ** 2).sum()) / scale
        rep[k] = (ours, ref)
        assert ours <= max(grad_factor * ref, grad_floor), (name, k, ours, ref)
    worst = max(rep.items(), key=lambda kv: kv[1][0] / max(kv[1][1], 1e-12))
    print(name, engine, "worst ours / reference-fp32 distance from fp64: %s %.1e / %.1e" % (worst[0], worst[1][0], worst[1][1]))


@pytest.mark.parametrize("engine", ENGINES)
def test_c4_inverse_depth_error_vs_fp64(engine):
    """Inverse-depth case (BASELINE config 4): our error is gated against the REFERENCE's OWN fp32 error on the same
    inputs, both measured from the exact (fp64) evaluation (tests/test_oracle_vs_golden.py::
    test_inverse_depth_conditioning_c4 explains the conditioning): outputs no further from the truth than 1.5x the
    reference is (floor: north_star's 1e-4); gradient tensors: 6x in relative L2 (floor 1e-3; measured 0.5x .. 4.4x --
    single entries behave like phase noise: our rays differ from the reference's in the last bit, and at t ~ 256 that
    alone moves an entry by ~1e-2)."""
    _error_vs_fp64("c4_inverse_pixels", engine, 1.5, 6.0, 1e-3)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["c1_coarse", "c3_barf_pose"])
def test_coarse_cases_error_vs_fp64(name, engine):
    """The same yardstick for the metric-depth goldens without a resampling step (c1; c3 with pose gradients, BARF mask
    and sigma noise): outputs within 2x and gradient tensors within 3x (relative L2) of the reference's own fp32 distance
    from the exact result, floors 1e-4 / 1e-3 -- the tight gate of the tensor-core engine's gradients, which the comparison
    with the golden alone (6e-2, the reference's own noise) cannot give.  (Hierarchical cases are excluded: a last-bit
    change of a coarse weight moves a resampled position discontinuously, in exact arithmetic as well; the headline-shape
    test tests/test_headline_parity.py covers the full-size batch the same way.)  The fp32 CUDA-core engine accumulates the
    per-ray gradients of a pose with fp32 atomics (measured 2.0e-3 on the pose embedding of c3): floor 3e-3 there."""
    _error_vs_fp64(name, engine, 2.0, 3.0, 3e-3 if engine == "simt_fp32" else 1e-3)


@pytest.mark.parametrize("engine", ENGINES)
def test_headline_shape_vs_oracle(engine):
    """1023 rays x 128 samples (BASELINE config 2, coarse): CUDA vs the fp32 oracle on identical rays."""
    import sparf_b200
    from sparf_b200 import ops
    from oracle import sparf_oracle as O
    sparf_b200.set_engine(engine)
    opt = common.make_opt(S=128)
    sd = common.det_weights(opt, 11, peaky=True, sigma_bias=-4.0)
    data = common.make_scene(11, 3, 300, 400)
    rng = np.random.default_rng(5)
    ray_idx = torch.from_numpy(rng.permutation(300 * 400)[:341].astype(np.int64))
    center, ray = O.rays_from_ray_idx(data.pose, data.intr, 300, 400, ray_idx)
    t = O.sample_depth(3, 341, 128, torch.tensor([1.2, 5.2]))
    params = {k: v.clone().requires_grad_(k != "progress") for k, v in sd.items()}
    with torch.no_grad():
        pts = center[:, :, None] + ray[:, :, None] * t[..., None]
        dens, rgb_s = O.mlp_forward(params, pts, ray)
        ref = O.composite(ray, dens, rgb_s, t)
    spec = ops.MLPSpec()
    plist = [sd[k].cuda() for k in sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], [])
             + ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]]
    R = 3 * 341
    sigma, rgb = ops.mlp_forward(spec, center.reshape(R, 3).cuda(), ray.reshape(R, 3).cuda(), t.reshape(R, 128).cuda(), plist)
    rgb_map, depth, opacity, weights, *_ = ops.composite(sigma, rgb, t.reshape(R, 128).cuda(), ray.reshape(R, 3).cuda())
    assert rel_err(rgb_map.cpu(), ref["rgb"].reshape(R, 3)) < 1e-4
    assert rel_err(depth.cpu(), ref["depth"].reshape(R)) < 1e-4
    assert rel_err(opacity.cpu(), ref["opacity"].reshape(R)) < 1e-4


def test_composite_properties_full_size():
    """Size-independent properties at the full batch (4096 rays x 384 samples): weights >= 0, opacity =
    sum(weights) <= 1 (+eps), depth within [t_min, t_max], all_cumulated = 1 - sum of all but the last two."""
    from sparf_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    R, S = 4096, 384
    sigma = torch.rand(R, S, device="cuda", generator=g) * 3
    rgb = torch.rand(R, S, 3, device="cuda", generator=g)
    t = torch.sort(torch.rand(R, S, device="cuda", generator=g) * 4 + 1, dim=1).values
    dirs = torch.randn(R, 3, device="cuda", generator=g)
    rgb_map, depth, opacity, weights, depth_var, rgb_var, all_cum = ops.composite(sigma, rgb, t, dirs)
    assert (weights >= 0).all()
    assert torch.allclose(opacity, weights.sum(1), atol=1e-5)
    assert (opacity <= 1 + 1e-5).all()
    assert ((depth >= t[:, 0] * opacity - 1e-4) & (depth <= t[:, -1] + 1e-4)).all()
    assert torch.allclose(all_cum, 1 - weights[:, :-2].sum(1), atol=2e-5)
    assert (rgb_map >= -1e-6).all() and (rgb_map <= 1 + 1e-5).all()


def test_gradcheck_composite_fp32_vs_autograd():
    """Composite backward kernel vs torch autograd over the oracle formula (same inputs, on the GPU)."""
    from sparf_b200 import ops
    from oracle import sparf_oracle as O
    g = torch.Generator(device="cuda").manual_seed(1)
    R, S = 257, 96
    sigma = (torch.rand(R, S, device="cuda", generator=g) * 2).requires_grad_(True)
    rgb = torch.rand(R, S, 3, device="cuda", generator=g).requires_grad_(True)
    t = torch.sort(torch.rand(R, S, device="cuda", generator=g) * 4 + 1, dim=1).values
    dirs = torch.randn(R, 3, device="cuda", generator=g).requires_grad_(True)
    wr = torch.randn(R, 3, device="cuda", generator=g)
    wd = torch.randn(R, device="cuda", generator=g)
    ww = torch.randn(R, S, device="cuda", generator=g) * 0.1

    def loss_of(rgb_map, depth, opacity, weights):
        return (rgb_map * wr).sum() + (depth * wd).sum() + 0.3 * (opacity * wd).sum() + (weights * ww).sum()

    a = ops.composite(sigma, rgb, t, dirs, True)
    loss_of(a[0], a[1], a[2], a[3]).backward()
    got = [sigma.grad.clone(), rgb.grad.clone(), dirs.grad.clone()]
    sigma.grad = rgb.grad = dirs.grad = None
    ref = O.composite(dirs[None], sigma[None], rgb[None], t[None], white_bg=True)
    loss_of(ref["rgb"][0], ref["depth"][0, :, 0], ref["opacity"][0, :, 0], ref["weights"][0, :, :, 0]).backward()
    for gk, rk in zip(got, [sigma.grad, rgb.grad, dirs.grad]):
        assert rel_err(gk, rk) < 2e-5


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("L", [1, 4, 10, 16])
@pytest.mark.parametrize("c2f,progress", [(None, 0.3), ((0.1, 0.5), 0.3), ((0.0, 0.5), 0.25)])
def test_standalone_posenc_matches_oracle(c2f, progress, L, C):
    """FrequencyEmbedder.__call__ / NeRF.positional_encoding as tensor ops (sparf_posenc_forward / _backward) vs the
    oracle's restatement of frequency_nerf.py:47-69, 248-257, for L bands of C channels (n * 2CL = 370CL values: never a
    multiple of the 256-thread block).  c2f (0, 0.5) at progress 0.25 puts alpha = L/2, so for L >= 4 one band sits
    exactly at alpha - j = 1 (weight 1) and the next at alpha - j = 0 (weight 0).
    Yardstick (as in _error_vs_fp64): distance from the fp64 oracle within 4x the fp32 oracle's own distance.  Both
    round the argument x * 2^j pi to fp32 alike, which dominates at the top band (~2^L pi |x| rad); floors: 8 unit
    round-offs (2^-24) for the values, 64 of the largest entry for the input gradient (a sum over 2L terms)."""
    from oracle import sparf_oracle as O
    from sparf_b200.frequency_nerf import FrequencyEmbedder, NeRF
    ulp = 2.0 ** -24
    opt = common.make_opt(barf_c2f=c2f)
    nerf = NeRF(opt).cuda()
    nerf.progress.data.fill_(progress)
    g = torch.Generator(device="cuda").manual_seed(4)
    x = ((torch.rand(5, 37, C, device="cuda", generator=g) - 0.5) * 4).requires_grad_(True)
    enc = nerf.positional_encoding(opt, x, FrequencyEmbedder(opt), L)
    w = torch.randn(enc.shape, device="cuda", generator=g)
    (enc * w).sum().backward()
    refs = []
    for dt in (torch.float64, torch.float32):
        mask = O.c2f_weights(L, progress, c2f, device="cuda", dtype=dt)
        xr = x.detach().to(dt).requires_grad_(True)
        ref = O.posenc(xr, L, mask)
        (ref * w.to(dt)).sum().backward()
        refs.append((ref, xr.grad))
    (ref64, gx64), (ref32, gx32) = refs
    assert enc.shape == ref64.shape == (5, 37, 2 * C * L)
    e_k, e_o = (enc.double() - ref64).abs().max().item(), (ref32.double() - ref64).abs().max().item()
    assert e_k <= 4 * e_o + 8 * ulp, (e_k, e_o)
    if c2f is not None and progress == 0.25 and L >= 4:
        j = L // 2
        assert (mask[j - 1] == 1).item() and (mask[j] == 0).item()
        assert (enc[..., j] == 0).all() and (enc[..., L + j] == 0).all()
    g_k, g_o = rel_err(x.grad, gx64), rel_err(gx32, gx64)
    assert g_k <= 4 * g_o + 64 * ulp, (g_k, g_o)
    plain = FrequencyEmbedder(opt)(opt, x.detach(), 4)
    assert (plain.double() - O.posenc(x.detach().double(), 4, None)).abs().max().item() < 1e-5
