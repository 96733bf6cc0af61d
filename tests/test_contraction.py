"""Contracted occupancy grids on the device (sparf_contracted_count / emit, occupancy.build_grid(contraction=...),
Graph.set_occupancy): the compaction equals the NumPy oracle (tests/contraction_oracle.py) byte for byte; a grid with
every cell occupied changes no bit of a render; a render with a random contracted grid, with or without early
termination, equals the dense render with σ and rgb zeroed at the samples the oracle skips; on an analytic
forward-facing inverse-depth scene the grid skips only empty samples, keeps the oracle's count and stays within the
bounds of what it skipped; and training, test-time optimisation, render_to_max and gradients ignore it."""
import os
import sys

import numpy as np
import pytest
import torch

import common
import contraction_oracle as C
import helpers as H
import occupancy_oracle as O
import termination_oracle as T
from test_occupancy import KEYS, _assert_same, _bits, _engine_or_skip, _np_bits

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

ALL_KEYS = KEYS + [k + "_fine" for k in KEYS]
f32 = np.float32


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


def _random_contracted_grid(res, p, seed, center=(0.0, 0.0, 0.0), radius=1.0):
    from sparf_b200.occupancy import CONTRACTED_RANGE, OccupancyGrid
    occ = np.random.default_rng(seed).random((res,) * 3) < p
    bits = torch.from_numpy(O.pack_bits(occ).view(np.int32).copy()).cuda()
    return OccupancyGrid(bits, res, CONTRACTED_RANGE, 0.01, contraction=(center, radius))


def _keep(g, o, d, t):
    """the oracle's kept mask of grid g (None: everything) on o, d [R,3], t [R,S] (device tensors)"""
    if g is None:
        return None
    args = (o.cpu().numpy(), d.cpu().numpy(), t.cpu().numpy())
    if g.contraction is None:
        return O.kept(_np_bits(g.bits), g.res, *g.range, *args)
    return C.kept(_np_bits(g.bits), g.res, *g.contraction, *args)


# ------------------------------------------------------------------------------------------------ kernels vs oracle
def _samples(rng, R, S, center, radius, res):
    """rays from inside and outside the linear region; t up to the inverse-depth maximum and past 1e8; some samples
    exactly on ||y||_inf = 1 and on cell planes of the linear region; some NaN / inf"""
    c = np.asarray(center, f32)
    o = (c + f32(radius) * rng.uniform(-3, 3, (R, 3))).astype(f32)
    d = rng.normal(size=(R, 3)).astype(f32)
    t = np.exp(rng.uniform(np.log(1e-3), np.log(3e8), (R, S))).astype(f32)
    t[:, 0] = np.where(rng.random(R) < 0.3, 0, t[:, 0])
    # on the edge of the linear region, or on a cell plane (u an integer), and staying there (d = 0)
    y = rng.uniform(-1, 1, (R, 3))
    ax = rng.integers(0, 3, R)
    y[np.arange(R), ax] = rng.choice([-1.0, 1.0], R)
    plane = rng.random(R) < 0.5
    y[plane] = (rng.integers(res // 4, 3 * res // 4 + 1, (plane.sum(), 3)) * 4.0 / res - 2)
    on = rng.random(R) < 0.3
    o[on] = (c + f32(radius) * y[on].astype(f32)).astype(f32)
    d[on & (rng.random(R) < 0.5)] = 0
    bad = rng.random((R, S))
    t[bad < 0.003] = np.nan
    t[(bad >= 0.003) & (bad < 0.006)] = np.inf
    t[(bad >= 0.006) & (bad < 0.009)] = 1e30
    d[rng.random(R) < 0.01, 0] = np.inf
    return o, d, t


@pytest.mark.parametrize("R,S", [(0, 5), (1, 1), (3, 700), (1000, 37), (4099, 64)])
def test_compaction_matches_oracle(R, S):
    from sparf_b200 import ops
    rng = np.random.default_rng(R * 17 + S)
    for res, center, radius in ((1, (0, 0, 0), 1.0), (8, (0.25, -1.5, 2.0), 1.33), (64, (0, 0, 0), 1.0)):
        o, d, t = _samples(rng, R, S, center, radius, res)
        og, dg, tg = _cuda(o, d, t)
        for p in (0.0, 0.4, 1.0):
            bits = O.pack_bits(rng.random((res,) * 3) < p)
            (bg,) = _cuda(bits.view(np.int32))
            windows = [(0, S, None)]
            if S > 1:
                windows += [(S // 3, S, (rng.random(R) < 0.6).astype(np.uint8)), (1, max(2, S // 2), None)]
            for k0, k1, alive in windows:
                ag = None if alive is None else _cuda(alive)[0]
                got = ops.contracted_compact(og, dg, tg, k0, k1, ag, bg, res, center, radius)
                want = C.compact(o, d, t, k0, k1, alive, (bits, res, center, radius))
                assert got[0].shape == want[0].shape, (res, p, k0, got[0].shape, want[0].shape)
                for g, w in zip(got, want):
                    g = g.cpu().numpy()
                    assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (res, p, k0)


def test_invalid_arguments_are_refused():
    from sparf_b200 import ops
    o, d = torch.zeros(2, 3, device="cuda"), torch.ones(2, 3, device="cuda")
    t = torch.ones(2, 4, device="cuda")
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    for center, radius in (((0, 0, 0), 0.0), ((0, 0, 0), -1.0), ((0, 0, 0), float("nan")), ((0, float("inf"), 0), 1.0)):
        with pytest.raises(RuntimeError, match="contracted_count"):
            ops.contracted_compact(o, d, t, 0, 4, None, bits, 2, center, radius)
    with pytest.raises(RuntimeError, match="contracted_count"):
        ops.contracted_compact(o, d, t, 2, 2, None, bits, 2, (0, 0, 0), 1.0)


# ------------------------------------------------------------------------------------------------ renders
def _inverse_scene(seed=5, H_=24, W_=32, identity=False):
    """c4's settings (inverse depth [1, 0], 128 samples, no fine network) with deterministic random weights"""
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=128, fine=False, depth_param="inverse", depth_range=(1, 0))
    net = Graph(opt, torch.device("cuda"))
    net.nerf.load_state_dict(common.det_weights(opt, seed, peaky=True))
    data = common.make_scene(21, 2, H_, W_, identity=identity)
    data.depth_range = torch.tensor([[1.0, 0.0]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].cuda()
    return net, opt, data


def _render(net, opt, data, mode="val"):
    Hh, Ww = data.image.shape[-2:]
    return net.render(opt, data.pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"),
                      depth_range=net._depth_range(opt, data), iter=10, mode=mode)


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("name", ["c10_val_full_image", "c11_eval_full_image", "inverse_c4_settings"])
def test_all_occupied_grid_renders_bit_identically(name, engine, engine_guard):
    """thres = 0: every cell is occupied, so the render must not change a bit"""
    import sparf_b200
    from sparf_b200 import occupancy
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    with torch.no_grad():
        if name.startswith("c1"):
            net, c, opt, data, *_ = H.build_graph(name)
            run = lambda: net.forward(opt, data, iter=10, mode=c["mode"])
        else:
            net, opt, data = _inverse_scene()
            run = lambda: _render(net, opt, data)
        dense = run()
        grids = [occupancy.build_grid(opt, m, res=16, thres=0.0, contraction=((0.1, -0.2, 0.3), 1.5))
                 for m in net.get_network_components()]
        assert all(g.occupied_fraction() == 1.0 and g.contraction is not None for g in grids)
        net.set_occupancy(*grids)
        sparse = run()
        for eps, window in ((1e-4, 16),):        # and with termination on top: the termination render
            net.set_early_termination(eps, window)
            term_grid = run()
            net.set_occupancy(None)
            term = run()
            net.set_early_termination(None)
    keys = [k for k in dense if torch.is_tensor(dense[k]) and dense[k].is_floating_point()]
    assert "rgb" in keys
    _assert_same(sparse, dense, keys)
    _assert_same(term_grid, term, keys)


def _masked_reference(net, opt, data, mode, eps, window, grids):
    """the dense render assembled from ops calls, with σ = rgb = 0 at the samples the oracles skip (eps 0: no
    termination)"""
    from sparf_b200 import ops
    Hh, Ww = data.image.shape[-2:]
    center, ray = ops.raygen(data.pose, data.intr, Ww, ray_idx=torch.arange(Hh * Ww, device="cuda"))
    B, N = center.shape[:2]
    o, d = center.reshape(-1, 3), ray.reshape(-1, 3)
    depth_range = net._depth_range(opt, data)
    white = bool(opt.nerf.setbg_opaque or opt.mask_img)

    def masked(nerf, g, t):
        sigma, rgb = ops.mlp_forward(nerf._spec(), o, d, t, nerf.kernel_params(), progress=nerf.progress)
        ev = torch.from_numpy(T.evaluated(sigma.cpu().numpy(), t.cpu().numpy(), d.cpu().numpy(), eps, window,
                                          _keep(g, o, d, t))).cuda()
        sigma = torch.where(ev, sigma, torch.zeros_like(sigma))
        rgb = torch.where(ev[..., None], rgb, torch.zeros_like(rgb))
        rgb_map, depth, opacity, weights, depth_var, rgb_var, all_cum = ops.composite(sigma, rgb, t, d, white)
        return dict(rgb=rgb_map, depth=depth, opacity=opacity, weights=weights, depth_var=depth_var, rgb_var=rgb_var,
                    all_cumulated=all_cum, density_samples=sigma, rgb_samples=rgb, t=t)

    t = net.sample_depth(opt, B, num_rays=N, n_samples=opt.nerf.sample_intvs, H=Hh, W=Ww, depth_range=depth_range,
                         mode=mode).reshape(B * N, -1)
    out = masked(net.nerf, grids[0], t)
    if opt.nerf.fine_sampling:
        t_all = net._resample_and_merge(opt, out["weights"].view(B, N, -1), t.view(B, N, -1), depth_range, True)
        out.update({k + "_fine": v for k, v in masked(net.nerf_fine, grids[1], t_all.reshape(B * N, -1)).items()})
    return out


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("name,fine_grid", [("c10_val_full_image", True), ("c10_val_full_image", False),
                                            ("inverse_c4_settings", False), ("inverse_wall", False)])
def test_random_grid_render_equals_masked_dense_reference(name, fine_grid, engine, engine_guard):
    """without termination, and with it at several (eps, window); a contracted fine grid or none, and a box fine grid
    under the contracted coarse grid"""
    import sparf_b200
    from test_occupancy import _random_grid
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    if name.startswith("c1"):
        net, c, opt, data, *_ = H.build_graph(name)
        mode = c["mode"]
    else:
        net, opt, data = _inverse_scene() if name == "inverse_c4_settings" else _wall_scene()
        mode = "val"
    fine = opt.nerf.fine_sampling
    g_fine = _random_contracted_grid(12, 0.6, 2, (0.0, 0.5, 0.0), 2.0) if fine_grid else None
    grids = (_random_contracted_grid(16, 0.5, 1, (0.2, 0.0, -0.3), 1.2), g_fine)
    keys = ALL_KEYS if fine else KEYS
    skipped = []
    for eps, window in ((None, None), (1e-4, 16), (0.3, 1), (0.9, 5)):
        net.set_occupancy(*grids)
        net.set_early_termination(*((eps, window) if eps is not None else (None,)))
        with torch.no_grad():
            out = _render(net, opt, data, mode)
            ref = _masked_reference(net, opt, data, mode, eps or 0.0, window or opt.nerf.sample_intvs, grids)
        _assert_same(out, ref, keys)
        skipped.append(round((out["density_samples"] == 0).float().mean().item(), 3))
    net.set_early_termination(None)
    print("%s fine grid %s: skipped fraction (coarse) per (eps, window): %s" % (name, fine_grid, skipped))
    assert 0.05 < skipped[0] < 0.95
    if name == "inverse_wall":
        assert max(skipped) > skipped[0] + 0.1                 # the wall does terminate rays
    if fine:                                       # a box fine grid under a contracted coarse grid
        net.set_occupancy(grids[0], _random_grid(12, 0.3, 3))
        with torch.no_grad():
            _assert_same(_render(net, opt, data, mode),
                         _masked_reference(net, opt, data, mode, 0.0, opt.nerf.sample_intvs,
                                           (grids[0], net._occupancy[1])), keys)


def _wall_scene():
    """forward-facing and inverse-depth: 2 identity cameras with LLFF's field of view, a wall σ = softplus(400 (z - 3))
    (wall_weights of tools/time_termination.py), 128 samples over disparity [1, 0], no fine network"""
    from sparf_b200.renderer import Graph
    from time_termination import wall_weights
    opt = common.make_opt(S=128, fine=False, depth_param="inverse", depth_range=(1, 0))
    net = Graph(opt, torch.device("cuda"))
    net.nerf.load_state_dict(wall_weights(opt, (0.0, 0.0, -1.0), -3.0, 400.0))
    data = common.make_scene(21, 2, 30, 40, focal=32.0, identity=True)
    data.depth_range = torch.tensor([[1.0, 0.0]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].cuda()
    return net, opt, data


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_analytic_inverse_depth_wall(engine, engine_guard):
    """every skipped sample's dense σ is below thres; the kept count is the oracle's on the grid's bits; rgb, opacity
    and depth differ from the dense render by at most what the skipped samples could absorb; and termination on top
    of the grid stays within termination's bounds of the grid render"""
    import sparf_b200
    from sparf_b200 import occupancy, ops
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    net, opt, data = _wall_scene()
    thres, res, contraction = 0.01, 128, ((0.0, 0.0, 0.0), 1.33)
    with torch.no_grad():
        dense = _render(net, opt, data)
        grid = occupancy.build_grid(opt, net.nerf, res=res, thres=thres, contraction=contraction)
        net.set_occupancy(grid)
        sparse = _render(net, opt, data)
    o, d = dense["origins"].reshape(-1, 3), dense["viewdirs"].reshape(-1, 3)
    t = dense["t"].reshape(o.shape[0], -1)
    keep = torch.from_numpy(_keep(grid, o, d, t)).cuda()
    idx = ops.contracted_compact(o, d, t, 0, t.shape[1], None, grid.bits, res, *contraction)[0]
    assert idx.numel() == keep.sum().item()
    frac = keep.float().mean().item()
    print("%s: occupied cells %.3f, kept samples %.4f" % (engine, grid.occupied_fraction(), frac))
    assert 0.3 < frac < 0.45
    sig_d = dense["density_samples"].reshape(keep.shape)
    assert (sig_d[~keep] < thres).all()
    assert sig_d.max().item() > 10 and dense["opacity"].min().item() > 0.99
    sig_s = sparse["density_samples"].reshape(keep.shape)
    assert torch.equal(_bits(sig_s[keep]), _bits(sig_d[keep])) and (sig_s[~keep] == 0).all()
    gap = torch.cat([t[:, 1:] - t[:, :-1], torch.full_like(t[:, :1], 1e10)], 1) * d.norm(dim=-1, keepdim=True)
    eps = torch.where(keep, torch.zeros_like(sig_d), sig_d.double() * gap.double()).sum(1)
    bound = (1 - torch.exp(-eps)).float()
    tol = 2e-6
    diff = lambda a, b, k: (a[k] - b[k]).reshape(o.shape[0], -1).abs().amax(1)
    dr, do, dd = diff(sparse, dense, "rgb"), diff(sparse, dense, "opacity"), diff(sparse, dense, "depth")
    assert (dr <= bound + tol).all(), (dr - bound).max().item()
    assert (do <= bound + tol).all(), (do - bound).max().item()
    assert (dd <= (bound + tol) * t.amax(1)).all(), (dd - bound * t.amax(1)).max().item()
    # grid + termination against the grid render: termination's bounds on the same samples
    term_eps = 1e-4
    with torch.no_grad():
        net.set_early_termination(term_eps, 16)
        both = _render(net, opt, data)
        net.set_early_termination(None)
    assert torch.equal(both["t"], sparse["t"])
    both_frac = (both["density_samples"] != 0).float().mean().item()
    print("%s: grid + termination evaluates %.4f" % (engine, both_frac))
    assert both_frac < 0.2
    tr, to, td = diff(both, sparse, "rgb"), diff(both, sparse, "opacity"), diff(both, sparse, "depth")
    assert (to < term_eps + tol).all() and (tr < term_eps + tol).all(), (to.max(), tr.max())
    assert (td < (term_eps + tol) * t.amax(1)).all()
    print("max |d rgb| %.3g, |d opacity| %.3g, |d depth| %.3g (grid); %.3g %.3g %.3g (termination on top)" % (
        dr.max(), do.max(), dd.max(), tr.max(), to.max(), td.max()))


# ------------------------------------------------------------------------------------------------ untouched paths
def test_grid_is_ignored_outside_inference(engine_guard):
    """contracted grids (and termination) attached, but mode train / test-optim, gradients on or render_to_max:
    bit-identical to the same call without them"""
    net, c, opt, data, *_ = H.build_graph("c10_val_full_image")
    Hh, Ww = data.image.shape[-2:]
    kw = dict(H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"), iter=10)
    grids = (_random_contracted_grid(16, 0.3, 5), _random_contracted_grid(16, 0.3, 6, (0, 0, 1.0), 2.0))
    depth_range = net._depth_range(opt, data)

    def run(mode, grad, attach, term=False, to_max=False):
        net.set_occupancy(*(grids if attach else (None, None)))
        net.set_early_termination(*((0.999999, 4) if term else (None,)))
        torch.manual_seed(1234)
        with torch.set_grad_enabled(grad):
            if to_max:
                out = net.render_to_max(opt, data.pose, mode=mode, depth_min=1.0,
                                        depth_max=torch.full((len(data.pose), Hh * Ww), 3.0, device="cuda"), **kw)
            else:
                out = net.render(opt, data.pose, mode=mode, depth_range=depth_range, **kw)
        return {k: v.detach() for k, v in out.items() if torch.is_tensor(v)}

    for term in (False, True):
        for mode, grad in (("train", False), ("train", True), ("test-optim", False), ("val", True)):
            _assert_same(run(mode, grad, True, term), run(mode, grad, False), ALL_KEYS)
        _assert_same(run("val", False, True, term, to_max=True), run("val", False, False, to_max=True), ALL_KEYS)
    sparse = run("val", False, True)                # and the grids do apply here: the same call differs
    assert not torch.equal(sparse["density_samples"], run("val", False, False)["density_samples"])
    net.set_occupancy(None)
