"""Early ray termination on the device (sparf_termination_count / emit / update, sparf_b200.termination,
Graph.set_early_termination): the kernels equal the NumPy oracle (tests/termination_oracle.py) byte for byte; a
termination render equals the dense render with σ and rgb zeroed at the samples the oracle skips, bit for bit; eps = 0
changes nothing; on an analytic scene the coarse composite is within the documented bounds; and every call it must not
touch (training, test-time optimisation, render_to_max, gradients, a detached setting) is bit-identical."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import common
import helpers as H
import occupancy_oracle as O
import termination_oracle as T
from test_occupancy import KEYS, _assert_same, _engine_or_skip, _np_bits, _random_grid, _samples

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

ALL_KEYS = KEYS + [k + "_fine" for k in KEYS]


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


# ------------------------------------------------------------------------------------------------ kernels vs oracle
@pytest.mark.parametrize("R,S", [(0, 5), (1, 1), (3, 70), (1000, 37), (4099, 64)])
def test_update_matches_oracle(R, S):
    from sparf_b200 import ops
    rng = np.random.default_rng(R * 7 + S)
    sigma = rng.exponential(1.0, (R, S)).astype(np.float32) * rng.choice([0, 0.1, 1, 30], (R, 1)).astype(np.float32)
    bad = rng.random((R, S))
    sigma[bad < 0.01] = np.nan
    sigma[(bad >= 0.01) & (bad < 0.02)] = np.inf
    t = np.sort(rng.uniform(0, 4, (R, S)), 1).astype(np.float32)
    t[rng.random((R, S)) < 0.005] = np.inf
    d = rng.normal(size=(R, 3)).astype(np.float32)
    d[rng.random(R) < 0.1] = 0                                   # zero-length directions
    for eps in (0.0, 1e-4, 0.3):
        for window in (1, 7, S):
            tau = rng.uniform(0, 3, R).astype(np.float32)
            alive = (rng.random(R) < 0.7).astype(np.uint8)
            tau_g, alive_g = _cuda(tau, alive)
            sig_g, t_g, d_g = _cuda(sigma, t, d)
            for k0 in range(0, S, window):                        # every window, the last (gap 1e10) included
                k1 = min(k0 + window, S)
                ops.termination_update(sig_g, t_g, d_g, k0, k1, float(T.tau_max(eps)), tau_g, alive_g)
                tau, alive = T.update(sigma, t, d, k0, k1, T.tau_max(eps), tau, alive)
                got = tau_g.cpu().numpy()                           # bit for bit; NaN payloads differ by platform
                assert np.array_equal(np.isnan(got), np.isnan(tau)), (eps, window, k0)
                assert got[~np.isnan(got)].tobytes() == tau[~np.isnan(tau)].tobytes(), (eps, window, k0)
                assert np.array_equal(alive_g.cpu().numpy(), alive), (eps, window, k0)


@pytest.mark.parametrize("R,S", [(0, 5), (1, 1), (3, 700), (1000, 37), (4099, 64)])
def test_compaction_matches_oracle(R, S):
    from sparf_b200 import ops
    rng = np.random.default_rng(R * 131 + S + 1)
    res, r0, r1 = 7, -0.7, 1.9
    o, d, t = _samples(rng, R, S, r0, r1, res)
    bits = O.pack_bits(rng.random((res,) * 3) < 0.3)
    og, dg, tg, bg = _cuda(o, d, t, bits.view(np.int32))
    for window in sorted({1, 5, max(S // 3, 1), S, S + 3}):
        starts = list(range(0, S, window))
        for k0 in sorted(set(starts[:3] + starts[-1:])):             # the first windows and the ragged last one
            k1 = min(k0 + window, S)
            for p_alive in (None, 0.0, 0.5):
                alive = None if p_alive is None else (rng.random(R) < p_alive).astype(np.uint8)
                ag = None if alive is None else _cuda(alive)[0]
                for grid in (None, (bits, res, r0, r1)):
                    kw = dict(bits=bg, res=res, range=(r0, r1)) if grid else {}
                    got = ops.termination_compact(og, dg, tg, k0, k1, ag, **kw)
                    want = T.compact(o, d, t, k0, k1, alive, grid)
                    for g, w in zip(got, want):
                        g = g.cpu().numpy()
                        assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), \
                            (window, k0, p_alive, grid is not None)


def test_compaction_above_2_31_samples():
    """R * (k1 - k0) = R * 4095 > 2^31 window samples: window positions, sample indices and offsets past 2^31.  Every
    sample sits inside an empty grid except whole rays moved outside the box and single samples pushed out along the
    ray; those of them in the window [1, 4096) of a live ray, and only those, come out, in order"""
    from sparf_b200 import _lib
    L = _lib.lib()
    S, k0, k1 = 4096, 1, 4096
    R = (1 << 31) // (k1 - k0) + 200
    n = R * S
    assert R * (k1 - k0) > (1 << 31)
    dev = "cuda"
    origins = torch.zeros(R, 3, device=dev)
    dirs = torch.full((R, 3), 0.5, device=dev)
    t = torch.zeros(R, S, device=dev)
    alive = torch.ones(R, dtype=torch.uint8, device=dev)
    out_rays = [0, 7, R // 2, (1 << 31) // S - 1, (1 << 31) // S, R - 3, R - 1]
    dead = [7, R - 3, 524289]
    origins[out_rays] = 5.0
    alive[dead] = 0
    singles = [1, 2047, 2048, 4097 * 3, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, (1 << 31) + 2048, n - 2, n - 1,
               1234567 * 1024 + 3, 524289 * S + 5, 524290 * S, 524290 * S + 1]
    t.view(-1)[singles] = 10.0                    # x = 0 + 10 * 0.5 = 5: outside
    cand = set(singles) | {r * S + k for r in out_rays for k in range(S)}
    want = sorted(m for m in cand if k0 <= m % S < k1 and m // S not in dead)
    res = 4
    bits = torch.zeros((res ** 3 + 31) // 32, dtype=torch.int32, device=dev)
    ws = torch.empty(L.sparf_termination_workspace_bytes(R, k1 - k0), dtype=torch.uint8, device=dev)
    K = torch.empty((), dtype=torch.int64, device=dev)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (R, S, k0, k1, p(origins), p(dirs), p(t), p(alive), p(bits), res, -1.2, 1.2)
    _lib.check(L.sparf_termination_count(*args, p(K), p(ws), ws.numel(), st), "termination_count")
    k = K.item()
    assert k == len(want)
    idx = torch.empty(k, dtype=torch.int64, device=dev)
    ok, dk, tk = torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev), torch.empty(k, device=dev)
    _lib.check(L.sparf_termination_emit(*args, p(idx), p(ok), p(dk), p(tk), p(ws), ws.numel(), st), "termination_emit")
    assert idx.cpu().tolist() == want
    r = idx // S
    assert torch.equal(ok, origins[r]) and torch.equal(dk, dirs[r]) and torch.equal(tk, t.view(-1)[idx])
    del t, ws


# ------------------------------------------------------------------------------------------------ renders
def _wall_net(opt, data):
    from time_termination import camera_normal, scene_graph
    return scene_graph(opt, ("wall", 0.0, 400.0), camera_normal(data.pose))


def _scene(name):
    """(net, opt, data, mode): a golden case, or an analytic wall every ray ends on (metric 64 + 64 samples, or inverse
    depth with 64 coarse samples and no fine network)"""
    if name.startswith("c1"):
        net, c, opt, data, *_ = H.build_graph(name)
        return net, opt, data, c["mode"]
    inverse = name == "wall_inverse"
    opt = common.make_opt(S=64, S_fine=64, fine=not inverse, depth_param="inverse" if inverse else "metric",
                          depth_range=(1, 0) if inverse else (1.5, 4.5))
    data = common.make_scene(21, 2, 24, 32)
    data.depth_range = torch.tensor([[1.5, 4.5]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].cuda()
    return _wall_net(opt, data), opt, data, "val"


def _render(net, opt, data, mode):
    Hh, Ww = data.image.shape[-2:]
    return net.render(opt, data.pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"),
                      depth_range=net._depth_range(opt, data), iter=10, mode=mode)


def _masked_reference(net, opt, data, mode, eps, window, grids):
    """the dense render assembled from ops calls, with σ = rgb = 0 at the samples the oracle skips"""
    from sparf_b200 import ops
    Hh, Ww = data.image.shape[-2:]
    center, ray = ops.raygen(data.pose, data.intr, Ww, ray_idx=torch.arange(Hh * Ww, device="cuda"))
    B, N = center.shape[:2]
    o, d = center.reshape(-1, 3), ray.reshape(-1, 3)
    depth_range = net._depth_range(opt, data)
    white = bool(opt.nerf.setbg_opaque or opt.mask_img)

    def masked(nerf, g, t):
        sigma, rgb = ops.mlp_forward(nerf._spec(), o, d, t, nerf.kernel_params(), progress=nerf.progress)
        keep = None if g is None else O.kept(_np_bits(g.bits), g.res, *g.range, o.cpu().numpy(), d.cpu().numpy(),
                                               t.cpu().numpy())
        ev = torch.from_numpy(T.evaluated(sigma.cpu().numpy(), t.cpu().numpy(), d.cpu().numpy(), eps, window,
                                          keep)).cuda()
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
@pytest.mark.parametrize("grid", [False, True])
@pytest.mark.parametrize("name", ["c10_val_full_image", "c11_eval_full_image", "wall_metric", "wall_inverse"])
def test_render_equals_masked_dense_reference(name, grid, engine, engine_guard):
    """several (eps, window) pairs, with and without grids, metric (with a fine pass) and inverse depth"""
    import sparf_b200
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    net, opt, data, mode = _scene(name)
    fine = opt.nerf.fine_sampling
    grids = (_random_grid(16, 0.6, 1), _random_grid(12, 0.6, 2) if fine else None) if grid else (None, None)
    keys = [k for k in (ALL_KEYS if fine else KEYS)]
    skipped = []
    for eps, window in ((1e-4, 16), (1e-3, 7), (0.3, 1), (0.9, 5), (0.5, 200)):
        net.set_occupancy(*grids)
        net.set_early_termination(eps, window)
        with torch.no_grad():
            out = _render(net, opt, data, mode)
            ref = _masked_reference(net, opt, data, mode, eps, window, grids)
        _assert_same(out, ref, keys)
        skipped.append(round((out["density_samples"] == 0).float().mean().item(), 3))
    print("%s grid=%s: skipped fraction (coarse) per (eps, window): %s" % (name, grid, skipped))
    if name.startswith("wall"):
        assert max(skipped) > 0.3                                  # the wall does terminate rays


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("name", ["c10_val_full_image", "c11_eval_full_image"])
def test_eps_zero_renders_bit_identically(name, engine, engine_guard):
    """eps = 0 (nothing terminates): the golden val / eval renders equal the dense render without a grid and the
    grid-only render with one, for every window"""
    import sparf_b200
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    net, c, opt, data, *_ = H.build_graph(name)
    grids = (_random_grid(16, 0.5, 3), _random_grid(16, 0.5, 4))
    with torch.no_grad():
        for g in ((None, None), grids):
            net.set_occupancy(*g)
            net.set_early_termination(None)
            base = net.forward(opt, data, iter=10, mode=c["mode"])
            keys = [k for k in base if torch.is_tensor(base[k]) and base[k].is_floating_point()]
            assert "rgb" in keys and (not c["fine"] or "rgb_fine" in keys)
            for window in (1, 16, 1000):
                net.set_early_termination(0.0, window)
                _assert_same(net.forward(opt, data, iter=10, mode=c["mode"]), base, keys)


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_analytic_scene_bounds(engine, engine_guard):
    """a sharp octahedron σ = softplus(400 (0.6 - |x|_1)): for the same samples the coarse composite differs from the
    dense one by less than eps in opacity and rgb and eps * max t in depth, and every ray that skipped samples has
    all_cumulated < eps in both renders.  The fine pass's samples move with the coarse weights; its difference is
    reported and held to 1e-2 (rgb, opacity) and 1e-2 * max t (depth)"""
    import sparf_b200
    from time_occupancy import octahedron_graph
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    opt = common.make_opt(S=128, S_fine=128, fine=True, depth_range=(1.5, 4.5))
    net = octahedron_graph(opt, 0.6, k=400.0)
    data = common.make_scene(21, 2, 24, 32)
    data.depth_range = torch.tensor([[1.5, 4.5]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].cuda()
    tol = 2e-6
    for eps, window in ((1e-4, 16), (1e-3, 32)):
        with torch.no_grad():
            net.set_early_termination(None)
            dense = _render(net, opt, data, "val")
            net.set_early_termination(eps, window)
            term = _render(net, opt, data, "val")
        assert torch.equal(term["t"], dense["t"])
        R = dense["t"].shape[0] * dense["t"].shape[1]
        t = dense["t"].reshape(R, -1)
        skipped = (term["density_samples"].reshape(R, -1) == 0) & (dense["density_samples"].reshape(R, -1) != 0)
        cut = skipped.any(1)
        assert 0.01 < cut.float().mean().item() < 0.99, cut.float().mean().item()
        d = {k: (term[k] - dense[k]).reshape(R, -1).abs().amax(1) for k in ("rgb", "opacity", "depth", "rgb_fine",
                                                                           "opacity_fine", "depth_fine")}
        assert (d["opacity"] < eps + tol).all() and (d["rgb"] < eps + tol).all(), (d["opacity"].max(), d["rgb"].max())
        assert (d["depth"] < (eps + tol) * t.amax(1)).all(), (d["depth"] - eps * t.amax(1)).max()
        for out in (dense, term):
            assert (out["all_cumulated"].reshape(R)[cut] < eps).all()
        print("%s eps %g window %d: rays cut %.3f, coarse max |d rgb| %.3g |d opacity| %.3g |d depth| %.3g; fine %.3g "
              "%.3g %.3g" % (engine, eps, window, cut.float().mean().item(), d["rgb"].max(), d["opacity"].max(),
                             d["depth"].max(), d["rgb_fine"].max(), d["opacity_fine"].max(), d["depth_fine"].max()))
        assert d["rgb_fine"].max() < 1e-2 and d["opacity_fine"].max() < 1e-2
        assert (d["depth_fine"] < 1e-2 * t.amax(1)).all()


# ------------------------------------------------------------------------------------------------ untouched paths
def test_termination_is_ignored_outside_inference(engine_guard):
    """early termination (and a grid) set, but mode train / test-optim, gradients on, or render_to_max: bit-identical
    to the same call without them; likewise after set_early_termination(None)"""
    net, c, opt, data, *_ = H.build_graph("c10_val_full_image")
    Hh, Ww = data.image.shape[-2:]
    kw = dict(H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"), iter=10)
    grids = (_random_grid(16, 0.3, 5), _random_grid(16, 0.3, 6))
    depth_range = net._depth_range(opt, data)

    def run(mode, grad, attach, to_max=False):
        net.set_occupancy(*(grids if attach == "grid" else (None, None)))
        net.set_early_termination(*((0.999999, 4) if attach else (None,)))
        torch.manual_seed(1234)                   # train / test-optim draw stratified offsets, noise and the fine grid
        with torch.set_grad_enabled(grad):
            if to_max:
                out = net.render_to_max(opt, data.pose, mode=mode, depth_min=1.0,
                                        depth_max=torch.full((len(data.pose), Hh * Ww), 3.0, device="cuda"), **kw)
            else:
                out = net.render(opt, data.pose, mode=mode, depth_range=depth_range, **kw)
        return {k: v.detach() for k, v in out.items() if torch.is_tensor(v)}

    for attach in ("term", "grid"):
        for mode, grad in (("train", False), ("train", True), ("test-optim", False), ("val", True)):
            _assert_same(run(mode, grad, attach), run(mode, grad, None), ALL_KEYS)
        _assert_same(run("val", False, attach, to_max=True), run("val", False, None, to_max=True), ALL_KEYS)
    net.set_early_termination(0.999999, 4)
    net.set_early_termination(None)
    with torch.no_grad():
        detached = net.render(opt, data.pose, mode="val", depth_range=depth_range, **kw)
    _assert_same(detached, run("val", False, None), ALL_KEYS)
    net.set_early_termination(0.999999, 4)         # and the setting does apply here: the same call differs
    with torch.no_grad():
        cut = net.render(opt, data.pose, mode="val", depth_range=depth_range, **kw)
    assert not torch.equal(cut["density_samples"], detached["density_samples"])
