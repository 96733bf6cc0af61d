"""Occupancy grids on the device (sparf_occupancy_build / count / emit, sparf_b200.occupancy, Graph.set_occupancy): the
bits and the compaction equal the NumPy oracle (tests/occupancy_oracle.py) byte for byte; a render with a grid equals
the dense render with σ and rgb zeroed at the skipped samples, bit for bit; an all-occupied grid changes nothing; the
error of a real grid on an analytic scene is within the bound of what it skipped; and every call the grid must not
touch (training, test-time optimisation, gradients, a detached grid) is bit-identical to a render without one."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import common
import helpers as H
import occupancy_oracle as O

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

KEYS = ["rgb", "rgb_var", "depth", "depth_var", "opacity", "weights", "all_cumulated", "density_samples", "rgb_samples", "t"]


def _engine_or_skip(engine):
    from sparf_b200 import _lib
    if not _lib.lib().sparf_engine_available(_lib.ENGINES[engine]):
        pytest.skip("%s not available" % engine)


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _bits(x):
    """a float tensor's bit pattern (bit-identity, NaN included)"""
    return x.detach().contiguous().view(torch.int32)


def _assert_same(a, b, keys):
    for k in keys:
        assert torch.equal(_bits(a[k].reshape(-1)), _bits(b[k].reshape(-1))), k


def _np_bits(bits):
    return bits.cpu().numpy().view(np.uint32)


def _random_grid(res, p, seed, device="cuda"):
    from sparf_b200.occupancy import OccupancyGrid
    occ = np.random.default_rng(seed).random((res,) * 3) < p
    bits = torch.from_numpy(O.pack_bits(occ).view(np.int32).copy()).to(device)
    return OccupancyGrid(bits, res, (-1.2, 1.2), 0.01)


# ------------------------------------------------------------------------------------------------ kernels vs oracle
@pytest.mark.parametrize("res", [1, 2, 5, 31, 32, 33, 128])
def test_build_matches_oracle(res):
    from sparf_b200 import ops
    rng = np.random.default_rng(100 + res)
    thres = np.float32(0.75)
    for hot in (0.0, 0.004, 0.03, 1.0):
        sigma = (rng.random((res + 1,) * 3) * 0.75).astype(np.float32)            # below thres
        sel = rng.random(sigma.shape)
        sigma[sel < hot / 4] = thres                                               # exactly at thres: occupied
        sigma[(sel >= hot / 4) & (sel < hot / 2)] = np.nan
        sigma[(sel >= hot / 2) & (sel < 3 * hot / 4)] = np.inf
        sigma[(sel >= 3 * hot / 4) & (sel < hot)] = thres + 1
        sigma[(sel >= hot) & (sel < hot + 0.01)] = np.nextafter(thres, np.float32(0))   # just below: empty
        sigma[(sel >= hot + 0.01) & (sel < hot + 0.02)] = -np.inf
        bits = ops.occupancy_build(torch.from_numpy(sigma).cuda(), float(thres))
        want = O.build(sigma, thres)
        assert bits.shape == want.shape
        assert np.array_equal(_np_bits(bits), want), (res, hot)


def _samples(rng, R, S, r0, r1, res):
    """rays from inside and outside the box; some samples exactly on its faces and on cell planes, some NaN / inf"""
    o = rng.uniform(r0 - 0.6, r1 + 0.6, (R, 3)).astype(np.float32)
    d = rng.normal(size=(R, 3)).astype(np.float32)
    t = rng.uniform(0, 1.5, (R, S)).astype(np.float32)
    f32 = np.float32
    planes = np.array([r0, r1, np.nextafter(f32(r1), f32(r0)), np.nextafter(f32(r0), f32(r0 - 1)), 0.5 * (r0 + r1)], f32)
    on = rng.random(R) < 0.3                       # these rays sit on a face / plane at t = 0 on one axis
    ax = rng.integers(0, 3, R)
    o[on, ax[on]] = planes[rng.integers(0, len(planes), on.sum())]
    d[on & (rng.random(R) < 0.5), :] = 0           # ... and stay there
    t[:, 0] = np.where(rng.random(R) < 0.5, 0, t[:, 0])
    bad = rng.random((R, S))
    t[bad < 0.002] = np.nan
    t[(bad >= 0.002) & (bad < 0.004)] = np.inf
    return o, d, t


@pytest.mark.parametrize("R,S", [(0, 5), (1, 1), (3, 700), (1000, 37), (4099, 64)])
def test_compaction_matches_oracle(R, S):
    from sparf_b200 import ops
    rng = np.random.default_rng(R * 131 + S)
    for res, (r0, r1) in ((1, (-1.2, 1.2)), (7, (-0.7, 1.9)), (64, (-1.2, 1.2))):
        o, d, t = _samples(rng, R, S, r0, r1, res)
        for p in (0.0, 0.3, 1.0):
            occ = rng.random((res,) * 3) < p
            bits = O.pack_bits(occ)
            got = ops.occupancy_compact(torch.from_numpy(bits.view(np.int32)).cuda(), res, (r0, r1), torch.from_numpy(o).cuda(),
                                        torch.from_numpy(d).cuda(), torch.from_numpy(t).cuda())
            want = O.compact(bits, res, r0, r1, o, d, t)
            assert got[0].shape == want[0].shape, (res, p, got[0].shape, want[0].shape)
            for g, w in zip(got, want):
                g = g.cpu().numpy()
                assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (res, p)


def test_compaction_above_2_31_samples():
    """R * S = 2^31 + 20480 samples: sample indices, tile indices and offsets past 2^31.  All samples sit inside an empty
    grid except whole rays moved outside the box and single samples pushed out along the ray; those, and only those, come
    out, in order"""
    from sparf_b200 import _lib
    L = _lib.lib()
    S = 4096
    R = (1 << 31) // S + 5
    n = R * S
    dev = "cuda"
    origins = torch.zeros(R, 3, device=dev)
    dirs = torch.full((R, 3), 0.5, device=dev)
    t = torch.zeros(R, S, device=dev)
    out_rays = [0, 7, R // 2, (1 << 31) // S - 1, (1 << 31) // S, R - 1]
    origins[out_rays] = 5.0
    singles = [1, 2047, 2048, 4097 * 3, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, (1 << 31) + 2048, n - 2, n - 1,
               1234567 * 1024 + 3]
    t.view(-1)[singles] = 10.0                    # x = 0 + 10 * 0.5 = 5: outside
    want = sorted(set(singles) | {r * S + k for r in out_rays for k in range(S)})
    res = 4
    bits = torch.zeros((res ** 3 + 31) // 32, dtype=torch.int32, device=dev)
    ws = torch.empty(L.sparf_occupancy_workspace_bytes(R, S), dtype=torch.uint8, device=dev)
    K = torch.empty((), dtype=torch.int64, device=dev)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (R, S, p(origins), p(dirs), p(t), p(bits), res, -1.2, 1.2)
    _lib.check(L.sparf_occupancy_count(*args, p(K), p(ws), ws.numel(), st), "occupancy_count")
    k = K.item()
    assert k == len(want)
    idx = torch.empty(k, dtype=torch.int64, device=dev)
    ok, dk, tk = torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev), torch.empty(k, device=dev)
    _lib.check(L.sparf_occupancy_emit(*args, p(idx), p(ok), p(dk), p(tk), p(ws), ws.numel(), st), "occupancy_emit")
    assert idx.cpu().tolist() == want
    r = idx // S
    assert torch.equal(ok, origins[r]) and torch.equal(dk, dirs[r]) and torch.equal(tk, t.view(-1)[idx])
    del t, ws


# ------------------------------------------------------------------------------------------------ renders
@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("name", ["c10_val_full_image", "c11_eval_full_image"])
def test_all_occupied_grid_renders_bit_identically(name, engine, engine_guard):
    """thres = 0: every cell is occupied (σ >= 0), so render_by_slices must not change a bit (coarse + fine, metric
    depth in c10; coarse only, inverse depth, opaque background and the BARF mask in c11)"""
    import sparf_b200
    from sparf_b200 import occupancy
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    net, c, opt, data, *_ = H.build_graph(name)
    with torch.no_grad():
        dense = net.forward(opt, data, iter=10, mode=c["mode"])
        grids = [occupancy.build_grid(opt, m, res=32, thres=0.0) for m in net.get_network_components()]
        assert all(g.occupied_fraction() == 1.0 for g in grids)
        net.set_occupancy(*grids)
        sparse = net.forward(opt, data, iter=10, mode=c["mode"])
    keys = [k for k in dense if torch.is_tensor(dense[k]) and dense[k].is_floating_point()]
    assert "rgb" in keys and (not c["fine"] or "rgb_fine" in keys)
    _assert_same(sparse, dense, keys)


def _masked_reference(net, opt, data, grid, grid_fine):
    """the dense render assembled from ops calls, with σ = rgb = 0 at the samples the oracle skips"""
    from sparf_b200 import ops
    from sparf_b200.renderer import Graph
    H_, W_ = data.image.shape[-2:]
    center, ray = ops.raygen(data.pose, data.intr, W_, ray_idx=torch.arange(H_ * W_, device="cuda"))
    B, N = center.shape[:2]
    o, d = center.reshape(-1, 3), ray.reshape(-1, 3)
    near, far, rng = Graph._range_floats(data.depth_range[0])
    white = bool(opt.nerf.setbg_opaque or opt.mask_img)

    def masked(nerf, g, t):
        sigma, rgb = ops.mlp_forward(nerf._spec(), o, d, t, nerf.kernel_params(), progress=nerf.progress)
        if g is not None:
            keep = torch.from_numpy(O.kept(_np_bits(g.bits), g.res, *g.range, o.cpu().numpy(), d.cpu().numpy(),
                                           t.cpu().numpy())).cuda()
            sigma = torch.where(keep, sigma, torch.zeros_like(sigma))
            rgb = torch.where(keep[..., None], rgb, torch.zeros_like(rgb))
        rgb_map, depth, opacity, weights, depth_var, rgb_var, all_cum = ops.composite(sigma, rgb, t, d, white)
        return dict(rgb=rgb_map, depth=depth, opacity=opacity, weights=weights, depth_var=depth_var, rgb_var=rgb_var,
                    all_cumulated=all_cum, density_samples=sigma, rgb_samples=rgb, t=t)

    t = ops.sample_depth(B * N, opt.nerf.sample_intvs, near, rng, device="cuda")
    out = masked(net.nerf, grid, t)
    grid_u = torch.linspace(0, 1, opt.nerf.sample_intvs_fine + 1, device="cuda")
    _, t_all = ops.sample_pdf_merge(out["weights"], t, 0.5 * (grid_u[:-1] + grid_u[1:]), near, far)
    out.update({k + "_fine": v for k, v in masked(net.nerf_fine, grid_fine, t_all).items()})
    return out


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("fine_grid", [True, False])
def test_random_grid_render_equals_masked_dense_reference(engine, fine_grid, engine_guard):
    import sparf_b200
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    net, c, opt, data, *_ = H.build_graph("c10_val_full_image")
    Hh, Ww = data.image.shape[-2:]
    grid, grid_fine = _random_grid(16, 0.5, 1), (_random_grid(12, 0.3, 2) if fine_grid else None)
    net.set_occupancy(grid, grid_fine)
    with torch.no_grad():
        out = net.render(opt, data.pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"),
                         depth_range=net._depth_range(opt, data), iter=10, mode="val")
        ref = _masked_reference(net, opt, data, grid, grid_fine)
    keys = KEYS + [k + "_fine" for k in KEYS]
    _assert_same(out, ref, keys)
    skipped = (out["density_samples"] == 0).float().mean().item()
    print("skipped fraction (coarse): %.3f" % skipped)
    assert 0.05 < skipped < 0.95


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_analytic_octahedron_scene(engine, engine_guard):
    """σ = softplus(c - k |x|_1) (octahedron_weights of tools/time_occupancy.py): every skipped sample's dense σ is below
    thres, the kept fraction is the oracle's, and rgb / depth / opacity differ from the dense render by at most what the
    skipped samples could absorb"""
    import sparf_b200
    from sparf_b200 import occupancy, ops
    from sparf_b200.renderer import Graph
    from time_occupancy import octahedron_weights
    _engine_or_skip(engine)
    sparf_b200.set_engine(engine)
    opt = common.make_opt(S=128, depth_range=(1.5, 4.5))
    net = Graph(opt, torch.device("cuda"))
    net.nerf.load_state_dict(octahedron_weights(opt, c=40 * 0.8, k=40.0))
    data = common.make_scene(21, 2, 24, 32)
    data.depth_range = torch.tensor([[1.5, 4.5]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].cuda()
    Hh, Ww = 24, 32
    kw = dict(H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"),
              depth_range=net._depth_range(opt, data), iter=10, mode="val")
    thres = 0.01
    with torch.no_grad():
        dense = net.render(opt, data.pose, **kw)
        grid = occupancy.build_grid(opt, net.nerf, res=64, range=(-1.2, 1.2), thres=thres)
        net.set_occupancy(grid)
        sparse = net.render(opt, data.pose, **kw)
    o, d = dense["origins"].reshape(-1, 3), dense["viewdirs"].reshape(-1, 3)
    t = dense["t"].reshape(o.shape[0], -1)
    keep = torch.from_numpy(O.kept(_np_bits(grid.bits), 64, -1.2, 1.2, o.cpu().numpy(), d.cpu().numpy(),
                                   t.cpu().numpy())).cuda()
    idx = ops.occupancy_compact(grid.bits, 64, (-1.2, 1.2), o, d, t)[0]
    assert idx.numel() == keep.sum().item()
    frac = keep.float().mean().item()
    print("%s: occupied cells %.3f, kept samples %.3f" % (engine, grid.occupied_fraction(), frac))
    assert 0.05 < frac < 0.9
    sig_d = dense["density_samples"].reshape(keep.shape)
    assert (sig_d[~keep] < thres).all()
    assert sig_d.max().item() > 10 and dense["opacity"].max().item() > 0.99
    sig_s = sparse["density_samples"].reshape(keep.shape)
    assert torch.equal(_bits(sig_s[keep]), _bits(sig_d[keep])) and (sig_s[~keep] == 0).all()
    # per ray: eps = sum over skipped samples of σ δ (δ as the composite takes it) bounds every output's change
    gap = torch.cat([t[:, 1:] - t[:, :-1], torch.full_like(t[:, :1], 1e10)], 1) * d.norm(dim=-1, keepdim=True)
    eps = torch.where(keep, torch.zeros_like(sig_d), sig_d.double() * gap.double()).sum(1)
    bound = (1 - torch.exp(-eps)).float()
    tol = 2e-6
    dr = (sparse["rgb"] - dense["rgb"]).reshape(-1, 3).abs().amax(1)
    do = (sparse["opacity"] - dense["opacity"]).reshape(-1).abs()
    dd = (sparse["depth"] - dense["depth"]).reshape(-1).abs()
    assert (dr <= bound + tol).all(), (dr - bound).max().item()
    assert (do <= bound + tol).all(), (do - bound).max().item()
    assert (dd <= (bound + tol) * t.amax(1)).all(), (dd - bound * t.amax(1)).max().item()
    print("max |d rgb| %.3g, |d opacity| %.3g, |d depth| %.3g, max bound %.3g" % (
        dr.max().item(), do.max().item(), dd.max().item(), bound.max().item()))


# ------------------------------------------------------------------------------------------------ untouched paths
def test_grid_is_ignored_outside_inference(engine_guard):
    """a grid attached, but mode train / test-optim or gradients on: bit-identical to no grid; likewise after
    set_occupancy(None)"""
    net, c, opt, data, *_ = H.build_graph("c10_val_full_image")
    Hh, Ww = data.image.shape[-2:]
    kw = dict(H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device="cuda"),
              depth_range=net._depth_range(opt, data), iter=10)
    grids = (_random_grid(16, 0.3, 5), _random_grid(16, 0.3, 6))

    def run(mode, grad, attach):
        net.set_occupancy(*(grids if attach else (None, None)))
        torch.manual_seed(1234)                   # train / test-optim draw stratified offsets, noise and the fine grid
        with torch.set_grad_enabled(grad):
            out = net.render(opt, data.pose, mode=mode, **kw)
        return {k: v.detach() for k, v in out.items() if torch.is_tensor(v)}

    for mode, grad in (("train", False), ("train", True), ("test-optim", False), ("val", True)):
        _assert_same(run(mode, grad, True), run(mode, grad, False), KEYS + [k + "_fine" for k in KEYS])
    net.set_occupancy(*grids)
    net.set_occupancy(None)
    with torch.no_grad():
        detached = net.render(opt, data.pose, mode="val", **kw)
    _assert_same(detached, run("val", False, False), KEYS + [k + "_fine" for k in KEYS])
    net.set_occupancy(*grids)       # and the grid does apply here: the same call differs
    with torch.no_grad():
        sparse = net.render(opt, data.pose, mode="val", **kw)
    assert not torch.equal(sparse["density_samples"], detached["density_samples"])
