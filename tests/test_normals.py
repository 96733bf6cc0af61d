"""The point gradient of the density (sparf_density_gradient, ops.density_gradient) and the normal maps built on it
(Graph.set_normals, sparf_b200/normals.py), on the GPU."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

C2F = (0.1, 0.5)
TRUNK_KEYS = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], [])
ENGINES = ["simt_fp32", "tc_3x", "tc_1x", "tc_3x_w1"]
OTHER_KEYS = ["rgb", "rgb_var", "depth", "depth_var", "opacity", "weights", "all_cumulated", "density_samples",
              "rgb_samples", "t", "origins", "viewdirs"]


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _engine(name):
    from sparf_b200 import _lib
    e = _lib.ENGINES[name]
    if not _lib.lib().sparf_engine_available(e):
        pytest.skip("%s not available on this device" % name)
    return e


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _problem(M, seed):
    import common
    from sparf_b200 import ops
    opt = common.make_opt(barf_c2f=C2F)
    sd = common.det_weights(opt, seed, progress=0.3)
    params = [sd[k].cuda() for k in TRUNK_KEYS]
    g = torch.Generator(device="cpu").manual_seed(seed)
    pts = (torch.rand(M, 3, generator=g) * 3 - 1.5).cuda()
    return ops.MLPSpec(barf_c2f=C2F), params, sd["progress"].cuda(), pts


# ------------------------------------------------------------------------------------------------ the entry point
# 2 x 32 768 + 5 crosses the density backward's chunk boundary twice, with a partial last chunk
@pytest.mark.parametrize("M", [1, 127, 128, 129, 2 * 32768 + 5])
@pytest.mark.parametrize("engine", ENGINES)
def test_gradient_equals_density_backward(engine, M):
    """grad_points is torch.equal to density_backward's d_points for d_raw = 1, d_feat = NULL; rows past M keep a
    sentinel; no parameter changes"""
    from sparf_b200 import _lib
    eng = _engine(engine)
    L = _lib.lib()
    spec, params, prog, pts = _problem(M, seed=M % 1000 + 17)
    m, keep = spec.fill(params, prog)
    before = [p.clone() for p in params]
    ws2 = L.sparf_density_workspace_bytes(ctypes.byref(m), M, 2, eng)
    ws1 = L.sparf_density_workspace_bytes(ctypes.byref(m), M, 1, eng)
    assert 0 < ws2 <= ws1, (ws2, ws1)
    ws = torch.empty(ws1, dtype=torch.uint8, device="cuda")
    out = torch.full((M + 7, 3), 12345.0, device="cuda")
    _lib.check(L.sparf_density_gradient(ctypes.byref(m), eng, M, _p(pts), _p(out), _p(ws), ws2, _stream()), "density_gradient")
    grads = [torch.zeros_like(p) for p in params]
    gs = spec.grad_struct(grads)
    d_raw = torch.ones(M, device="cuda")
    d_pts = torch.zeros_like(pts)
    _lib.check(L.sparf_density_backward(ctypes.byref(m), eng, M, _p(pts), _p(d_raw), None, ctypes.byref(gs), _p(d_pts),
                                        _p(ws), ws.numel(), _stream()), "density_backward")
    torch.cuda.synchronize()
    assert torch.equal(out[:M], d_pts)
    assert (out[M:] == 12345.0).all()
    assert all(torch.equal(a, b) for a, b in zip(params, before))
    # and the same through ops.density_gradient with the points as [..., 3]
    from sparf_b200 import ops
    g = ops.density_gradient(spec, pts.view(1, M, 3), params, progress=prog, engine=eng)
    assert g.shape == (1, M, 3) and torch.equal(g.view(M, 3), d_pts)


@pytest.mark.parametrize("engine", ENGINES)
def test_gradient_of_no_points_launches_nothing(engine):
    from sparf_b200 import _lib
    eng = _engine(engine)
    L = _lib.lib()
    spec, params, prog, _ = _problem(1, seed=3)
    m, keep = spec.fill(params, prog)
    torch.cuda.synchronize()
    c0 = L.sparf_launch_count()
    _lib.check(L.sparf_density_gradient(ctypes.byref(m), eng, 0, None, None, None, 0, _stream()), "density_gradient")
    assert L.sparf_launch_count() == c0


def test_gradient_matches_fp64():
    """against fp64 autograd of density_oracle.raw_density, within test_density.py's bound on the points' gradient
    (2e-3 or 4 x the SIMT engine's own error), points whose ReLU pattern flips in fp32 taken out as there.  The engines
    test_density.py bounds so: tc_1x multiplies single bf16 halves by design (test_tc_engine.py bounds it)."""
    from density_oracle import raw_density
    from sparf_b200 import _lib, ops
    M = 4096
    spec, params, prog, pts = _problem(M, seed=23)
    p64 = {k: v.double() for k, v in zip(TRUNK_KEYS, params)}
    p64["progress"] = prog
    x64 = pts.double().requires_grad_(True)
    raw, _ = raw_density(p64, x64, barf_c2f=C2F)
    (truth,) = torch.autograd.grad(raw.sum(), x64)
    names = [n for n in ("simt_fp32", "tc_3x", "tc_3x_w1") if _lib.lib().sparf_engine_available(_lib.ENGINES[n])]
    got = {n: ops.density_gradient(spec, pts, params, progress=prog, engine=_lib.ENGINES[n]).double() for n in names}
    scale = truth.abs().max()
    per_point = torch.stack([(got[n] - truth).abs().amax(-1) / scale for n in names]).amax(0)
    keep = per_point <= 1e-4
    assert int((~keep).sum()) <= M // 100
    err = {n: ((got[n] - truth).abs()[keep].max() / scale).item() for n in names}
    print("point-gradient error vs fp64:", err)
    for n in names[1:]:
        assert err[n] < max(2e-3, 4 * err["simt_fp32"]), (n, err)


@pytest.mark.parametrize("engine", ENGINES)
def test_octahedron_normals_are_analytic(engine):
    """sigma = softplus(c - k |x|_1): the normal is sign(x) / sqrt(3) away from the coordinate planes"""
    import common
    from time_occupancy import octahedron_weights
    from sparf_b200 import mesh, ops
    eng = _engine(engine)
    opt = common.make_opt()
    sd = octahedron_weights(opt, c=24.0, k=40.0)
    params = [sd[k].cuda() for k in TRUNK_KEYS]
    g = torch.Generator(device="cpu").manual_seed(4)
    x = (torch.rand(20000, 3, generator=g) * 2 - 1)
    x = x[(x.abs() > 1e-3).all(-1)].cuda()
    n = mesh.unit_normals(ops.density_gradient(ops.MLPSpec(), x, params, progress=sd["progress"].cuda(), engine=eng))
    assert (n - torch.sign(x) / 3 ** 0.5).abs().max().item() <= 1e-5


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_mesh_normals_equal_autograd_path(engine, engine_guard):
    """mesh.density_normals against the autograd path it replaced (density backward with d_raw = 1)"""
    import common
    from sparf_b200 import mesh, ops
    from sparf_b200.frequency_nerf import NeRF
    eng = _engine(engine)
    opt = common.make_opt(barf_c2f=C2F)
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v for k, v in common.det_weights(opt, 31, progress=0.3).items()}, strict=False)
    pts = (torch.rand(mesh.NORMAL_CHUNK + 1000, 3, generator=torch.Generator().manual_seed(31)) * 3 - 1.5).cuda()
    got = mesh.density_normals(nerf, pts, engine=eng)
    spec, trunk = nerf._spec(), mesh._trunk(nerf)
    ref = torch.empty_like(pts)
    for c0 in range(0, pts.shape[0], mesh.NORMAL_CHUNK):
        x = pts[c0:c0 + mesh.NORMAL_CHUNK].detach().clone().requires_grad_(True)
        with torch.enable_grad():
            raw, _ = ops.density_forward(spec, x, trunk, progress=nerf.progress.detach(), engine=eng, features=False)
            (g,) = torch.autograd.grad(raw.sum(), x)
        norm = g.norm(dim=-1, keepdim=True)
        ref[c0:c0 + mesh.NORMAL_CHUNK] = torch.where(norm > 0, -g / norm, torch.zeros_like(g))
    assert torch.equal(got, ref)


# ------------------------------------------------------------------------------------------------ normal maps
def _scene(kind="octahedron", S=48, S_fine=48, H=20, W=28, B=2):
    import common
    from time_occupancy import octahedron_graph
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=S, S_fine=S_fine, fine=True, depth_range=(1.5, 4.5))
    data = common.make_scene(3, B, H, W, focal=float(max(H, W)) * 1.3)
    for key in ("image", "intr", "pose"):
        data[key] = data[key].cuda()
    data.depth_range = torch.tensor([[1.5, 4.5]] * B).cuda()
    if kind == "octahedron":
        net = octahedron_graph(opt, 0.6)
    else:
        net = Graph(opt, torch.device("cuda"))
        for i, m in enumerate(net.get_network_components()):
            m.load_state_dict(common.det_weights(opt, 40 + i, peaky=True), strict=False)
    return net, opt, data


def _render(net, opt, data, mode="val"):
    H, W = data.image.shape[-2:]
    return net.render(opt, data.pose, H=H, W=W, intr=data.intr, ray_idx=torch.arange(H * W, device="cuda"),
                      depth_range=data.depth_range[0], iter=None, mode=mode)


def _formula(nerf, pred, suffix):
    """the documented normal over the render's own w != 0 samples, summed per ray in NumPy sequential fp32; also the
    number of those samples"""
    from sparf_b200 import mesh, ops
    center, ray = pred["origins"], pred["viewdirs"]
    t, w = pred["t" + suffix], pred["weights" + suffix]
    B, N, S = t.shape[:3]
    R = B * N
    wf = w.reshape(-1)
    idx = torch.nonzero(wf != 0).reshape(-1)
    r = idx // S
    o, d = center.reshape(R, 3), ray.reshape(R, 3)
    x = o[r] + d[r] * t.reshape(-1)[idx, None]
    g = ops.density_gradient(nerf._spec(), x, mesh._trunk(nerf), progress=nerf.progress.detach())
    v = (wf[idx, None] * mesh.unit_normals(g)).cpu().numpy()
    rows = r.cpu().numpy()
    out = np.zeros((R, 3), np.float32)
    counts = np.bincount(rows, minlength=R)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    for j in range(int(counts.max()) if len(rows) else 0):
        live = np.nonzero(counts > j)[0]
        out[live] = out[live] + v[starts[live] + j]            # fp32, in increasing k
    return torch.from_numpy(out).view(B, N, 3), idx.numel()


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("kind", ["octahedron", "random"])
def test_normal_maps_are_the_formula(kind, engine, engine_guard):
    from sparf_b200 import ops
    ops.set_engine(_engine(engine))
    net, opt, data = _scene(kind)
    with torch.no_grad():
        off = _render(net, opt, data)
        net.set_normals(True)
        on = _render(net, opt, data)
        net.set_normals(False)
        again = _render(net, opt, data)
    assert "normal" not in off and "normal" not in again
    for k in OTHER_KEYS + [k + "_fine" for k in OTHER_KEYS if k not in ("origins", "viewdirs")]:
        assert torch.equal(on[k], off[k]), k
    for nerf, suffix in ((net.nerf, ""), (net.nerf_fine, "_fine")):
        want, _ = _formula(nerf, on, suffix)
        assert on["normal" + suffix].shape == want.shape
        assert torch.equal(on["normal" + suffix].cpu(), want), suffix
        assert (on["normal" + suffix].norm(dim=-1) <= on["opacity" + suffix][..., 0] * (1 + 1e-5) + 1e-6).all()


@pytest.mark.parametrize("kind", ["octahedron"])
def test_normal_maps_match_fp64_oracle(kind, engine_guard):
    """against normals_oracle.normal_map (fp64 weights and normals on the render's samples).  Tolerance: 2e-3 per
    component on 99 % of the rays and 5e-2 on all; a sample whose octahedron face differs between fp32 and fp64 moves
    its ray's normal by its weight times an O(1) change.  The random peaky network of test_normal_maps_are_the_formula
    is not bounded here: its fp32 normal maps were measured up to 0.26 (99th percentile 4e-2) from this oracle."""
    from normals_oracle import normal_map
    from sparf_b200 import ops
    ops.set_engine(_engine("tc_3x"))
    net, opt, data = _scene(kind)
    net.set_normals(True)
    with torch.no_grad():
        pred = _render(net, opt, data)
    for nerf, suffix in ((net.nerf, ""), (net.nerf_fine, "_fine")):
        t = pred["t" + suffix]
        B, N, S = t.shape[:3]
        sd = {k: v.cpu().numpy() for k, v in nerf.state_dict().items() if k.startswith("mlp_feat.")}
        ref, _ = normal_map(sd, pred["origins"].reshape(-1, 3).cpu().numpy(), pred["viewdirs"].reshape(-1, 3).cpu().numpy(),
                            t.reshape(B * N, S).cpu().numpy(), progress=float(nerf.progress))
        err = np.abs(pred["normal" + suffix].reshape(-1, 3).cpu().numpy() - ref).max(-1)
        print(kind, suffix, "max err %.2e, 99th percentile %.2e" % (err.max(), np.quantile(err, 0.99)))
        assert np.quantile(err, 0.99) <= 2e-3 and err.max() <= 5e-2


@pytest.mark.parametrize("config", ["box_grid", "contracted_grid", "termination", "termination_grid"])
def test_normals_over_grids_and_termination(config, engine_guard):
    """the normal is the formula over the render's own weights; the points differentiated are the w != 0 samples"""
    from sparf_b200 import occupancy, ops
    ops.set_engine(_engine("tc_3x"))
    net, opt, data = _scene("octahedron")
    with torch.no_grad():
        if config == "contracted_grid":
            grids = [occupancy.build_grid(opt, m, res=64, contraction=((0.0, 0.0, 0.0), 1.0))
                     for m in net.get_network_components()]
        else:
            grids = [occupancy.build_grid(opt, m, res=64) for m in net.get_network_components()]
        if "grid" in config:
            net.set_occupancy(*grids)
        if config.startswith("termination"):
            net.set_early_termination(1e-4, 8)
        net.set_normals(True)
        e0 = ops.EVALS["bwd"]
        pred = _render(net, opt, data)
        evals = ops.EVALS["bwd"] - e0
        kept = 0
        for nerf, suffix in ((net.nerf, ""), (net.nerf_fine, "_fine")):
            want, n = _formula(nerf, pred, suffix)
            kept += n
            assert torch.equal(pred["normal" + suffix].cpu(), want), suffix
    assert evals == kept


def test_render_by_slices_and_scope(engine_guard):
    from sparf_b200 import ops
    ops.set_engine(_engine("tc_3x"))
    net, opt, data = _scene("octahedron")
    H, W = data.image.shape[-2:]
    net.set_normals(True)
    with torch.no_grad():
        whole = _render(net, opt, data)
        net.full_image_rays_per_launch = 2 * 128
        opt.nerf.rand_rays = 128
        sliced = net.render_by_slices(opt, data.pose, H, W, data.intr, data.depth_range[0], iter=None, mode="val")
        assert torch.equal(sliced["normal"], whole["normal"]) and torch.equal(sliced["normal_fine"], whole["normal_fine"])
        train = _render(net, opt, data, mode="train")
    with torch.enable_grad():
        val_grad = _render(net, opt, data)
    for pred in (train, val_grad):
        assert "normal" not in pred and "normal_fine" not in pred


def test_octahedron_normals_face_the_camera(engine_guard):
    """a sharp octahedron (k = 400) sampled finely: a soft one mixes in the normals of the faces behind the silhouette"""
    from time_occupancy import octahedron_graph
    from sparf_b200 import ops
    ops.set_engine(_engine("tc_3x"))
    _, opt, data = _scene("octahedron", S=128, S_fine=128, H=40, W=56)
    net = octahedron_graph(opt, 0.6, k=400.0)
    net.set_normals(True)
    with torch.no_grad():
        pred = _render(net, opt, data)
    for suffix in ("", "_fine"):
        hit = pred["opacity" + suffix][..., 0] > 0.5
        dot = (pred["normal" + suffix] * pred["viewdirs"]).sum(-1)[hit]
        assert hit.sum() > 100
        assert (dot < 0).float().mean().item() >= 0.99, suffix
