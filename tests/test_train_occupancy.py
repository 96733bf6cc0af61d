"""Occupancy grids in training steps (ops.mlp_forward_grid, Graph.set_training_occupancy, occupancy.refresh_) on the
device: the taped MLP pair with a device row count against the taped pair at R = K; a training render with a grid
against the dense render with σ and rgb zeroed at the skipped samples, forward bit for bit and gradients to rounding; an
all-occupied grid against the dense training render; a captured step across an in-place refresh against the eager step,
with no synchronisation; and a graphed training run that converges with a grid."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import common
import occupancy_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda")


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _bits(x):
    return x.detach().contiguous().view(torch.int32)


def _p(x):
    return ctypes.c_void_p(0 if x is None else x.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _net(seed=5, noise=False, stratified=True, S=64):
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=S, S_fine=S, fine=True, stratified=stratified, noise=noise, depth_range=(1.2, 5.2))
    net = Graph(opt, DEV)
    net.nerf.load_state_dict(common.det_weights(opt, seed, peaky=True, sigma_bias=-2.0))
    net.nerf_fine.load_state_dict(common.det_weights(opt, seed + 1, peaky=True, sigma_bias=-2.0))
    data = common.make_scene(seed, 2, 16, 24)
    data.depth_range = torch.tensor([[1.2, 5.2]] * 2)
    for k in ("image", "intr", "pose", "depth_range"):
        data[k] = data[k].to(DEV)
    return net, opt, data


def _random_grid(res, p, seed, contraction=None):
    from sparf_b200.occupancy import CONTRACTED_RANGE, OccupancyGrid
    occ = np.random.default_rng(seed).random((res,) * 3) < p
    bits = torch.from_numpy(O.pack_bits(occ).view(np.int32).copy()).to(DEV)
    return OccupancyGrid(bits, res, CONTRACTED_RANGE if contraction else (-1.2, 1.2), 0.01, contraction)


# ------------------------------------------------------------------------------------------------ engine contract
def _taped_pass(nerf, engine, o, d, t, noise, g_sigma, g_rgb, K=None, sentinel=None):
    """forward + backward of the taped pair (K None: R = rows of o) or of the *_rows pair with *rows = K at the capacity
    of o; outputs pre-filled with `sentinel` where given -> sigma, rgb, d_o, d_d, flat parameter gradient"""
    from sparf_b200 import _lib
    L = _lib.lib()
    spec, params = nerf._spec(), nerf.kernel_params()
    m, keep = spec.fill(params, nerf.progress)
    R = o.shape[0]
    fill = (lambda *s: torch.full(s, sentinel, device=DEV)) if sentinel is not None else (lambda *s: torch.zeros(*s, device=DEV))
    sigma, rgb, d_o, d_d = fill(R, 1), fill(R, 1, 3), fill(R, 3), fill(R, 3)
    if sentinel is not None:      # the rows the call owns start at 0 (the backward accumulates)
        k = int(K)
        d_o[:k], d_d[:k] = 0, 0
    flat = torch.zeros(sum(p.numel() for p in params), device=DEV)
    grads, off = [], 0
    for p in params:
        grads.append(flat[off:off + p.numel()].view(p.shape))
        off += p.numel()
    gs = spec.grad_struct(grads)
    tape_bytes = L.sparf_mlp_tape_bytes(ctypes.byref(m), engine, R, 1)
    tape = torch.empty(tape_bytes, dtype=torch.uint8, device=DEV)
    wsb = max(L.sparf_mlp_workspace_bytes(ctypes.byref(m), R, 1, b, engine) for b in (0, 2))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    if K is None:
        _lib.check(L.sparf_mlp_forward_tape(ctypes.byref(m), engine, R, 1, _p(o), _p(d), _p(t), _p(noise), _p(sigma), _p(rgb),
                                            _p(tape), tape_bytes, _p(ws), wsb, _stream()), "forward_tape")
        _lib.check(L.sparf_mlp_backward_tape(ctypes.byref(m), engine, R, 1, _p(o), _p(d), _p(t), _p(sigma), _p(rgb),
                                             _p(g_sigma), _p(g_rgb), ctypes.byref(gs), _p(d_o), _p(d_d), _p(tape), tape_bytes,
                                             _p(ws), wsb, _stream()), "backward_tape")
    else:
        rows = torch.tensor(int(K), dtype=torch.int64, device=DEV)
        _lib.check(L.sparf_mlp_forward_tape_rows(ctypes.byref(m), engine, R, 1, _p(rows), _p(o), _p(d), _p(t), _p(noise),
                                                 _p(sigma), _p(rgb), _p(tape), tape_bytes, _p(ws), wsb, _stream()),
                   "forward_tape_rows")
        _lib.check(L.sparf_mlp_backward_tape_rows(ctypes.byref(m), engine, R, 1, _p(rows), _p(o), _p(d), _p(t), _p(sigma),
                                                  _p(rgb), _p(g_sigma), _p(g_rgb), ctypes.byref(gs), _p(d_o), _p(d_d), _p(tape),
                                                  tape_bytes, _p(ws), wsb, _stream()), "backward_tape_rows")
    torch.cuda.synchronize()
    return sigma, rgb, d_o, d_d, flat


def _close(a, b, rel=1e-5):
    return (a - b).abs().max().item() <= rel * max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("engine", ["tc_3x", "tc_1x", "tc_3x_w1"])
@pytest.mark.parametrize("C,Ks", [(1000, (0, 1, 127, 128, 129, 1000)), (131072 + 4096, (131072 + 300, 131072 - 1))])
def test_rows_pair_equals_taped_pair_at_K(engine, C, Ks, engine_guard):
    """capacity C, *rows = K: σ, rgb, d_o, d_d bit-identical to the taped pair at R = K on rows [0, K); pad input rows
    (NaN) never read and pad output rows (sentinel) never written; parameter gradients equal up to atomic order"""
    from sparf_b200 import _lib
    net, opt, _ = _net()
    eng = _lib.ENGINES[engine]
    g = torch.Generator(device=DEV).manual_seed(C)
    o = torch.randn(C, 3, device=DEV, generator=g) * 0.3
    d = torch.nn.functional.normalize(torch.randn(C, 3, device=DEV, generator=g), dim=-1)
    t = torch.rand(C, 1, device=DEV, generator=g) * 4 + 1
    noise = torch.randn(C, 1, device=DEV, generator=g)
    gsig, grgb = torch.randn(C, 1, device=DEV, generator=g), torch.randn(C, 1, 3, device=DEV, generator=g)
    sentinel = -12345.0
    for K in Ks:
        pad = lambda x: torch.cat([x[:K], torch.full_like(x[K:], float("nan"))])
        got = _taped_pass(net.nerf, eng, pad(o), pad(d), pad(t), pad(noise), pad(gsig), pad(grgb), K=K, sentinel=sentinel)
        for x in got[:4]:
            assert (x[K:] == sentinel).all(), K
        if K == 0:
            assert (got[4] == 0).all()
            continue
        want = _taped_pass(net.nerf, eng, o[:K], d[:K], t[:K], noise[:K], gsig[:K], grgb[:K])
        for a, b, name in zip(got[:4], want[:4], ("sigma", "rgb", "d_o", "d_d")):
            assert torch.equal(_bits(a[:K]), _bits(b)), (K, name)
        assert _close(got[4], want[4]), (K, (got[4] - want[4]).abs().max().item())


def test_simt_engine_is_refused():
    from sparf_b200 import _lib, ops
    net, opt, _ = _net()
    o, d, t = torch.zeros(4, 3, device=DEV), torch.ones(4, 3, device=DEV), torch.ones(4, 8, device=DEV)
    with pytest.raises(ValueError, match="simt_fp32"):
        ops.mlp_forward_grid(net.nerf._spec(), o, d, t, _random_grid(4, 1.0, 0), net.nerf.kernel_params(),
                             engine=_lib.ENGINE_SIMT_FP32)
    L = _lib.lib()
    m, keep = net.nerf._spec().fill(net.nerf.kernel_params(), net.nerf.progress)
    rows = torch.tensor(4, dtype=torch.int64, device=DEV)
    out = torch.empty(4, device=DEV)
    rc = L.sparf_mlp_forward_tape_rows(ctypes.byref(m), _lib.ENGINE_SIMT_FP32, 4, 1, _p(rows), _p(o), _p(d), _p(t), None,
                                       _p(out), _p(out), _p(out), 1 << 20, _p(out), 1 << 20, _stream())
    assert rc != 0 and b"tensor-core" in L.sparf_last_error()


# ------------------------------------------------------------------------------------------------ renders
def _keep_mask(grid, center, ray, depth_samples):
    from sparf_b200 import ops
    B, N, S = depth_samples.shape[:3]
    o, d, t = center.reshape(-1, 3), ray.reshape(-1, 3), depth_samples.reshape(B * N, S)
    if grid.contraction is None:
        idx = ops.occupancy_compact(grid.bits, grid.res, grid.range, o, d, t)[0]
    else:
        idx = ops.contracted_compact(o, d, t, 0, S, None, grid.bits, grid.res, *grid.contraction)[0]
    keep = torch.zeros(B * N * S, dtype=torch.bool, device=DEV)
    keep[idx] = True
    return keep.view(B, N, S)


def _step(net, opt, data, pose, seed):
    """one training render of every pixel at `pose` and a photometric loss -> (outputs, loss, gradients of the network
    parameters and of the pose)"""
    Hh, Ww = data.image.shape[-2:]
    torch.manual_seed(seed)
    out = net.render(opt, pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device=DEV),
                     depth_range=net._depth_range(opt, data), iter=10, mode="train")
    target = data.image.flatten(2).transpose(1, 2)
    loss = ((out["rgb"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean()
    params = [p for m in net.get_network_components() for p in m.kernel_params()]
    grads = torch.autograd.grad(loss, params + [pose])
    return out, loss, grads


KEYS = ["rgb", "depth", "opacity", "weights", "density_samples", "rgb_samples", "t"]


def _compare(a, b, exact_keys, tol=1e-5):
    out_a, loss_a, g_a = a
    out_b, loss_b, g_b = b
    for k in exact_keys:
        assert torch.equal(_bits(out_a[k].reshape(-1)), _bits(out_b[k].reshape(-1))), k
    assert torch.equal(_bits(loss_a), _bits(loss_b))
    worst = 0.0
    for x, y in zip(g_a, g_b):
        scale = y.abs().max().item()
        err = (x - y).abs().max().item()
        worst = max(worst, err / max(scale, 1e-30))
        assert err <= tol * scale + 1e-12, (err, scale)
    return worst


@pytest.mark.parametrize("kind", ["box", "contracted"])
@pytest.mark.parametrize("noise", [False, True])
def test_training_render_equals_masked_dense(kind, noise, engine_guard):
    """grids on the coarse and the fine pass: the outputs are those of the dense training render with σ and rgb
    multiplied by the kept mask, bit for bit (same stratified offsets and density noise); the network and pose gradients
    of a photometric loss agree to 1e-5 of their max"""
    net, opt, data = _net(noise=noise)
    if noise:
        opt.nerf.density_noise_reg = 1.0
    contraction = ((0.0, 0.0, 0.0), 1.0) if kind == "contracted" else None
    grids = (_random_grid(16, 0.4, 1, contraction), _random_grid(12, 0.5, 2, contraction))
    pose = data.pose.clone().requires_grad_()

    net.set_training_occupancy(*grids)
    sparse = _step(net, opt, data, pose, 7)
    net.set_training_occupancy(None)
    for nerf, g in zip(net.get_network_components(), grids):     # the reference: the dense pass, masked
        dense_fs = nerf.forward_samples

        def masked(opt_, center, ray, depth_samples, _f=dense_fs, _g=g, **kw):
            out = _f(opt_, center, ray, depth_samples, **kw)
            keep = _keep_mask(_g, center, ray, depth_samples).float()
            return dict(density_samples=out["density_samples"] * keep, rgb_samples=out["rgb_samples"] * keep[..., None])
        nerf.forward_samples = masked
    ref = _step(net, opt, data, pose, 7)
    kept = (sparse[0]["density_samples"] != 0).float().mean().item()
    worst = _compare(sparse, ref, KEYS + [k + "_fine" for k in KEYS])
    print("%s noise=%d: kept %.3f, worst gradient difference %.2e of max" % (kind, noise, kept, worst))
    assert 0.05 < kept < 0.95


def test_all_occupied_grid_in_train_mode(engine_guard):
    """every cell occupied: the training render is the dense one bit for bit, its gradients agree to 1e-5 of max"""
    from sparf_b200.occupancy import OccupancyGrid
    net, opt, data = _net(noise=True)
    opt.nerf.density_noise_reg = 1.0
    full = OccupancyGrid(torch.full(((16 ** 3 + 31) // 32,), -1, dtype=torch.int32, device=DEV), 16, (-1.2, 1.2), 0.01)
    pose = data.pose.clone().requires_grad_()
    dense = _step(net, opt, data, pose, 3)
    net.set_training_occupancy(full, full)
    sparse = _step(net, opt, data, pose, 3)
    _compare(sparse, dense, KEYS + [k + "_fine" for k in KEYS])


def test_captured_step_across_refresh_equals_eager(engine_guard):
    """a whole step (render -> loss -> backward) with grids, captured by GraphedStep and replayed after occupancy.refresh_
    rewrote the grids in place, equals the eager step; and the eager step never synchronises"""
    from sparf_b200 import mesh, occupancy
    from sparf_b200.graphs import GraphedStep
    net, opt, data = _net(stratified=False)
    grids = []
    for i, nerf in enumerate(net.get_network_components()):
        g = _random_grid(16, 0.5, 10 + i)
        g.thres = float(torch.quantile(mesh.density_grid(opt, nerf, res=16, range=(-1.2, 1.2)).flatten(), 0.995))
        grids.append(g)
    net.set_training_occupancy(*grids)
    pose = data.pose.clone().requires_grad_()

    def fn():
        out, loss, grads = _step(net, opt, data, pose, 0)
        return (loss.detach(),) + tuple(grads)

    step = GraphedStep(fn, (), warmup=2)
    before = [g.bits.clone() for g in grids]
    for g, nerf in zip(grids, net.get_network_components()):
        occupancy.refresh_(g, opt, nerf)
    assert any(not torch.equal(a, g.bits) for a, g in zip(before, grids))
    assert any(g.occupied_fraction() < 1 for g in grids)
    replay = [x.clone() for x in step()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = fn()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(_bits(replay[0]), _bits(eager[0]))
    for x, y in zip(replay[1:], eager[1:]):
        assert (x - y).abs().max().item() <= 1e-5 * y.abs().max().item() + 1e-12


def test_graphed_training_with_grid_converges(engine_guard):
    """train_synthetic with a grid refreshed every 16 steps: the bounds of test_training_loop_converges, and the grid
    ends up skipping samples (at thres 0.5: the teacher's empty space has σ = softplus(-2) = 0.13, above the default
    0.01)"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sparf_b200
    import train_synthetic
    for fine, poses in ((0, 0), (1, 0), (0, 1)):
        try:
            res = train_synthetic.main(["--steps", "300", "--quiet", "--fine", str(fine), "--poses", str(poses), "--rays", "768",
                                        "--grid", "64", "--grid-every", "16", "--grid-thres", "0.5"])
        finally:
            sparf_b200.set_engine("auto")
        first, last, kept = res[0], res[1], res[-1]
        print("fine=%d poses=%d: loss %.5f -> %.5f, kept fraction %.3f" % (fine, poses, first, last, kept))
        assert last == last and first == first
        assert last < (0.85 if poses else 0.6) * first, (first, last)
        assert kept < 1.0
