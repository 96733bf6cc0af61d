"""Early ray termination in training steps (ops.mlp_forward_terminated, Graph.set_training_termination) on the device:
the span forward against the rows forward on the same rows moved to row 0; one backward over the rows of several spans
against the rows pair on the concatenated rows; the appending compaction and the segment ray sum against their NumPy
oracles; a training render against the dense render masked by the oracle's kept set (tests/termination_oracle.py, from
the dense noisy σ); eps = 0; a captured step against the eager one; the engine gate; the grid and terminated passes'
in-place parameter gradients against their returned ones; and a graphed training run that converges."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import common
import occupancy_oracle as O
import termination_oracle as T
from test_train_occupancy import KEYS, _bits, _close, _compare, _keep_mask, _net, _p, _random_grid, _stream, _taped_pass

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
DEV = torch.device("cuda")
ENGINES = ["tc_3x", "tc_1x", "tc_3x_w1"]
ALL_KEYS = KEYS + [k + "_fine" for k in KEYS]


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _i64(*v):
    return torch.tensor(v, dtype=torch.int64, device=DEV)


def _span_forward(nerf, engine, C, cap, begin, end, o, d, t, noise, sigma, rgb, tape):
    from sparf_b200 import _lib
    L = _lib.lib()
    m, keep = nerf._spec().fill(nerf.kernel_params(), nerf.progress)
    ws = torch.empty(L.sparf_mlp_workspace_bytes(ctypes.byref(m), cap, 1, 0, engine), dtype=torch.uint8, device=DEV)
    _lib.check(L.sparf_mlp_forward_tape_span(ctypes.byref(m), engine, C, cap, _p(begin), _p(end), _p(o), _p(d), _p(t),
                                             _p(noise), _p(sigma), _p(rgb), _p(tape), tape.numel(), _p(ws), ws.numel(),
                                             _stream()), "mlp_forward_tape_span")


def _inputs(C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    o = torch.randn(C, 3, device=DEV, generator=g) * 0.3
    d = torch.nn.functional.normalize(torch.randn(C, 3, device=DEV, generator=g), dim=-1)
    t = torch.rand(C, 1, device=DEV, generator=g) * 4 + 1
    noise = torch.randn(C, 1, device=DEV, generator=g)
    return o, d, t, noise


# ------------------------------------------------------------------------------------------------ span forward
def _tape_rows(tape, nerf, C):
    """the tape of capacity C (S = 1) as its per-buffer row views, int32 [C, words], in the layout of csrc/mlp.cu
    (tape_layout: encodings, view encodings, colour-head activations, softplus argument, the trunk activations, the
    trunk's ReLU mask bits; each buffer 256-byte aligned)"""
    spec = nerf._spec()
    pad8 = lambda n: (n + 7) // 8 * 8
    widths = [pad8(3 + 6 * spec.L_xyz), pad8(3 + 6 * spec.L_view), spec.head_width, 1] + [spec.width] * spec.n_trunk
    widths += [spec.width // 32] * (spec.n_trunk - 2)          # the fused trunk's mask bits (width 256)
    words = tape.view(torch.int32)
    views, off = [], 0
    for w in widths:
        views.append(words[off:off + C * w].view(C, w))
        off += (C * w * 4 + 255) // 256 * 256 // 4
    assert off * 4 + 256 == tape.numel(), "the tape layout changed"
    return views


def _rows_forward(nerf, engine, n, o, d, t, noise, pattern):
    """forward_tape_rows on rows [0, n) at capacity n into a tape filled with `pattern` -> (sigma, rgb, tape)"""
    from sparf_b200 import _lib
    L = _lib.lib()
    m, keep = nerf._spec().fill(nerf.kernel_params(), nerf.progress)
    tape = torch.empty(L.sparf_mlp_tape_bytes(ctypes.byref(m), engine, n, 1), dtype=torch.uint8, device=DEV)
    tape.view(torch.int32).fill_(pattern)
    ws = torch.empty(L.sparf_mlp_workspace_bytes(ctypes.byref(m), n, 1, 0, engine), dtype=torch.uint8, device=DEV)
    sigma, rgb = torch.empty(n, 1, device=DEV), torch.empty(n, 1, 3, device=DEV)
    rows = _i64(n)
    _lib.check(L.sparf_mlp_forward_tape_rows(ctypes.byref(m), engine, n, 1, _p(rows[0:1]), _p(o), _p(d), _p(t), _p(noise),
                                             _p(sigma), _p(rgb), _p(tape), tape.numel(), _p(ws), ws.numel(), _stream()),
               "mlp_forward_tape_rows")
    return sigma, rgb, tape


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("cap,C,begins,lens", [
    (1024, 131077 + 1024 + 8, (0, 1, 127, 128, 129, 131071, 131077), (0, 1, 128, 1024)),
    (140000, 160008, (20001,), (140000, 131073))])
def test_span_forward_equals_rows_forward(engine, cap, C, begins, lens, engine_guard):
    """rows [b, b + n) of capacity-C buffers, NaN in every other input row, a sentinel in every other output row and a
    byte pattern in the whole tape: σ, rgb and every tape buffer's rows bit-identical to forward_tape_rows on the same
    rows moved to row 0, and every other row of the outputs and of the tape untouched.  The second case's span starts
    at row 20001 and runs past its first 131 072-row chunk, so that its second chunk adds both offsets"""
    from sparf_b200 import _lib
    net, opt, _ = _net()
    eng = _lib.ENGINES[engine]
    L = _lib.lib()
    m, keep = net.nerf._spec().fill(net.nerf.kernel_params(), net.nerf.progress)
    tape = torch.empty(L.sparf_mlp_tape_bytes(ctypes.byref(m), eng, C, 1), dtype=torch.uint8, device=DEV)
    views = _tape_rows(tape, net.nerf, C)
    o, d, t, noise = _inputs(cap, 11)
    sentinel, pattern = -12345.0, 0x5A5A5A5A
    for b in begins:
        for n in lens:
            big = [torch.full((C,) + x.shape[1:], float("nan"), device=DEV) for x in (o, d, t, noise)]
            for x, y in zip(big, (o, d, t, noise)):
                x[b:b + n] = y[:n]
            sigma, rgb = torch.full((C, 1), sentinel, device=DEV), torch.full((C, 1, 3), sentinel, device=DEV)
            tape.view(torch.int32).fill_(pattern)
            _span_forward(net.nerf, eng, C, cap, _i64(b), _i64(b + n), *big, sigma, rgb, tape)
            torch.cuda.synchronize()
            for x in (sigma, rgb):
                assert (x[:b] == sentinel).all() and (x[b + n:] == sentinel).all(), (b, n)
            for i, v in enumerate(views):
                assert (v[:b] == pattern).all() and (v[b + n:] == pattern).all(), (b, n, "tape buffer", i)
            if n == 0:
                continue
            w_sigma, w_rgb, w_tape = _rows_forward(net.nerf, eng, n, o[:n], d[:n], t[:n], noise[:n], pattern)
            torch.cuda.synchronize()
            assert torch.equal(_bits(sigma[b:b + n]), _bits(w_sigma)), (b, n)
            assert torch.equal(_bits(rgb[b:b + n]), _bits(w_rgb)), (b, n)
            for i, (v, w) in enumerate(zip(views, _tape_rows(w_tape, net.nerf, n))):
                assert torch.equal(v[b:b + n], w), (b, n, "tape buffer", i)
            del w_tape


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("R,S,window,lens", [(40, 64, 16, None), (2 * 341, 256, 224, (20000, 150000))])
def test_one_backward_over_appended_spans(engine, R, S, window, lens, engine_guard):
    """W span forwards into one tape, then one backward_tape_rows over rows [0, ends[W]): σ, rgb, per-sample d_o / d_d
    bit-identical to the rows pair on the concatenated rows, parameter gradients within 1e-5 of their max.  The second
    shape (fine pass, 2 x 341 rays x 256 samples, capacity 152 768 per span) has a second span that starts at row 20000
    and holds 150 000 rows: its second chunk runs with both a device start and a chunk offset, and the backward's rows
    cross the 131 072-row chunk boundary"""
    from sparf_b200 import _lib
    net, opt, _ = _net()
    eng = _lib.ENGINES[engine]
    L = _lib.lib()
    C, cap = R * S, R * window
    W = -(-S // window)
    if lens is None:
        lens = [int(x) for x in np.random.default_rng(R + S).integers(0, cap + 1, W)]
        lens[0] = 0                                   # an empty window before full ones
    assert len(lens) == W and max(lens) <= cap and sum(lens) <= C
    ends = _i64(*np.concatenate([[0], np.cumsum(lens)]).tolist())
    K = int(ends[-1])
    o, d, t, noise = _inputs(C, 5)
    gsig, grgb = torch.randn(C, 1, device=DEV), torch.randn(C, 1, 3, device=DEV)
    m, keep = net.nerf._spec().fill(net.nerf.kernel_params(), net.nerf.progress)
    tape = torch.empty(L.sparf_mlp_tape_bytes(ctypes.byref(m), eng, C, 1), dtype=torch.uint8, device=DEV)
    sigma, rgb = torch.zeros(C, 1, device=DEV), torch.zeros(C, 1, 3, device=DEV)
    for w in range(W):
        _span_forward(net.nerf, eng, C, cap, ends[w:w + 1], ends[w + 1:w + 2], o, d, t, noise, sigma, rgb, tape)
    params = net.nerf.kernel_params()
    flat = torch.zeros(sum(p.numel() for p in params), device=DEV)
    grads, off = [], 0
    for p in params:
        grads.append(flat[off:off + p.numel()].view(p.shape))
        off += p.numel()
    gs = net.nerf._spec().grad_struct(grads)
    d_o, d_d = torch.zeros(C, 3, device=DEV), torch.zeros(C, 3, device=DEV)
    ws = torch.empty(L.sparf_mlp_workspace_bytes(ctypes.byref(m), C, 1, 2, eng), dtype=torch.uint8, device=DEV)
    _lib.check(L.sparf_mlp_backward_tape_rows(ctypes.byref(m), eng, C, 1, _p(ends[W:]), _p(o), _p(d), _p(t), _p(sigma),
                                              _p(rgb), _p(gsig), _p(grgb), ctypes.byref(gs), _p(d_o), _p(d_d), _p(tape),
                                              tape.numel(), _p(ws), ws.numel(), _stream()), "backward_tape_rows")
    torch.cuda.synchronize()
    want = _taped_pass(net.nerf, eng, o, d, t, noise, gsig, grgb, K=K)
    for a, b, name in zip((sigma, rgb, d_o, d_d), want[:4], ("sigma", "rgb", "d_o", "d_d")):
        assert torch.equal(_bits(a[:K]), _bits(b[:K])), name
    assert _close(flat, want[4]), (flat - want[4]).abs().max().item()


# ------------------------------------------------------------------------------------------------ movers vs oracles
def _append_all(o, d, t, window, alive_masks, grid):
    """the appending compaction of every window with the given alive masks -> (ends, idx, o_k, d_k, t_k) on the host"""
    from sparf_b200 import ops
    R, S = t.shape
    C = R * S
    W = -(-S // window)
    og, dg, tg = (torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in (o, d, t))
    ends = torch.zeros(W + 1, dtype=torch.int64, device=DEV)
    idx = torch.full((C,), -7, dtype=torch.int64, device=DEV)
    o_k, d_k, t_k = torch.zeros(C, 3, device=DEV), torch.zeros(C, 3, device=DEV), torch.zeros(C, 1, device=DEV)
    for w in range(W):
        alive = torch.from_numpy(alive_masks[w].astype(np.uint8)).to(DEV)
        ops._window_append(grid, og, dg, tg, w * window, min((w + 1) * window, S), alive, ends, w, idx, o_k, d_k, t_k)
    return [x.cpu().numpy() for x in (ends, idx, o_k, d_k, t_k)]


@pytest.mark.parametrize("kind", ["none", "box", "contracted"])
@pytest.mark.parametrize("R,S,window", [(1, 1, 1), (37, 50, 16), (1000, 64, 32)])
def test_append_and_segment_ray_sum_match_oracles(kind, R, S, window):
    """the appended windows equal the concatenation of termination_oracle.compact per window (alive masks: all, then
    random, then none, so that a K = 0 window comes before full ones); the segment ray sum equals the sequential fp32
    oracle"""
    from sparf_b200 import _lib
    from test_train_termination_cpu import append_oracle, segment_ray_sum_oracle
    L = _lib.lib()
    rng = np.random.default_rng(R * 3 + S)
    res = 9
    o = rng.normal(0, 0.4, (R, 3)).astype(np.float32)
    d = rng.normal(0, 1, (R, 3)).astype(np.float32)
    t = np.sort(rng.uniform(0.0, 2.0, (R, S)), 1).astype(np.float32)
    W = -(-S // window)
    masks = [np.ones(R, bool) if w % 3 == 0 else (rng.random(R) < 0.5) if w % 3 == 1 else np.zeros(R, bool)
             for w in range(W)]
    if W > 2:
        masks[0], masks[1] = np.zeros(R, bool), np.ones(R, bool)
    grid, keep = None, None
    if kind != "none":
        contraction = ((0.1, -0.1, 0.2), 0.7) if kind == "contracted" else None
        grid = _random_grid(res, 0.4, R + S, contraction)
        bits = grid.bits.cpu().numpy().view(np.uint32)
        keep = O.kept(bits, res, *grid.range, o, d, t) if contraction is None else None
        if contraction is not None:
            import contraction_oracle as CO
            keep = CO.kept(bits, res, np.asarray(contraction[0], np.float32), np.float32(contraction[1]), o, d, t)
    got = _append_all(o, d, t, window, masks, grid)
    want = append_oracle(o, d, t, window, masks, keep)
    assert got[0].tolist() == want[0].tolist()
    K = int(want[0][-1])
    for g, w_ in zip(got[1:], want[1:]):
        assert g[:K].tobytes() == w_.tobytes()
    assert (got[1][K:] == -7).all()
    src = rng.normal(0, 1, (R * S, 3)).astype(np.float32)
    ends_g, idx_g, src_g = (torch.from_numpy(x).to(DEV) for x in (got[0], got[1], src))
    dst = torch.empty(R, 3, device=DEV)
    _lib.check(L.sparf_compact_ray_sum_segments(R, S, W, _p(ends_g), _p(idx_g), 3, _p(src_g), _p(dst), _stream()),
               "ray_sum_segments")
    assert dst.cpu().numpy().tobytes() == segment_ray_sum_oracle(R, S, got[0], got[1], src).tobytes()


def test_every_ray_dead():
    """alive all zero after the first window: the later windows append nothing and ends stays flat"""
    R, S, window = 64, 40, 8
    rng = np.random.default_rng(1)
    o, d = rng.normal(0, 0.3, (R, 3)).astype(np.float32), rng.normal(0, 1, (R, 3)).astype(np.float32)
    t = np.sort(rng.uniform(0, 3, (R, S)), 1).astype(np.float32)
    masks = [np.ones(R, bool)] + [np.zeros(R, bool)] * 4
    ends = _append_all(o, d, t, window, masks, None)[0]
    assert ends.tolist() == [0] + [R * window] * 5


# ------------------------------------------------------------------------------------------------ renders
def _wall_setup(fine, inverse=False, noise=False, stratified=True):
    from time_termination import camera_normal, scene_graph
    opt = common.make_opt(S=64, S_fine=64, fine=fine, stratified=stratified, noise=noise,
                          depth_param="inverse" if inverse else "metric", depth_range=(1, 0) if inverse else (1.5, 4.5))
    if noise:
        opt.nerf.density_noise_reg = 1.0
    data = common.make_scene(21, 2, 16, 24)
    data.depth_range = torch.tensor([[1.5, 4.5]] * 2)
    for key in ("image", "intr", "pose", "depth_range"):
        data[key] = data[key].to(DEV)
    return scene_graph(opt, ("wall", 0.0, 400.0), camera_normal(data.pose)), opt, data


def _step(net, opt, data, pose, seed, fine):
    Hh, Ww = data.image.shape[-2:]
    torch.manual_seed(seed)
    out = net.render(opt, pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device=DEV),
                     depth_range=net._depth_range(opt, data), iter=10, mode="train")
    target = data.image.flatten(2).transpose(1, 2)
    loss = ((out["rgb"] - target) ** 2).mean()
    if fine:
        loss = loss + ((out["rgb_fine"] - target) ** 2).mean()
    params = [p for m in net.get_network_components() for p in m.kernel_params()]
    return out, loss, torch.autograd.grad(loss, params + [pose])


def _masked_reference(net, grids, eps, window):
    """nerf.forward_samples replaced by the dense pass masked with the oracle's kept set from its own (noisy) σ"""
    for nerf, g in zip(net.get_network_components(), grids):
        dense_fs = nerf.forward_samples

        def masked(opt_, center, ray, depth_samples, _f=dense_fs, _g=g, **kw):
            out = _f(opt_, center, ray, depth_samples, **kw)
            B, N, S = depth_samples.shape[:3]
            keep = None if _g is None else _keep_mask(_g, center, ray, depth_samples).reshape(B * N, S).cpu().numpy()
            ev = T.evaluated(out["density_samples"].detach().reshape(B * N, S).cpu().numpy(),
                             depth_samples.reshape(B * N, S).cpu().numpy(), ray.reshape(-1, 3).detach().cpu().numpy(),
                             eps, window, keep)
            m = torch.from_numpy(ev).to(DEV).float().view(B, N, S)
            return dict(density_samples=out["density_samples"] * m, rgb_samples=out["rgb_samples"] * m[..., None])
        nerf.forward_samples = masked


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("fine,grid_kind,noise,eps,window", [
    (False, None, False, 1e-4, 16), (False, None, True, 1e-2, 1), (False, "box", True, 1e-4, 64),
    (True, None, True, 1e-4, 16), (True, "box", False, 1e-2, 16), (True, "contracted", True, 1e-4, 16),
    (True, None, False, 1e-2, 64)])
def test_training_render_equals_masked_dense(engine, fine, grid_kind, noise, eps, window, engine_guard):
    """the training render with termination (and a grid) equals the dense render masked by the oracle's kept set, bit
    for bit; network and pose gradients within 1e-5 of their max; rays really terminate"""
    import sparf_b200
    sparf_b200.set_engine(engine)
    net, opt, data = _wall_setup(fine, noise=noise)
    contraction = ((0.0, 0.0, 0.0), 1.0) if grid_kind == "contracted" else None
    grids = (None, None)
    if grid_kind:
        grids = (_random_grid(16, 0.6, 1, contraction), _random_grid(12, 0.7, 2, contraction))
        net.set_training_occupancy(*grids)
    pose = data.pose.clone().requires_grad_()
    net.set_training_termination(eps, window)
    sparse = _step(net, opt, data, pose, 7, fine)
    net.set_training_termination(None)
    net.set_training_occupancy(None)
    _masked_reference(net, grids, eps, window)
    ref = _step(net, opt, data, pose, 7, fine)
    kept = (sparse[0]["density_samples"] != 0).float().mean().item()
    worst = _compare(sparse, ref, ALL_KEYS if fine else KEYS)
    print("fine=%d grid=%s noise=%d eps=%g window=%d: kept %.3f, worst gradient %.2e of max"
          % (fine, grid_kind, noise, eps, window, kept, worst))
    assert kept < 0.9


def test_inverse_depth_wall_with_contracted_grid(engine_guard):
    """coarse only, inverse depth, an all-occupied contracted grid: the masked-dense equality, with termination"""
    from sparf_b200.occupancy import OccupancyGrid
    net, opt, data = _wall_setup(False, inverse=True)
    full = OccupancyGrid(torch.full(((16 ** 3 + 31) // 32,), -1, dtype=torch.int32, device=DEV), 16, (-2.0, 2.0), 0.01,
                         ((0.0, 0.0, 0.0), 1.33))
    net.set_training_occupancy(full)
    net.set_training_termination(1e-4, 16)
    pose = data.pose.clone().requires_grad_()
    sparse = _step(net, opt, data, pose, 3, False)
    net.set_training_termination(None)
    net.set_training_occupancy(None)
    _masked_reference(net, (full, None), 1e-4, 16)
    ref = _step(net, opt, data, pose, 3, False)
    _compare(sparse, ref, KEYS)
    assert (sparse[0]["density_samples"] != 0).float().mean().item() < 0.9


@pytest.mark.parametrize("with_grid", [False, True])
def test_eps_zero_changes_nothing(with_grid, engine_guard):
    """eps = 0 terminates nothing: the outputs are those of the grid training path (with a grid) or of the dense
    training render (without one), bit for bit"""
    net, opt, data = _wall_setup(True, noise=True)
    grids = (_random_grid(16, 0.6, 1), _random_grid(12, 0.7, 2)) if with_grid else (None, None)
    net.set_training_occupancy(*grids)
    pose = data.pose.clone().requires_grad_()
    base = _step(net, opt, data, pose, 5, True)
    net.set_training_termination(0.0, 16)
    term = _step(net, opt, data, pose, 5, True)
    for k in ALL_KEYS:
        assert torch.equal(_bits(term[0][k].reshape(-1)), _bits(base[0][k].reshape(-1))), k
    _compare(term, base, ALL_KEYS)


def test_detach_restores_and_simt_refused(engine_guard):
    """set_training_termination(None) gives today's outputs bit for bit; simt_fp32 raises before any work"""
    import sparf_b200
    from sparf_b200 import _lib, ops
    net, opt, data = _wall_setup(True, noise=True)
    pose = data.pose.clone().requires_grad_()
    base = _step(net, opt, data, pose, 9, True)
    net.set_training_termination(1e-4, 16)
    _step(net, opt, data, pose, 9, True)
    net.set_training_termination(None)
    again = _step(net, opt, data, pose, 9, True)
    for k in ALL_KEYS:
        assert torch.equal(_bits(again[0][k].reshape(-1)), _bits(base[0][k].reshape(-1))), k
    o, d, t = torch.zeros(4, 3, device=DEV), torch.ones(4, 3, device=DEV), torch.ones(4, 8, device=DEV)
    n0 = _lib.lib().sparf_launch_count()
    with pytest.raises(ValueError, match="simt_fp32"):
        ops.mlp_forward_terminated(net.nerf._spec(), o, d, t, None, 1e-4, 4, net.nerf.kernel_params(),
                                   engine=_lib.ENGINE_SIMT_FP32)
    assert _lib.lib().sparf_launch_count() == n0
    sparf_b200.set_engine("simt_fp32")
    net.set_training_termination(1e-4, 16)
    with pytest.raises(ValueError, match="simt_fp32"):
        _step(net, opt, data, pose, 9, True)


def test_captured_step_equals_eager(engine_guard):
    """a whole step (render -> loss -> backward) with training grids and termination, captured by GraphedStep and
    replayed after occupancy.refresh_ rewrote the grids in place, equals the eager step, which never synchronises"""
    from sparf_b200 import occupancy
    from sparf_b200.graphs import GraphedStep
    net, opt, data = _wall_setup(True, stratified=False)     # nothing random: replay and eager see the same samples
    grids = [_random_grid(16, 0.6, 10 + i) for i in range(2)]
    for g in grids:
        g.thres = 0.5
    net.set_training_occupancy(*grids)
    net.set_training_termination(1e-4, 16)
    pose = data.pose.clone().requires_grad_()

    def fn():
        out, loss, grads = _step(net, opt, data, pose, 0, True)
        return (loss.detach(), out["density_samples"].detach()) + tuple(grads)

    step = GraphedStep(fn, (), warmup=2)
    before = [g.bits.clone() for g in grids]
    for g, nerf in zip(grids, net.get_network_components()):
        occupancy.refresh_(g, opt, nerf)
    assert any(not torch.equal(a, g.bits) for a, g in zip(before, grids))
    replay = [x.clone() for x in step()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = fn()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(_bits(replay[0]), _bits(eager[0]))
    assert torch.equal(_bits(replay[1]), _bits(eager[1]))
    assert (replay[1] != 0).float().mean().item() < 0.9
    for x, y in zip(replay[2:], eager[2:]):
        assert (x - y).abs().max().item() <= 1e-5 * y.abs().max().item() + 1e-12


def test_captured_sparf_step_equals_eager(engine_guard, monkeypatch):
    """the full SPARF step of tests/test_losses.py (photometric + correspondence + depth-consistency in device-side mode,
    six render calls, gradients to both networks and the poses) with training grids on both networks and termination:
    captured by GraphedStep and replayed after occupancy.refresh_ rewrote the grids in place, it equals the eager step,
    which runs under set_sync_debug_mode("error") and goes through the terminated pass on every render.  The losses'
    random draws are drawn once beforehand and the depth samples are deterministic, so that replay and eager step see
    the same inputs."""
    from sparf_b200 import mesh, occupancy, ops
    from sparf_b200.distributed import FlatGradients
    from sparf_b200.graphs import GraphedStep
    from sparf_b200.losses import define_loss
    from test_losses import _TrainData, _sparf_problem, _sparf_step
    c, opt, data, ray_idx, net, pose_net = _sparf_problem(DEV, stratified=False)
    opt.nerf.density_noise_reg = 0.0
    flow = common.FakeFlowNet(c["B"], c["H"], c["W"])
    loss_module = define_loss(opt.loss_type, opt, net, _TrainData(data, c["B"]), DEV, flow_net=flow, device_side=True)
    corres_mod, dc_mod = loss_module.loss_modules[1], loss_module.loss_modules[2]
    g = torch.Generator(device=DEV).manual_seed(3)
    pair = torch.zeros(1, dtype=torch.int64, device=DEV)
    keys = torch.rand(c["H"] * c["W"], device=DEV, generator=g)
    image = torch.ones(1, dtype=torch.int64, device=DEV)
    weight = torch.full((), 0.3, device=DEV)
    torch.manual_seed(5)
    px = dc_mod._rand_pixels(c["H"], c["W"], max(1024, opt.nerf.rand_rays)).clone()
    corres_mod._rand_pair = lambda: pair
    corres_mod._rand_keys = lambda n: keys
    dc_mod._rand_image = lambda B: image
    dc_mod._rand_weight = lambda: weight
    dc_mod._rand_pixels = lambda H_, W_, n: px
    grids = []
    for i, nerf in enumerate(net.get_network_components()):
        grid = _random_grid(16, 0.6, 20 + i)
        grid.thres = float(torch.quantile(mesh.density_grid(opt, nerf, res=16, range=(-1.2, 1.2)).flatten(), 0.5))
        grids.append(grid)
    net.set_training_occupancy(*grids)
    net.set_training_termination(1e-4, 16)
    fg = FlatGradients([net, pose_net])
    calls = [0]
    terminated = ops.mlp_forward_terminated

    def counted(*a, **k):
        calls[0] += 1
        return terminated(*a, **k)
    monkeypatch.setattr(ops, "mlp_forward_terminated", counted)

    def step(idx):
        fg.zero_()
        loss = _sparf_step(c, opt, data, idx, net, loss_module)
        return loss["all"].detach(), loss["corres"].detach(), loss["depth_cons"].detach()

    graphed = GraphedStep(step, (ray_idx.clone(),), warmup=2)
    before = [grid.bits.clone() for grid in grids]
    for grid, nerf in zip(grids, net.get_network_components()):
        occupancy.refresh_(grid, opt, nerf)
    assert any(not torch.equal(a, grid.bits) for a, grid in zip(before, grids))
    replay = [x.clone() for x in graphed(ray_idx)]
    replay_grad = fg.flat.clone()
    torch.cuda.synchronize()
    calls[0] = 0
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = step(ray_idx)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert calls[0] >= 6, calls[0]
    for a, b in zip(replay, eager):
        assert torch.isfinite(b) and torch.equal(_bits(a), _bits(b)), (a.item(), b.item())
    assert fg.flat.abs().sum() > 0
    err, scale = (replay_grad - fg.flat).abs().max().item(), fg.flat.abs().max().item()
    print("SPARF step with grids and termination: %d terminated passes, losses %s, gradient difference %.2e of max"
          % (calls[0], [float(x) for x in eager], err / scale))
    assert err <= 1e-5 * scale


@pytest.mark.parametrize("kind", ["grid", "terminated"])
def test_inplace_param_grads_equal_returned(kind):
    """the grid and the terminated pass accumulating into the parameters' own .grad (FlatGradients marks them
    _sparf_inplace_grad) give the parameter gradients they return otherwise, bit for bit, and return None for them.
    64 samples fit one row tile, so no gradient element is summed by two CTAs and the bits do not depend on the order of
    the atomic adds"""
    from sparf_b200 import ops
    net, opt, _ = _net()
    nerf = net.nerf
    params = nerf.kernel_params()
    R, S = 4, 16
    g = torch.Generator(device=DEV).manual_seed(13)
    o = torch.randn(R, 3, device=DEV, generator=g) * 0.3
    d = torch.nn.functional.normalize(torch.randn(R, 3, device=DEV, generator=g), dim=-1)
    t = torch.sort(torch.rand(R, S, device=DEV, generator=g) + 0.1, 1).values
    w_sigma, w_rgb = torch.randn(R, S, device=DEV, generator=g), torch.randn(R, S, 3, device=DEV, generator=g)
    grid = _random_grid(16, 0.6, 4)

    def loss():
        if kind == "grid":
            sigma, rgb = ops.mlp_forward_grid(nerf._spec(), o, d, t, grid, params, progress=nerf.progress)
        else:
            sigma, rgb = ops.mlp_forward_terminated(nerf._spec(), o, d, t, grid, 1e-2, 4, params, progress=nerf.progress)
        assert 0 < (sigma != 0).sum().item() < R * S
        return (sigma * w_sigma).sum() + (rgb * w_rgb).sum()

    returned = torch.autograd.grad(loss(), params)
    for p in params:
        p._sparf_inplace_grad = True
        p.grad = torch.zeros_like(p)
    assert all(x is None for x in torch.autograd.grad(loss(), params, allow_unused=True))
    assert max(x.abs().max().item() for x in returned) > 0
    for p, x in zip(params, returned):
        assert torch.equal(_bits(p.grad), _bits(x))


def test_graphed_training_with_termination_converges(engine_guard):
    """train_synthetic with a grid and termination: the bounds of test_training_loop_converges"""
    import sparf_b200
    import train_synthetic
    for fine, poses in ((0, 0), (1, 0), (0, 1)):
        try:
            res = train_synthetic.main(["--steps", "300", "--quiet", "--fine", str(fine), "--poses", str(poses), "--rays", "768",
                                        "--grid", "64", "--grid-every", "16", "--grid-thres", "0.5", "--term", "1e-4"])
        finally:
            sparf_b200.set_engine("auto")
        first, last, kept = res[0], res[1], res[-1]
        print("fine=%d poses=%d: loss %.5f -> %.5f, kept fraction %.3f" % (fine, poses, first, last, kept))
        assert last == last and first == first
        assert last < (0.85 if poses else 0.6) * first, (first, last)
        assert kept < 1.0
