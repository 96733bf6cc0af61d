"""The occupancy grid update (ops.occupancy_sample, ops.occupancy_ema_, occupancy.update_, build_grid(ema=True)) on the
device: the sampled cells and points and the density EMA against the NumPy oracle bit for bit, update_ end to end
against the oracle EMA of the density query at the oracle's points, the initial density, no synchronisation, a
captured training step with the update against the eager sequence, and a graphed training run that converges with
grids updated inside the step."""
import os
import sys

import numpy as np
import pytest
import torch

import common
import contraction_oracle as C
import grid_update_oracle as G
import occupancy_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda")
CONTRACTION = ((0.25, -0.5, 0.125), 1.5)
BOX = (-1.3, 0.7)


@pytest.fixture
def engine_guard():
    from sparf_b200 import ops
    prev = ops.get_engine()
    yield
    ops.set_engine(prev)


def _bits_tensor(occ):
    return torch.from_numpy(O.pack_bits(occ).view(np.int32).copy()).to(DEV)


def _occupancy(res, contracted, kind, rng):
    """bool [res]^3 with none, exactly one, about 30 % or all interior cells occupied (the shell of a contracted grid
    set, as the build leaves it)"""
    inner = G.interior(res, contracted)
    occ = np.zeros(res ** 3, bool)
    if kind == "one":
        occ[rng.choice(np.nonzero(inner)[0])] = True
    elif kind == "p30":
        occ = rng.random(res ** 3) < 0.3
    elif kind == "all":
        occ[:] = True
    return (occ | ~inner).reshape(res, res, res)


def _draws(n, rng):
    u_cell = rng.random(n, dtype=np.float32)
    u_jit = rng.random((n, 3), dtype=np.float32)
    edge = np.array([0.0, 1 - 2 ** -24], np.float32)
    u_cell[:4] = np.tile(edge, 2)
    u_cell[n // 2:n // 2 + 4] = np.tile(edge, 2)
    u_jit[:2] = edge[:, None]
    u_jit[n // 2:n // 2 + 2] = edge[:, None]
    return u_cell, u_jit


@pytest.mark.parametrize("occupied", ["none", "one", "p30", "all"])
@pytest.mark.parametrize("res", [8, 33, 128])
@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_sample_matches_oracle(kind, res, occupied):
    from sparf_b200 import ops
    rng = np.random.default_rng(res * 7 + len(occupied))
    contraction = CONTRACTION if kind == "contracted" else None
    occ = _occupancy(res, contraction is not None, occupied, rng)
    bits = O.pack_bits(occ)
    for n_u, n_o in ((1500, 1500), (0, 2000), (2000, 0)):
        u_cell, u_jit = _draws(n_u + n_o, rng)
        cells, pts = ops.occupancy_sample(_bits_tensor(occ), res, BOX, contraction, n_u, n_o,
                                          torch.from_numpy(u_cell).to(DEV), torch.from_numpy(u_jit).to(DEV))
        want_cells, want_pts = G.sample(bits, res, *BOX, contraction, n_u, n_o, u_cell, u_jit)
        assert np.array_equal(cells.cpu().numpy(), want_cells), (n_u, n_o)
        assert np.array_equal(pts.cpu().numpy().view(np.int32), want_pts.view(np.int32)), (n_u, n_o)
        if contraction is not None:     # each point's lookup: its drawn cell, or the neighbour across a face it lies on
            p = pts.cpu().numpy()
            u = C.contract_u(p, np.zeros_like(p), np.zeros((len(p), 1), np.float32), *contraction, res)[:, 0]
            got = np.floor(u).astype(np.int64)
            want = np.stack([want_cells // (res * res), want_cells // res % res, want_cells % res], -1)
            off = np.abs(got - want)
            at_face = (u_jit < 1e-4) | (u_jit > 1 - 1e-4)
            assert off.max() <= 1 and not (off.astype(bool) & ~at_face).any()
            assert (off.sum(-1) == 0).mean() > 0.9


@pytest.mark.parametrize("decay", [1.0, 0.95])
@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_ema_matches_oracle(kind, decay):
    from sparf_b200 import ops
    res = 33
    contracted = kind == "contracted"
    rng = np.random.default_rng(3)
    density = (rng.random(res ** 3, dtype=np.float32) * 2).astype(np.float32)
    density[rng.integers(0, res ** 3, 50)] = G.FLT_MAX
    inner = np.nonzero(G.interior(res, contracted))[0]
    n = 20000
    cells = inner[rng.integers(0, inner.size, n)]
    cells[n // 2:n // 2 + 500] = cells[:500]                    # repeated cells
    sigma = (rng.random(n, dtype=np.float32) * 3).astype(np.float32)
    sigma[rng.integers(0, n, 40)] = np.nan
    sigma[rng.integers(0, n, 40)] = np.inf
    thres = 0.8
    d = torch.from_numpy(density).to(DEV)
    bits = torch.zeros((res ** 3 + 31) // 32, dtype=torch.int32, device=DEV)
    ops.occupancy_ema_(d, bits, res, contracted, torch.from_numpy(cells).to(DEV), torch.from_numpy(sigma).to(DEV),
                       decay, thres)
    want_d, want_bits = G.ema(density, res, contracted, cells, sigma, decay, thres)
    got_d = d.cpu().numpy()
    assert np.array_equal(got_d.view(np.int32), want_d.view(np.int32))
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), want_bits)
    if contracted:
        shell = C.shell(res).reshape(-1)
        assert np.array_equal(got_d[shell].view(np.int32), density[shell].view(np.int32))
        assert O.unpack_bits(bits.cpu().numpy(), res).reshape(-1)[shell].all()
    assert 0 < O.unpack_bits(bits.cpu().numpy(), res).mean() < 1


def _net(seed=5, S=64):
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=S, S_fine=S, fine=True, depth_range=(1.2, 5.2))
    net = Graph(opt, DEV)
    net.nerf.load_state_dict(common.det_weights(opt, seed, peaky=True, sigma_bias=-2.0))
    net.nerf_fine.load_state_dict(common.det_weights(opt, seed + 1, peaky=True, sigma_bias=-2.0))
    data = common.make_scene(seed, 2, 16, 24)
    data.depth_range = torch.tensor([[1.2, 5.2]] * 2)
    for k in ("image", "intr", "pose", "depth_range"):
        data[k] = data[k].to(DEV)
    return net, opt, data


def _build(opt, nerf, kind, res, thres, ema=True):
    from sparf_b200 import occupancy
    if kind == "box":
        return occupancy.build_grid(opt, nerf, res=res, range=(-1.2, 1.2), thres=thres, ema=ema)
    return occupancy.build_grid(opt, nerf, res=res, thres=thres, contraction=CONTRACTION, ema=ema)


@pytest.mark.parametrize("engine", ["tc_3x", "simt_fp32"])
@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_update_end_to_end(kind, engine, engine_guard):
    """draws that visit every interior cell once: the density is the oracle EMA of σ = softplus(ops.density_forward)
    at the oracle's points, and the bits its threshold"""
    from sparf_b200 import _lib, occupancy, ops
    ops.set_engine(engine)
    net, opt, _ = _net()
    nerf, res, thres = net.nerf, 16, 0.5
    grid = _build(opt, nerf, kind, res, thres)
    I = int(G.interior(res, kind == "contracted").sum())
    u_cell = ((np.arange(I) + 0.5) / I).astype(np.float32)
    u_jit = np.random.default_rng(1).random((I, 3), dtype=np.float32)
    density0, bits0 = grid.density.cpu().numpy(), grid.bits.cpu().numpy()
    occupancy.update_(grid, nerf, I, 0, decay=0.95, draws=(torch.from_numpy(u_cell).to(DEV), torch.from_numpy(u_jit).to(DEV)))
    cells, pts = G.sample(bits0, res, *grid.range, grid.contraction, I, 0, u_cell, u_jit)
    assert np.array_equal(cells, np.nonzero(G.interior(res, kind == "contracted"))[0])
    raw, _ = ops.density_forward(nerf._spec(), torch.from_numpy(pts).to(DEV),
                                 [p.detach() for p in nerf.kernel_params()[:2 * len(nerf.mlp_feat)]],
                                 progress=nerf.progress.detach(), engine=_lib.ENGINES[engine], features=False)
    sigma = torch.nn.functional.softplus(raw).cpu().numpy()
    want_d, want_bits = G.ema(density0, res, kind == "contracted", cells, sigma, 0.95, thres)
    assert np.array_equal(grid.density.cpu().numpy().view(np.int32), want_d.view(np.int32))
    assert np.array_equal(grid.bits.cpu().numpy().view(np.uint32), want_bits)
    frac = grid.occupied_fraction()
    print("%s %s: occupied fraction after one full sweep %.3f" % (kind, engine, frac))
    assert 0 < frac < 1


@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_build_grid_ema(kind):
    """the density is the corner max of the build's lattice σ, the bits those of a grid built without ema; refresh_
    rewrites both"""
    from sparf_b200 import mesh, occupancy
    net, opt, _ = _net()
    res = 24
    grid = _build(opt, net.nerf, kind, res, 0.5)
    plain = _build(opt, net.nerf, kind, res, 0.5, ema=False)
    assert plain.density is None
    assert torch.equal(grid.bits, plain.bits)

    def lattice():
        if kind == "box":
            return mesh.density_grid(opt, net.nerf, res=res, range=(-1.2, 1.2))
        return mesh.lattice_density(net.nerf, mesh.lattice_axis(res, occupancy.CONTRACTED_RANGE),
                                    warp=occupancy.contracted_warp(*CONTRACTION))
    want = G.corner_max(lattice().cpu().numpy())
    assert np.array_equal(grid.density.cpu().numpy().view(np.int32), want.view(np.int32))
    with torch.no_grad():
        for p in net.nerf.parameters():
            p.mul_(0.9)
    occupancy.refresh_(grid, opt, net.nerf)
    assert np.array_equal(grid.density.cpu().numpy().view(np.int32), G.corner_max(lattice().cpu().numpy()).view(np.int32))
    assert torch.equal(grid.bits, _build(opt, net.nerf, kind, res, 0.5, ema=False).bits)


@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_update_does_not_synchronise(kind):
    from sparf_b200 import occupancy
    net, opt, _ = _net()
    grid = _build(opt, net.nerf, kind, 32, 0.5)
    occupancy.update_(grid, net.nerf, 4096, 4096)      # warm: workspaces, library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            occupancy.update_(grid, net.nerf, 4096, 4096)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def _trainer(kind, draws):
    """a network with res-16 grids (density kept) and a step render -> photometric loss -> backward -> Adam -> update_
    on both networks; draws: per network (u_cell, u_jit) static tensors.  Returns (net, grids, step, the tensors that
    hold the training state)"""
    from sparf_b200 import occupancy
    from sparf_b200.optim import FlatParameters, FusedAdam
    net, opt, data = _net()
    comps = net.get_network_components()
    grids = [_build(opt, m, kind, 16, 0.5) for m in comps]
    net.set_training_occupancy(*grids)
    flat = FlatParameters(comps)
    adam = FusedAdam(flat, lr=1e-3)
    Hh, Ww = data.image.shape[-2:]
    target = data.image.flatten(2).transpose(1, 2)

    def fn():
        flat.zero_grad()
        out = net.render(opt, data.pose, H=Hh, W=Ww, intr=data.intr, ray_idx=torch.arange(Hh * Ww, device=DEV),
                         depth_range=net._depth_range(opt, data), iter=10, mode="train")
        loss = ((out["rgb"] - target) ** 2).mean() + ((out["rgb_fine"] - target) ** 2).mean()
        loss.backward()
        adam.step()
        for i, (g, m) in enumerate(zip(grids, comps)):
            occupancy.update_(g, m, NU, NO, draws=draws[i])
        return loss.detach(), flat.flat
    state = [flat.flat_param, adam.exp_avg, adam.exp_avg_sq, adam.steps, adam.scratch]
    state += [t for g in grids for t in (g.density, g.bits)]
    return net, grids, fn, state


NU, NO = 1024, 1024


@pytest.mark.parametrize("kind", ["box", "contracted"])
def test_captured_step_with_update_equals_eager(kind, engine_guard):
    """a GraphedStep of render -> loss -> backward -> Adam -> update_ on both networks, with draws from static tensors
    refilled before each replay.  Over 5 replays: each replayed update leaves density and bits bit-identical to an eager
    update_ of the grids as they were before the replay, with the same draws, at the weights the replay's Adam step
    left; and the eager step from the same state (parameters, Adam moments, grids) with the same draws gives the same
    loss bit for bit and gradients within 1e-5 of their max (the backward's float atomics are not ordered, so the
    weights after two runs of a step can differ in the last bits, and the grids with them)."""
    from sparf_b200 import occupancy
    from sparf_b200.graphs import GraphedStep
    from sparf_b200.occupancy import OccupancyGrid
    gen = torch.Generator(device=DEV).manual_seed(0)
    static = [(torch.rand(NU + NO, device=DEV, generator=gen), torch.rand(NU + NO, 3, device=DEV, generator=gen))
              for _ in range(2)]
    net, grids, fn, state = _trainer(kind, static)
    step = GraphedStep(fn, (), warmup=2)
    changed = 0
    for it in range(5):
        for uc, uj in static:
            uc.copy_(torch.rand(NU + NO, device=DEV, generator=gen))
            uj.copy_(torch.rand(NU + NO, 3, device=DEV, generator=gen))
        saved = [t.clone() for t in state]
        loss_r, grad_r = [x.clone() for x in step()]
        for g, m, dr, (d0, b0) in zip(grids, net.get_network_components(), static,
                                      zip(saved[5::2], saved[6::2])):
            shadow = OccupancyGrid(b0.clone(), g.res, g.range, g.thres, g.contraction, d0.clone())
            occupancy.update_(shadow, m, NU, NO, draws=dr)
            assert torch.equal(shadow.density.view(torch.int32), g.density.view(torch.int32)), it
            assert torch.equal(shadow.bits, g.bits), it
            changed += int(not torch.equal(b0, g.bits))
        for t, s in zip(state, saved):                     # the eager step from the replay's starting state
            t.copy_(s)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss_e, grad_e = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert torch.equal(loss_r.view(torch.int32), loss_e.view(torch.int32)), it
        assert (grad_r - grad_e).abs().max().item() <= 1e-5 * grad_e.abs().max().item() + 1e-12, it
    print("%s: the bits changed in %d of 10 grid updates" % (kind, changed))
    assert changed > 0
    assert any(0 < g.occupied_fraction() < 1 for g in grids)


def test_capture_that_draws_inside_the_graph_changes_the_grid():
    """update_ with its own torch.rand draws, captured alone (decay 1, density cleared): each replay samples new cells,
    so the density keeps changing and covers more cells"""
    from sparf_b200 import occupancy
    from sparf_b200.graphs import GraphedStep
    net, opt, _ = _net()
    grid = _build(opt, net.nerf, "box", 32, 0.5)
    step = GraphedStep(lambda: occupancy.update_(grid, net.nerf, 2048, 2048, decay=1.0).density, (), warmup=1)
    grid.density.zero_()
    seen = []
    for _ in range(3):
        step()
        seen.append(grid.density.clone())
    assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2])
    assert (seen[0] != 0).sum() < (seen[1] != 0).sum() < (seen[2] != 0).sum()


def test_graphed_training_with_grid_update_converges():
    """train_synthetic with grids updated inside the captured step: the bounds of test_training_loop_converges, and the
    grids end up skipping samples (at thres 0.5, as test_graphed_training_with_grid_converges: the teacher's empty
    space has σ = softplus(-2) = 0.13)"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sparf_b200
    import train_synthetic
    for fine, poses in ((0, 0), (1, 0), (0, 1)):
        try:
            res = train_synthetic.main(["--steps", "300", "--quiet", "--fine", str(fine), "--poses", str(poses), "--rays", "768",
                                        "--grid", "64", "--grid-update", "4096", "--grid-thres", "0.5"])
        finally:
            sparf_b200.set_engine("auto")
        first, last, kept = res[0], res[1], res[-1]
        print("fine=%d poses=%d: loss %.5f -> %.5f, kept fraction %.3f" % (fine, poses, first, last, kept))
        assert last == last and first == first
        assert last < (0.85 if poses else 0.6) * first, (first, last)
        assert kept < 1.0
