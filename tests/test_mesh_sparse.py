"""Sparse marching cubes on the device (sparf_mcubes_sparse_*, ops.marching_cubes_sparse, mesh.extract_mesh_sparse)
against the NumPy restatement (tests/sparse_mcubes_oracle.py) and against the dense extractor: analytic and random ±1
volumes under random active subsets, the octahedron NeRF at res 256 (byte-equal to extract_mesh) and at res 2048 (one
H100), CUDA-graph capture, and tools/extract_mesh.py --sparse."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import mcubes_oracle as O
import sparse_mcubes_oracle as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RADIUS, K, ISO = 0.6, 40.0, 1.0


def _slots(ids, nb):
    slots = torch.full((nb ** 3,), -1, dtype=torch.int32)
    slots[torch.as_tensor(ids, dtype=torch.int64)] = torch.arange(len(ids), dtype=torch.int32)
    return slots.cuda(), torch.as_tensor(ids, dtype=torch.int64).cuda()


def _sparse(vol, ids, iso):
    from sparf_b200 import ops
    res = vol.shape[0] - 1
    slots, bid = _slots(ids, res // 8)
    sig = torch.from_numpy(S.block_points(vol, ids, res // 8)).cuda()
    v, f = ops.marching_cubes_sparse(sig, res, slots, bid, iso)
    torch.cuda.synchronize()
    return v.cpu().numpy(), f.cpu().numpy()


def _equal(got, ref):
    (v, f), (rv, rf) = got, ref
    assert v.shape == rv.shape and f.shape == rf.shape, (v.shape, rv.shape, f.shape, rf.shape)
    assert np.array_equal(v.view(np.uint32), rv.view(np.uint32)), "vertices differ in %d places" % (v != rv).sum()
    assert np.array_equal(f, rf)


def _gaussians(res, seed, n=5):
    rng = np.random.default_rng(seed)
    x = np.stack(np.meshgrid(*[np.arange(res + 1, dtype=np.float64)] * 3, indexing="ij"), -1)
    out = np.zeros(x.shape[:3])
    for _ in range(n):
        c, w = rng.random(3) * res, 2 + 5 * rng.random()
        out += rng.uniform(0.5, 1.5) * np.exp(-((x - c) ** 2).sum(-1) / (2 * w * w))
    return out.astype(np.float32)


@pytest.mark.parametrize("kind", ["gaussians", "pm1", "ties"])
def test_sparse_mc_matches_oracle_on_random_subsets(kind):
    """σ blocks cut from a volume, under random active subsets and with every block active: byte-equal to the oracle,
    and to the dense extractor when every block is active"""
    from sparf_b200 import ops
    table = O.case_table()
    res, nb = 40, 5
    seen = set()
    for seed in range(4):
        rng = np.random.default_rng(seed)
        if kind == "gaussians":
            vol, iso = _gaussians(res, seed), 0.4
        elif kind == "pm1":
            vol, iso = np.where(rng.random((res + 1,) * 3) < 0.5, 1.0, -1.0).astype(np.float32), 0.0
        else:
            vol, iso = rng.integers(-2, 3, (res + 1,) * 3).astype(np.float32), 0.0
        seen |= set(np.unique(O.cell_cases(vol, iso)).tolist())
        for frac in (0.1, 0.5, 1.0):
            ids = np.flatnonzero(rng.random(nb ** 3) < frac) if frac < 1 else np.arange(nb ** 3)
            got = _sparse(vol, ids, iso)
            _equal(got, S.marching_cubes_blocks(S.block_points(vol, ids, nb), ids, res, iso, table))
            if frac == 1.0:
                v, f = ops.marching_cubes(torch.from_numpy(vol).cuda(), iso)
                _equal(got, (v.cpu().numpy(), f.cpu().numpy()))
    if kind == "pm1":
        assert seen == set(range(256))
    assert _sparse(_gaussians(res, 0), np.zeros(0, np.int64), 0.4)[1].shape == (0, 3)


def test_classify_and_points_match_oracle():
    from sparf_b200 import mesh, ops
    rng = np.random.default_rng(3)
    for nb in (1, 4, 7):
        coarse = rng.standard_normal((nb + 1,) * 3).astype(np.float32)
        coarse[rng.random(coarse.shape) < 0.02] = np.nan
        slots, ids = ops.mcubes_sparse_classify(torch.from_numpy(coarse).cuda(), 0.8)
        act = S.classify(coarse, 0.8).reshape(-1)
        ref = np.full(nb ** 3, -1, np.int32)
        ref[act] = np.arange(act.sum())
        assert np.array_equal(slots.cpu().numpy(), ref) and np.array_equal(ids.cpu().numpy(), np.flatnonzero(act))
    res = 56
    axis = mesh.lattice_axis(res, (-0.9, 1.3))
    lat = torch.stack(torch.meshgrid(axis, axis, axis, indexing="ij"), -1).numpy()
    ids = torch.tensor([0, 5, 17, 200, 342], dtype=torch.int64).cuda()
    pts = ops.mcubes_sparse_points(axis.cuda(), ids, 1, 3).cpu().numpy().reshape(3, 9, 9, 9, 3)
    for r, b in enumerate([5, 17, 200]):
        bi, bj, bk = np.unravel_index(b, (7, 7, 7))
        assert np.array_equal(pts[r], lat[8 * bi:8 * bi + 9, 8 * bj:8 * bj + 9, 8 * bk:8 * bk + 9])


def test_workspace_bytes_sane():
    from sparf_b200 import _lib
    L = _lib.lib()
    for res, n, v in ((8, 1, 0), (64, 100, 0), (64, 100, 5000), (512, 100, 5000), (2048, 200000, 10 ** 7)):
        b = L.sparf_mcubes_sparse_workspace_bytes(res, n, v)
        fixed = max(4 * (res // 8) ** 3, 8 * 130 * n + 44 * v)
        assert fixed <= b <= fixed + (64 << 20) + 16 * v, (res, n, v, b)
    assert L.sparf_mcubes_sparse_workspace_bytes(2048, 1000, 10 ** 6) > L.sparf_mcubes_sparse_workspace_bytes(2048, 1000, 0)
    assert L.sparf_mcubes_sparse_workspace_bytes(12, 0, 0) == 0


def _octahedron(engine="tc_3x"):
    import common
    from sparf_b200 import _lib
    from sparf_b200.frequency_nerf import NeRF
    if not _lib.lib().sparf_engine_available(_lib.ENGINES[engine]):
        pytest.skip("%s not available" % engine)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from time_occupancy import octahedron_weights
    opt = common.make_opt()
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in octahedron_weights(opt, c=K * RADIUS, k=K).items()})
    return opt, nerf


def test_octahedron_res256_equals_extract_mesh():
    from sparf_b200 import mesh, ops
    from sparf_b200.utils.edict import edict
    opt, nerf = _octahedron()
    res = 256
    opt.trimesh = edict(res=res, range=[-1.2, 1.2], thres=ISO)
    prev = ops.get_engine()
    ops.set_engine("tc_3x")
    try:
        dense_sigma = mesh.density_grid(opt, nerf)
        axis = mesh.lattice_axis(res, (-1.2, 1.2))
        coarse = mesh.coarse_density(nerf, axis)
        assert torch.equal(coarse.view(torch.int32), dense_sigma[::8, ::8, ::8].contiguous().view(torch.int32))
        slots, ids = ops.mcubes_sparse_classify(coarse, ISO)
        fine = mesh.block_density(nerf, axis, ids)
        cut = torch.from_numpy(S.block_points(dense_sigma.cpu().numpy(), ids.cpu().numpy(), res // 8))
        assert torch.equal(fine.cpu().view(torch.int32), cut.view(torch.int32))
        # every cell the surface crosses lies in an active block
        case = O.cell_cases(dense_sigma.cpu().numpy(), ISO)
        ci, cj, ck = np.nonzero((case != 0) & (case != 255))
        act = (slots.cpu().numpy() >= 0).reshape((res // 8,) * 3)
        assert len(ci) and act[ci // 8, cj // 8, ck // 8].all()
        print("res 256: %d of %d blocks active" % (ids.numel(), (res // 8) ** 3))
        ref = mesh.extract_mesh(opt, nerf, normals=True)
        got = mesh.extract_mesh_sparse(opt, nerf, normals=True)
    finally:
        ops.set_engine(prev)
    for k in ("vertices", "faces", "normals"):
        a, b = got[k].cpu().numpy(), ref[k].cpu().numpy()
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), k


def test_no_active_block_gives_the_empty_mesh():
    """an iso value above every density (and a constant coarse lattice) leaves no block active: classification lists
    none, and extract_mesh_sparse returns the empty mesh, as extract_mesh does"""
    from sparf_b200 import mesh, ops
    from sparf_b200.utils.edict import edict
    slots, ids = ops.mcubes_sparse_classify(torch.full((5, 5, 5), 0.5, device="cuda"), 1.0)
    assert ids.shape == (0,) and (slots == -1).all()
    opt, nerf = _octahedron()
    opt.trimesh = edict(res=64, range=[-1.2, 1.2], thres=100.0)          # σ <= c = 24 everywhere
    ref = mesh.extract_mesh(opt, nerf, normals=True)
    stats = {}
    got = mesh.extract_mesh_sparse(opt, nerf, normals=True, stats=stats)
    assert stats["n_active"] == 0
    for k in ("vertices", "faces", "normals"):
        assert got[k].shape == ref[k].shape == (0, 3) and got[k].dtype == ref[k].dtype, k


def test_marching_cubes_sparse_refuses_a_slot_table_of_another_res():
    from sparf_b200 import ops
    slots, ids = _slots(np.arange(8), 2)
    sig = torch.zeros(8, 9, 9, 9, device="cuda")
    with pytest.raises(AssertionError):
        ops.marching_cubes_sparse(sig, 24, slots, ids, 0.5)


def _area(v, f):
    return 0.5 * np.linalg.norm(O.face_normals(v, f), axis=1).sum()


def test_octahedron_res2048_on_one_gpu():
    """res 2048 (the dense volume and its workspace would need ~100 GB): a closed, oriented genus-0 mesh whose area is
    at least as close to the analytic octahedron's as the dense mesh's at res 512"""
    from sparf_b200 import mesh, ops
    from sparf_b200.utils.edict import edict
    opt, nerf = _octahedron()
    r_iso = (K * RADIUS - math.log(math.expm1(ISO))) / K
    exact = 4 * math.sqrt(3) * r_iso ** 2
    prev = ops.get_engine()
    ops.set_engine("tc_3x")
    try:
        opt.trimesh = edict(res=512, range=[-1.2, 1.2], thres=ISO)
        d = mesh.extract_mesh(opt, nerf)
        err512 = abs(_area(d["vertices"].cpu().numpy(), d["faces"].cpu().numpy()) / exact - 1)
        del d
        torch.cuda.empty_cache()
        opt.trimesh = edict(res=2048, range=[-1.2, 1.2], thres=ISO)
        stats = {}
        m = mesh.extract_mesh_sparse(opt, nerf, stats=stats)
        torch.cuda.synchronize()
    finally:
        ops.set_engine(prev)
    v, f = m["vertices"].cpu().numpy(), m["faces"].cpu().numpy()
    err = abs(_area(v, f) / exact - 1)
    print("res 2048: %s, V %d, F %d, area error %.3g (dense res 512: %.3g)" % (stats, len(v), len(f), err, err512))
    assert len(f) > 10 ** 6 and f.min() >= 0 and f.max() < len(v)
    assert O.is_closed_and_oriented(f) and O.euler_characteristic(f) == 2
    assert err <= err512


def test_count_emit_capture_and_replay():
    """classification outputs fixed, count + emit captured in one CUDA graph: replays give the eager call's bytes, also
    on new σ contents"""
    from sparf_b200 import _lib, ops
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    res, nb = 48, 6
    ids_np = np.flatnonzero(np.random.default_rng(1).random(nb ** 3) < 0.6)
    slots, ids = _slots(ids_np, nb)
    sigs = [torch.from_numpy(S.block_points(_gaussians(res, s), ids_np, nb)).cuda() for s in (20, 21)]
    sig = sigs[0].clone()
    ref = [ops.marching_cubes_sparse(x, res, slots, ids, 0.4) for x in sigs]
    cap_v, cap_f = max(r[0].shape[0] for r in ref), max(r[1].shape[0] for r in ref)
    n = len(ids_np)
    ws = torch.empty(L.sparf_mcubes_sparse_workspace_bytes(res, n, cap_v), dtype=torch.uint8, device="cuda")
    totals = torch.zeros(2, dtype=torch.int64, device="cuda")
    verts = torch.zeros(cap_v, 3, device="cuda")
    faces = torch.zeros(cap_f, 3, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.sparf_mcubes_sparse_count(p(sig), res, p(slots), p(ids), n, 0.4, p(totals), p(ws), ws.numel(), st),
                   "count")
        _lib.check(L.sparf_mcubes_sparse_emit(p(sig), res, p(slots), p(ids), n, 0.4, cap_v, cap_f, p(verts), p(faces),
                                              p(ws), ws.numel(), st), "emit")
    for x, (rv, rf) in zip(sigs + sigs[:1], ref + ref[:1]):
        sig.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        V, F = totals.tolist()
        assert (V, F) == (rv.shape[0], rf.shape[0])
        assert torch.equal(verts[:V].view(torch.int32), rv.view(torch.int32)) and torch.equal(faces[:F], rf)


def test_extract_mesh_tool_sparse(tmp_path):
    """tools/extract_mesh.py --sparse writes extract_mesh_sparse's mesh"""
    import common
    from sparf_b200 import mesh
    from sparf_b200.renderer import Graph
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    opt = common.make_opt(fine=True)
    graph = Graph(opt, torch.device("cuda"))
    graph.nerf.load_state_dict(common.det_weights(opt, 5, peaky=True, sigma_bias=-2.0, progress=1.0))
    graph.nerf_fine.load_state_dict(common.det_weights(opt, 82, peaky=True, sigma_bias=-2.0, progress=1.0))
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": graph.state_dict()}, ckpt)
    sigma = mesh.density_grid(opt, graph.nerf, res=64)
    thres = torch.quantile(sigma.view(-1), 0.8).item()
    out = str(tmp_path / "mesh.ply")
    tool.main([ckpt, "--res", "64", "--thres", str(thres), "--sparse", "--out", out])
    props, faces = O.read_ply(out)
    opt.trimesh = dict(res=64, range=[-1.2, 1.2], thres=thres)
    ref = mesh.extract_mesh_sparse(opt, graph.nerf)
    assert len(faces) > 0 and np.array_equal(faces, ref["faces"].cpu().numpy())
    assert np.array_equal(np.stack([props[k] for k in "xyz"], 1), ref["vertices"].cpu().numpy())
