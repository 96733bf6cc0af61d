"""GPU tests of the mesh components (csrc/mesh_components.cu): labels, face counts and selection against the NumPy oracle
(tests/components_oracle.py) on soups, deep trees, stars and empty meshes; determinism; floater removal that gives the
mesh of the region alone byte for byte; the three extractors; CUDA-graph capture; the tool."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import components_oracle as CO
import mcubes_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(faces_np, V, seed=0):
    """ops.mesh_components and ops.mesh_select (a random keep mask) against the oracle, torch.equal"""
    from sparf_b200 import ops
    faces = torch.from_numpy(np.asarray(faces_np, np.int64).reshape(-1, 3)).cuda()
    labels, counts = ops.mesh_components(faces, V)
    rl, rc = CO.components(faces_np, V)
    assert labels.dtype == torch.int32 and counts.dtype == torch.int64
    assert torch.equal(labels.cpu(), torch.from_numpy(rl)) and torch.equal(counts.cpu(), torch.from_numpy(rc))
    keep = (np.random.default_rng(seed).random(len(rc)) < 0.5).astype(np.uint8)
    vert_ids, f = ops.mesh_select(faces, V, labels, torch.from_numpy(keep).cuda())
    rv, rf = CO.select(faces_np, rl, keep)
    assert torch.equal(vert_ids.cpu(), torch.from_numpy(rv)) and torch.equal(f.cpu(), torch.from_numpy(rf))
    return labels, counts


# ------------------------------------------------------------------------------------------------ 1. against the oracle
@pytest.mark.parametrize("V,F,groups", [(1000, 1500, 100), (200_000, 300_000, 30_000), (100_000, 400_000, 10),
                                        (50_000, 20_000, 40_000)])
def test_random_soups_match_oracle(V, F, groups):
    _check(CO.random_soup(V, F, seed=V + F, n_groups=groups), V, seed=1)


@pytest.mark.parametrize("permuted", [False, True])
def test_million_vertex_strip(permuted):
    """faces (i, i+1, i+2): one component whose union-find tree is as deep as it gets with ordered ids"""
    V = 1 << 20
    i = np.arange(V - 2)
    f = np.stack([i, i + 1, i + 2], 1)
    if permuted:
        f = np.random.default_rng(3).permutation(V)[f]
    labels, counts = _check(f, V)
    assert counts.tolist() == [V - 2] and labels.max().item() == 0


@pytest.mark.parametrize("hub", ["first", "last"])
def test_star(hub):
    V = 300_000
    h = 0 if hub == "first" else V - 1
    rim = np.setdiff1d(np.arange(V), [h])
    f = np.stack([np.full(V - 2, h), rim[:-1], rim[1:]], 1)
    _check(f, V)
    _check(np.roll(f, 1, axis=1), V + 5)            # the hub last in each face, and 5 unused vertices


def test_disjoint_triangles():
    F = 500_000
    labels, counts = _check(np.arange(3 * F).reshape(F, 3), 3 * F + 7)
    assert counts.numel() == F + 7 and (counts[:F] == 1).all() and (counts[F:] == 0).all()


def test_one_component():
    V = 100_000
    rng = np.random.default_rng(4)
    i = np.arange(V - 2)
    f = np.concatenate([np.stack([i, i + 1, i + 2], 1), rng.integers(0, V, (200_000, 3))])
    labels, counts = _check(rng.permutation(f), V)
    assert counts.tolist() == [len(f)]


def test_tiny_and_empty():
    from sparf_b200 import ops
    for f, V in ((np.zeros((0, 3), np.int64), 0), (np.zeros((0, 3), np.int64), 1), (np.zeros((1, 3), np.int64), 1),
                 (np.zeros((0, 3), np.int64), 6), (np.array([[2, 2, 2]]), 4)):
        _check(f, V)
    labels, counts = ops.mesh_components(torch.zeros(0, 3, dtype=torch.int64, device="cuda"), 0)
    assert labels.shape == counts.shape == (0,)
    with pytest.raises(ValueError):
        ops.mesh_components(torch.tensor([[0, 1, 5]], device="cuda"), 5)
    with pytest.raises(ValueError):
        ops.mesh_components(torch.tensor([[0, -1, 2]], device="cuda"), 5)
    f = torch.tensor([[0, 1, 2]], device="cuda")
    labels, counts = ops.mesh_components(f, 4)
    with pytest.raises(ValueError):         # a label past keep
        ops.mesh_select(f, 4, labels, torch.ones(1, dtype=torch.uint8, device="cuda"))


def test_face_order_and_repeat_do_not_change_the_bytes():
    from sparf_b200 import ops
    V = 300_000
    f = CO.random_soup(V, 500_000, seed=9, n_groups=20_000)
    faces = torch.from_numpy(f).cuda()
    l1, c1 = ops.mesh_components(faces, V)
    l2, c2 = ops.mesh_components(faces, V)
    perm = torch.from_numpy(np.random.default_rng(2).permutation(len(f))).cuda()
    l3, c3 = ops.mesh_components(faces[perm].roll(1, dims=1), V)
    assert torch.equal(l1, l2) and torch.equal(c1, c2) and torch.equal(l1, l3)
    assert c1.sum().item() == c3.sum().item() == len(f)


# ------------------------------------------------------------------------------------------------ 2. floater removal
def _ball(shape, center, radius):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) for n in shape], indexing="ij"), -1)
    return np.float32(radius) - np.linalg.norm(g - np.asarray(center, np.float32), axis=-1).astype(np.float32)


BIG = ((40, 48, 48), 25.0)
SMALL = [((85, 10, 10), 3.0), ((85, 85, 85), 2.5), ((10, 85, 20), 3.5), ((82, 48, 48), 2.0), ((10, 10, 85), 4.0)]


def _sphere_and_blobs(n=96):
    big = _ball((n,) * 3, *BIG)
    vol = big.copy()
    for c, r in SMALL:
        vol = np.maximum(vol, _ball((n,) * 3, c, r))      # exact: the big sphere's values where no blob is near
    return torch.from_numpy(big).cuda(), torch.from_numpy(vol).cuda()


def _equal_mesh(a, b):
    for k in b:
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype, k
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k


def test_selection_gives_the_region_alone():
    from sparf_b200 import mesh, ops
    big, vol = _sphere_and_blobs()
    v, f = ops.marching_cubes(big, 0.0)
    alone = dict(vertices=v, faces=f)
    v, f = ops.marching_cubes(vol, 0.0)
    m = dict(vertices=v, faces=f)
    labels, counts = ops.mesh_components(f, v.shape[0])
    assert counts.numel() == 1 + len(SMALL)
    small_max = sorted(counts.tolist())[-2]
    stats = {}
    _equal_mesh(mesh.keep_components(m, largest=1, stats=stats), alone)
    assert stats == dict(n_components=1 + len(SMALL), n_kept=1, faces_removed=f.shape[0] - alone["faces"].shape[0])
    _equal_mesh(mesh.keep_components(m, min_faces=small_max + 1), alone)
    _equal_mesh(mesh.keep_components(m, min_faces=0), m)
    assert mesh.keep_components(m, min_faces=f.shape[0] + 1)["faces"].shape == (0, 3)


def _torus(shape, center, R, r):
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij"), -1) - center
    q = np.sqrt(g[..., 0] ** 2 + g[..., 1] ** 2) - R
    return (r - np.sqrt(q ** 2 + g[..., 2] ** 2)).astype(np.float32)


def test_euler_characteristic_per_component():
    from sparf_b200 import mesh, ops
    n = 128
    vol = np.maximum(_torus((n,) * 3, (45, 64, 64), 25.0, 8.0), _ball((n,) * 3, (100, 64, 64), 18.0))
    for c, r in SMALL:
        vol = np.maximum(vol, _ball((n,) * 3, c, r))
    v, f = ops.marching_cubes(torch.from_numpy(vol).cuda(), 0.0)
    m = mesh.keep_components(dict(vertices=v, faces=f), largest=2)
    labels, counts = ops.mesh_components(m["faces"], m["vertices"].shape[0])
    assert counts.numel() == 2
    chis = []
    for c in range(2):
        keep = torch.zeros(2, dtype=torch.uint8, device="cuda")
        keep[c] = 1
        _, fc = ops.mesh_select(m["faces"], m["vertices"].shape[0], labels, keep)
        fc = fc.cpu().numpy()
        assert O.is_closed_and_oriented(fc)
        chis.append(O.euler_characteristic(fc))
    assert sorted(chis) == [0, 2]


# ------------------------------------------------------------------------------------------------ 3. the extractors
K, OFFSET, ISO = 40.0, 5.0, 5.0
MAIN = ((0.0, 0.0, 0.0), 0.6)
BLOBS = [((0.875, 0.875, 0.875), 0.125), ((-0.875, 0.75, -0.625), 0.1), ((0.875, -0.875, 0.0), 0.15)]


def blob_weights(opt, blobs, seed=0):
    """state_dict of a NeRF whose density is softplus(sum_j relu(c_j - K |x - b_j|_1) - OFFSET): one octahedron per
    blob (b_j, radius r_j; c_j set so that the iso surface sigma = ISO lies at |x - b_j|_1 = r_j).  Layer 0 holds
    relu(+-(x_a - b_ja)), layer 1 the blobs' units, the next layers pass them through, the density row sums them.
    Where the supports |x - b_j|_1 < c_j / K do not overlap, a point's density depends on its own blob's units alone,
    so adding a blob changes no value away from it, bit for bit.  The colour head has small random weights."""
    import common
    s = float(np.log(np.expm1(ISO))) + OFFSET
    rng = np.random.default_rng(seed)
    sd = {}
    n_trunk = len(opt.arch.layers_feat) - 1
    nb = len(blobs)
    for li, (name, k_out, k_in) in enumerate(common.layer_shapes(opt)):
        w = np.zeros((k_out, k_in), np.float32)
        b = np.zeros(k_out, np.float32)
        if li == 0:
            for j, (ctr, _) in enumerate(blobs):
                for a in range(3):
                    w[6 * j + 2 * a, a], b[6 * j + 2 * a] = 1, -ctr[a]
                    w[6 * j + 2 * a + 1, a], b[6 * j + 2 * a + 1] = -1, ctr[a]
        elif li == 1:
            for j, (_, r) in enumerate(blobs):
                w[j, 6 * j:6 * j + 6], b[j] = -K, s + K * r
        elif li < n_trunk - 1:
            w[np.arange(nb), np.arange(nb)] = 1
        elif li == n_trunk - 1:
            w[0, :nb], b[0] = 1, -OFFSET
            w[1 + np.arange(nb), np.arange(nb)] = 1
        else:
            w = rng.normal(0, 0.3, (k_out, k_in)).astype(np.float32)
            b = rng.normal(0, 0.1, k_out).astype(np.float32)
        sd[name + ".weight"], sd[name + ".bias"] = torch.from_numpy(w), torch.from_numpy(b)
    sd["progress"] = torch.tensor(1.0)
    return sd


def _nerfs(res):
    import common
    from sparf_b200.frequency_nerf import NeRF
    from sparf_b200.utils.edict import edict
    opt = common.make_opt()
    opt.trimesh = edict(res=res, range=[-1.2, 1.2], thres=ISO)
    nets = []
    for blobs in ([MAIN], [MAIN] + BLOBS):
        nerf = NeRF(opt).cuda()
        nerf.load_state_dict({k: v.cuda() for k, v in blob_weights(opt, blobs).items()})
        nets.append(nerf)
    return opt, nets


def _gathered(got, m, keys):
    """the kept vertices' per-vertex data equal the originals gathered with the oracle's vert_ids, bit for bit"""
    labels, counts = CO.components(m["faces"].cpu().numpy(), m["vertices"].shape[0])
    vert_ids, faces = CO.select(m["faces"].cpu().numpy(), labels, CO.keep_mask(counts, largest=1))
    assert np.array_equal(got["faces"].cpu().numpy(), faces)
    for k in keys:
        assert got[k].cpu().numpy().tobytes() == m[k].cpu().numpy()[vert_ids].tobytes(), k


@pytest.mark.parametrize("sparse", [False, True])
def test_extractors_lose_exactly_the_blobs(sparse):
    from sparf_b200 import mesh
    opt, (alone, blobs) = _nerfs(res=128)
    extract = mesh.extract_mesh_sparse if sparse else mesh.extract_mesh
    ref = extract(opt, alone)
    m = extract(opt, blobs, normals=True)
    stats = {}
    got = mesh.keep_components(m, largest=1, stats=stats)
    assert stats["n_components"] == 1 + len(BLOBS) and stats["n_kept"] == 1
    _equal_mesh({k: got[k] for k in ref}, ref)
    _gathered(got, m, ["vertices", "normals"])


def _ring_cams(n, H, W, radius=3.0, seed=0):
    """n views around the box, at varied heights"""
    import common
    rng = np.random.default_rng(seed)
    poses = []
    for b in range(n):
        a = 2 * math.pi * b / n
        poses.append(common.look_at_w2c((radius * math.sin(a), rng.uniform(-1.5, 1.5), -radius * math.cos(a))))
    f = 1.1 * max(H, W)
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]], np.float32)
    return np.stack(poses), np.stack([K] * n)


# a smaller main octahedron leaves room for blobs big enough to survive fusion at res 64 (voxel 0.0375)
MAIN_TSDF = ((0.0, 0.0, 0.0), 0.4)
BLOBS_TSDF = [((0.7, 0.7, 0.0), 0.2), ((-0.75, 0.0, -0.75), 0.2), ((0.0, -0.75, 0.75), 0.2)]


def test_tsdf_mesh_loses_the_blobs():
    import common
    from sparf_b200 import mesh, tsdf
    from sparf_b200.renderer import Graph
    opt = common.make_opt(fine=True, depth_range=(1.5, 4.5))
    graph = Graph(opt, torch.device("cuda"))
    for i, net in enumerate(graph.get_network_components()):
        net.load_state_dict({k: v.cuda() for k, v in blob_weights(opt, [MAIN_TSDF] + BLOBS_TSDF, seed=i).items()})
    B, H, W = 12, 60, 80
    poses, Kc = _ring_cams(B, H, W)
    vol = tsdf.TSDFVolume(res=64)
    tsdf.fuse_renders(opt, graph, vol, torch.from_numpy(poses), torch.from_numpy(Kc), H, W, (1.5, 4.5))
    m = tsdf.extract_mesh(vol)
    stats = {}
    got = mesh.keep_components(m, largest=1, stats=stats)
    _gathered(got, m, ["vertices", "colors"])
    v = m["vertices"].cpu().numpy()
    near_blob = np.zeros(len(v), bool)
    for ctr, r in BLOBS_TSDF:
        near_blob |= np.abs(v - np.asarray(ctr)).sum(1) < r + 0.15
    kept = np.zeros(len(v), bool)
    labels, counts = CO.components(m["faces"].cpu().numpy(), len(v))
    kept[labels == np.argmax(counts)] = True
    print("TSDF: %s, %d vertices near blobs" % (stats, near_blob.sum()))
    assert near_blob.any() and stats["n_components"] > 1
    assert not (kept & near_blob).any()                             # every blob vertex is removed
    assert np.abs(np.abs(v[kept]).sum(1) - MAIN_TSDF[1]).max() < 0.25     # and what is kept is the main surface


# ------------------------------------------------------------------------------------------------ 4. capture
def test_capture_and_replay():
    """sparf_mesh_components and the select pair captured in CUDA graphs: replays give the eager bytes, also on new
    face contents of the same size"""
    from sparf_b200 import _lib, ops
    L = _lib.lib()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    V, F = 50_000, 60_000
    soups = [torch.from_numpy(CO.random_soup(V, F, seed=s, n_groups=5000)[:F - 100]).cuda() for s in (5, 6)]
    F = min(s.shape[0] for s in soups)
    soups = [s[:F].contiguous() for s in soups]
    faces = soups[0].clone()
    ws = torch.empty(L.sparf_mesh_components_workspace_bytes(V, F), dtype=torch.uint8, device="cuda")
    labels = torch.zeros(V, dtype=torch.int32, device="cuda")
    n_comp = torch.zeros(1, dtype=torch.int64, device="cuda")
    keep = torch.zeros(V, dtype=torch.uint8, device="cuda")
    totals = torch.zeros(2, dtype=torch.int64, device="cuda")
    vert_ids = torch.zeros(V, dtype=torch.int64, device="cuda")
    faces_out = torch.zeros(F, 3, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1, stream=s):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.sparf_mesh_components(p(faces), F, V, p(labels), p(n_comp), p(ws), ws.numel(), st), "components")
    with torch.cuda.graph(g2, stream=s):
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.sparf_mesh_select_count(p(faces), F, V, p(labels), p(keep), V, p(totals), p(ws), ws.numel(), st),
                   "select_count")
        _lib.check(L.sparf_mesh_select_emit(p(faces), F, V, p(labels), p(keep), V, p(vert_ids), p(faces_out), p(ws),
                                            ws.numel(), st), "select_emit")
    for x in soups + soups[:1]:
        faces.copy_(x)
        rl, rc = ops.mesh_components(x, V)
        rk = (rc >= 3).to(torch.uint8)
        rv, rf = ops.mesh_select(x, V, rl, rk)
        g1.replay()
        torch.cuda.synchronize()
        assert n_comp.item() == rc.numel() and torch.equal(labels, rl)
        keep.zero_()
        keep[:rc.numel()] = rk
        g2.replay()
        torch.cuda.synchronize()
        nv, nf = totals.tolist()
        assert (nv, nf) == (rv.numel(), rf.shape[0])
        assert torch.equal(vert_ids[:nv], rv) and torch.equal(faces_out[:nf], rf)


# ------------------------------------------------------------------------------------------------ 5. the tool
def test_extract_mesh_tool_keep_largest(tmp_path):
    """tools/extract_mesh.py --keep-largest 1 writes the bytes of keep_components + write_ply"""
    from sparf_b200 import mesh
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_mesh as tool
    opt, (_, blobs) = _nerfs(res=64)
    ckpt = str(tmp_path / "model.pth.tar")
    torch.save({"state_dict": {"nerf." + k: v for k, v in blobs.state_dict().items()}}, ckpt)
    for extra, extract in (([], mesh.extract_mesh), (["--sparse"], mesh.extract_mesh_sparse)):
        out = str(tmp_path / "tool.ply")
        tool.main([ckpt, "--res", "64", "--thres", str(ISO), "--normals", "--keep-largest", "1", "--out", out] + extra)
        m = mesh.keep_components(extract(opt, blobs, normals=True), largest=1)
        ref = str(tmp_path / "ref.ply")
        mesh.write_ply(ref, m["vertices"], m["faces"], m["normals"])
        assert m["faces"].shape[0] > 100
        with open(out, "rb") as a, open(ref, "rb") as b:
            assert a.read() == b.read(), extra
