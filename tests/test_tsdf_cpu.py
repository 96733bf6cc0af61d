"""TSDF fusion without a GPU: the NumPy oracle (tests/tsdf_oracle.py) on hand-worked views, the argument checks of
tsdf.integrate_ and of the C entry points, and the PLY writer's colours."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch

import tsdf_oracle as T

INVALID = 1     # SPARF_ERR_INVALID


def _view(H=4, W=6, f=4.0, cz=-2.0):
    """identity rotation, camera at (0, 0, cz) looking along +z, principal point at the image centre"""
    pose = np.array([[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, -cz]]], np.float32)
    K = np.array([[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]], np.float32)
    return pose, K


def test_oracle_hand_worked_view():
    """lattice {-1, 0, 1}^3, camera 2 in front of it: the centre line of points lands in the image centre's pixel"""
    axis = np.array([-1, 0, 1], np.float32)
    pose, K = _view()
    depth = np.full((1, 4, 6), 2.5, np.float32)            # a surface at z = 0.5
    rgb = np.zeros((1, 4, 6, 3), np.float32)
    rgb[..., 1] = 0.25
    tsdf, weight, color = T.integrate(axis, 0.75, pose, K, depth, rgb)
    pts = T.lattice_points(axis)
    # point (0, 0, z): camera z = z + 2, pixel (3, 2); s = 2.5 - (z + 2) = 0.5 - z
    for z, want in ((-1.0, 1.0), (0.0, 0.5 / 0.75), (1.0, None)):     # z = 1: s = -0.5 >= -0.75, f = -2/3
        p = int(np.flatnonzero((pts == [0, 0, z]).all(1))[0])
        assert weight[p] == 1
        assert tsdf[p] == pytest.approx(want if want is not None else -0.5 / 0.75, abs=1e-7)
        assert color[p].tolist() == [0.0, 0.25, 0.0]
    # point (1, 1, -1): camera (1, 1, 1), u = 4 * 1 / 1 + 3 = 7 >= W: outside the image
    p = int(np.flatnonzero((pts == [1, 1, -1]).all(1))[0])
    assert weight[p] == 0 and tsdf[p] == 1


def test_oracle_skips_and_averages():
    axis = np.array([-1, 0, 1], np.float32)
    pose, K = _view()
    pts = T.lattice_points(axis)
    centre = (pts[:, 0] == 0) & (pts[:, 1] == 0)
    # occluded: the surface at z = -0.5 hides z = 1 (s = -1.5 < -trunc) but not z = -1
    tsdf, weight, _ = T.integrate(axis, 0.75, pose, K, np.full((1, 4, 6), 1.5, np.float32))
    assert weight[centre].tolist() == [1, 1, 0]
    # non-finite or non-positive depth and invalid pixels are skipped
    for d in (np.nan, np.inf, 0.0, -1.0):
        _, weight, _ = T.integrate(axis, 0.75, pose, K, np.full((1, 4, 6), d, np.float32))
        assert weight.sum() == 0
    _, weight, _ = T.integrate(axis, 0.75, pose, K, np.full((1, 4, 6), 2.5, np.float32), valid=np.zeros((1, 4, 6), bool))
    assert weight.sum() == 0
    # two views: the running average, and integrating them one by one gives the same state
    pose2, K2 = np.concatenate([pose, pose]), np.concatenate([K, K])
    depth = np.stack([np.full((4, 6), 2.5, np.float32), np.full((4, 6), 2.2, np.float32)])
    rgb = np.stack([np.full((4, 6, 3), 0.2, np.float32), np.full((4, 6, 3), 0.6, np.float32)])
    both = T.integrate(axis, 0.75, pose2, K2, depth, rgb)
    one = T.integrate(axis, 0.75, pose, K, depth[:1], rgb[:1])
    two = T.integrate(axis, 0.75, pose, K, depth[1:], rgb[1:], state=one)
    for a, b in zip(both, two):
        assert np.array_equal(a, b)
    p = int(np.flatnonzero((pts == [0, 0, 0]).all(1))[0])
    assert both[1][p] == 2
    assert both[0][p] == pytest.approx((0.5 / 0.75 + np.float32(0.2) / np.float32(0.75)) / 2, abs=1e-6)
    assert both[2][p] == pytest.approx([(0.2 + 0.6) / 2] * 3, abs=1e-7)


def test_oracle_masked_marching_cubes_without_nan_is_dense():
    rng = np.random.default_rng(3)
    vol = rng.standard_normal((9, 10, 11)).astype(np.float32)
    v, f = T.masked_marching_cubes(vol, 0.2)
    rv, rf = T.O.marching_cubes(vol, 0.2)
    assert np.array_equal(v, rv) and np.array_equal(f, rf)
    vol[4, 5, 6] = np.nan
    v, f = T.masked_marching_cubes(vol, 0.2)
    assert len(f) < len(rf) and f.max() < len(v) and len(np.unique(f)) == len(v)


# ------------------------------------------------------------------------------------------------ argument checks
def _vol(res=4):
    from sparf_b200 import tsdf
    return tsdf.TSDFVolume(res=res, device="cpu")


def test_volume_defaults_and_reset():
    from sparf_b200 import mesh, tsdf
    vol = _vol(8)
    assert vol.range == mesh.TRIMESH_DEFAULTS["range"] and vol.n == 9
    assert vol.trunc == pytest.approx(tsdf.TRUNC_VOXELS * 2.4 / 8)
    assert vol.tsdf.shape == (9, 9, 9) and vol.color.shape == (9, 9, 9, 3)
    assert torch.equal(vol.axis, mesh.lattice_axis(8, mesh.TRIMESH_DEFAULTS["range"]))
    vol.tsdf.zero_(), vol.weight.fill_(3), vol.color.fill_(0.5)
    vol.reset_()
    assert (vol.tsdf == 1).all() and (vol.weight == 0).all() and (vol.color == 0).all()
    with pytest.raises(ValueError):
        tsdf.TSDFVolume(res=8, trunc=0.0, device="cpu")
    with pytest.raises(ValueError):
        tsdf.TSDFVolume(res=0, device="cpu")


def test_integrate_rejects_bad_arguments():
    from sparf_b200 import tsdf
    vol = _vol()
    B, H, W = 2, 5, 7
    good = dict(depth=torch.ones(B, H, W), pose_w2c=torch.zeros(B, 3, 4), intr=torch.eye(3),
                rgb=torch.zeros(B, H, W, 3), valid=torch.ones(B, H, W, dtype=torch.bool))
    bad = [
        ("depth", torch.ones(H, W)), ("depth", torch.ones(0, H, W)), ("depth", torch.ones(B, H, W, dtype=torch.float64)),
        ("depth", np.ones((B, H, W), np.float32)),
        ("pose_w2c", torch.zeros(B, 4, 4)), ("pose_w2c", torch.zeros(B + 1, 3, 4)), ("pose_w2c", torch.zeros(3, 4)),
        ("pose_w2c", torch.zeros(B, 3, 4, dtype=torch.float16)),
        ("intr", torch.eye(4)), ("intr", torch.zeros(B + 1, 3, 3)), ("intr", torch.eye(3, dtype=torch.float64)),
        ("rgb", torch.zeros(B, H, W)), ("rgb", torch.zeros(B, W, H, 3)), ("rgb", torch.zeros(B, H, W, 3, dtype=torch.uint8)),
        ("valid", torch.ones(B, H, W + 1, dtype=torch.bool)), ("valid", torch.ones(B, H, W)),
        ("depth", torch.ones(B, H, W, device="meta")), ("rgb", torch.zeros(B, H, W, 3, device="meta")),
        ("pose_w2c", torch.zeros(B, 3, 4, device="meta")),
    ]
    for name, value in bad:
        kw = dict(good, **{name: value})
        with pytest.raises(ValueError):
            tsdf.integrate_(vol, **kw)
    with pytest.raises(ValueError, match="CUDA"):      # everything well formed, but the volume is not on a GPU
        tsdf.integrate_(vol, **good)


def test_c_entry_points_reject_invalid_sizes():
    """SPARF_ERR_INVALID before anything is read or launched (the pointers are host dummies)"""
    from sparf_b200 import _lib
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = dict(n=5, trunc=0.1, B=2, H=4, W=6)

    def call(n, trunc, B, H, W, rgb=None, color=p, axis=p):
        return L.sparf_tsdf_integrate(axis, n, trunc, B, H, W, p, p, p, rgb, None, p, p, color, None)

    cases = [dict(n=1), dict(n=0), dict(n=-3), dict(n=1 << 13), dict(n=(1 << 31) - 1), dict(trunc=0.0), dict(trunc=-1.0),
             dict(trunc=float("nan")), dict(trunc=float("inf")), dict(B=0), dict(B=-1), dict(H=0), dict(W=0),
             dict(W=(1 << 24) + 1), dict(H=(1 << 24) + 1), dict(B=(1 << 31) - 1, H=1 << 24, W=1 << 24)]
    for c in cases:
        assert call(**dict(ok, **c)) == INVALID, c
        assert L.sparf_last_error()
    assert call(**ok, rgb=p, color=None) == INVALID          # colours need a colour volume
    assert call(**ok, axis=None) == INVALID
    assert L.sparf_mcubes_count_masked(p, 1, 5, 5, 0.0, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mcubes_emit_masked(p, 5, 5, 1, 0.0, p, p, p, 1 << 20, None) == INVALID
    assert L.sparf_mcubes_count_masked(None, 5, 5, 5, 0.0, p, p, 1 << 20, None) == INVALID


# ------------------------------------------------------------------------------------------------ PLY colours
def _mesh():
    rng = np.random.default_rng(5)
    v = rng.standard_normal((7, 3)).astype(np.float32)
    f = np.array([[0, 1, 2], [2, 3, 4], [4, 5, 6], [6, 0, 3]])
    n = rng.standard_normal((7, 3)).astype(np.float32)
    return v, f, n


# sha256 of the files the parent commit's write_ply wrote for _mesh() (without normals, with normals) and for no mesh
PARENT_PLY_SHA256 = {
    "plain": "71e0b2450e2a5ad3ce31e7880dfceaeef8fb8bf139a85adb4dcfd9326c9118b0",
    "normals": "4afa16f16f35e1c4cf9107e595838006a6bc6e50ee7cf8f155bd8cadf17c77ec",
    "empty": "b6732ab7f2e04692ecde8f47833cd5009c6a08caa6c8710b00742424959d9ca0",
}


def test_write_ply_without_colors_is_unchanged(tmp_path):
    from sparf_b200 import mesh
    v, f, n = _mesh()
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))
    for name, args in (("plain", (v, f)), ("normals", (v, f, n)), ("empty", empty)):
        path = tmp_path / (name + ".ply")
        mesh.write_ply(str(path), *args)
        assert hashlib.sha256(path.read_bytes()).hexdigest() == PARENT_PLY_SHA256[name], name


@pytest.mark.parametrize("with_normals", [False, True])
def test_write_ply_colors_round_trip(tmp_path, with_normals):
    from sparf_b200 import mesh
    v, f, n = _mesh()
    c = np.array([[0, 1, 0.5], [-0.2, 1.3, np.float32(0.5) / 255], [1 / 255, 254.5 / 255, 0.3], [0.999, 0.001, 0.75],
                  [0.2, 0.4, 0.6], [1, 1, 1], [0, 0, 0]], np.float32)
    path = str(tmp_path / "c.ply")
    mesh.write_ply(path, torch.from_numpy(v), torch.from_numpy(f), torch.from_numpy(n) if with_normals else None,
                   colors=torch.from_numpy(c))
    header, vert, faces = T.read_ply(path)
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if with_normals else [])
    assert header[3:3 + len(names)] == ["property float %s" % k for k in names]
    assert header[3 + len(names):6 + len(names)] == ["property uchar red", "property uchar green", "property uchar blue"]
    assert np.array_equal(faces, f)
    assert np.array_equal(np.stack([vert[k] for k in "xyz"], 1), v)
    if with_normals:
        assert np.array_equal(np.stack([vert[k] for k in ("nx", "ny", "nz")], 1), n)
    got = np.stack([vert[k] for k in ("red", "green", "blue")], 1)
    want = np.round(np.clip(c, 0, 1) * np.float32(255)).astype(np.uint8)
    assert np.array_equal(got, want)
    assert got[0].tolist() == [0, 255, 128] and got[1].tolist() == [0, 255, 0] and got[5].tolist() == [255] * 3
