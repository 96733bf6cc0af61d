"""Properties of the contracted occupancy grid's oracle (tests/contraction_oracle.py), on the CPU: the map is continuous
at the edge of the linear region and monotone along rays, the build's lattice inverse agrees with the forward map, the
points at infinity give the always-occupied outer shell, and on a forward-facing inverse-depth wall scene the grid
keeps the sample counts pinned below."""
import numpy as np
import pytest

import contraction_oracle as C
import occupancy_oracle as O
import termination_oracle as T

f32 = np.float32


def _axis(res):
    from sparf_b200 import mesh
    return mesh.lattice_axis(res, (-2.0, 2.0)).numpy()


def test_map_is_continuous_at_the_linear_region_edge():
    rng = np.random.default_rng(0)
    y = rng.normal(size=(1000, 3))
    y /= np.abs(y).max(-1, keepdims=True)                           # ||y||_inf = 1
    for eps in (1e-3, 1e-6, 1e-9):
        lo, hi = C.contract64(y * (1 - eps)), C.contract64(y * (1 + eps))
        assert np.abs(hi - lo).max() <= 3 * eps
    # the fp32 lookup: u at m = 1 and at the next float above differ by a few ulps of u only
    res = 128
    o = (y * 1.0).astype(f32)
    d = np.zeros_like(o)
    t = np.zeros((len(o), 1), f32)
    u1 = C.contract_u(o, d, t, (0, 0, 0), 1.0, res)
    u2 = C.contract_u(np.nextafter(o, f32(2) * np.sign(o)).astype(f32), d, t, (0, 0, 0), 1.0, res)
    assert np.abs(u2 - u1).max() < 1e-4


def test_map_is_monotone_along_rays():
    """along a ray from the center each contracted coordinate moves one way and ||v||_inf grows (fp64 map); the fp32
    lookup's cell index never moves back by more than rounding at a cell plane"""
    rng = np.random.default_rng(1)
    d = rng.normal(size=(500, 3))
    t = np.geomspace(1e-3, 1e8, 4000)
    v = C.contract64(d[:, None, :] * t[None, :, None])
    dv = np.diff(v, axis=1)
    assert (dv * np.sign(d)[:, None, :] >= -1e-15).all()
    n = np.abs(v).max(-1)
    assert (np.diff(n, axis=1) >= -1e-15).all() and (n < 2).all()
    # rays from anywhere: ||v||_inf of x far out along the ray grows towards 2
    o = rng.uniform(-3, 3, (500, 3))
    far = C.contract64(o[:, None, :] + d[:, None, :] * t[None, -500:, None])
    nf = np.abs(far).max(-1)
    assert (np.diff(nf, axis=1) >= -1e-12).all()
    # fp32 lookup along the ray of the same directions: u matches the fp64 map to fp32 accuracy
    u = C.contract_u(np.zeros((500, 3), f32), d.astype(f32), np.broadcast_to(t.astype(f32), (500, 4000)), (0, 0, 0),
                     1.0, 128)
    u64 = (C.contract64(d.astype(f32).astype(np.float64)[:, None, :] * t.astype(f32).astype(np.float64)[None, :, None])
           + 2) * 0.25 * 128
    assert np.abs(u - u64).max() < 1e-3


@pytest.mark.parametrize("res", [8, 33, 128])
def test_lattice_inverse_round_trips(res):
    a = _axis(res).astype(np.float64)
    v = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    inner = np.abs(v).max(-1) < 2
    back = C.contract64(C.uncontract64(v[inner]))
    assert np.abs(back - v[inner]).max() < 1e-12
    # lattice_world: the world points, contracted again with the same center and radius, land on the lattice
    center, radius = (0.25, -1.0, 3.0), 1.33
    x, far = C.lattice_world(a, center, radius)
    assert np.array_equal(far.reshape(-1), ~inner)
    y = (x.reshape(-1, 3)[inner].astype(np.float64) - np.asarray(center, f32)) / float(f32(radius))
    # fp32 rounding of the world point moves it by a relative 2^-24, which the contraction amplifies near n = 2
    n = np.abs(v[inner]).max(-1)
    err = np.abs(C.contract64(y) - v[inner]).max(-1)
    assert (err <= 1e-6 * (1 + 1 / (2 - n) ** 2)).all()


@pytest.mark.parametrize("res", [8, 16, 64])
def test_points_at_infinity_give_the_outer_shell(res):
    """σ = 0 everywhere at finite points: exactly the outer two-cell shell is occupied, and no finite point is
    evaluated as NaN"""
    bits = C.build(_axis(res), (0, 0, 0), 1.0, lambda x: np.zeros(x.shape[:-1], f32), 0.01)
    occ = O.unpack_bits(bits, res)
    assert np.array_equal(occ, C.shell(res))
    # the shell starts at ||x - c||_inf = radius * res / 8: samples beyond it are kept whatever the grid says
    o = np.zeros((1, 3), f32)
    d = np.array([[0, 0, 1]], f32)
    t = np.array([[res / 8 * 0.98, res / 8 * 1.02, 1e8, np.inf]], f32)
    assert C.kept(bits, res, (0, 0, 0), 1.0, o, d, t).tolist() == [[False, True, True, True]]


def test_nan_inf_and_extreme_samples_are_kept():
    res = 16
    bits = O.pack_bits(np.zeros((res,) * 3, bool))
    o = np.zeros((1, 3), f32)
    d = np.array([[0.3, -0.2, 1]], f32)
    t = np.array([[0.5, np.nan, np.inf, -np.inf, f32(3e38), 1e30]], f32)
    assert C.kept(bits, res, (0, 0, 0), 1.0, o, d, t).tolist() == [[False, True, True, True, True, True]]
    # m > 2^24: 2 - q rounds to 2 and u reaches res
    u = C.contract_u(o, np.array([[0, 0, 1]], f32), np.array([[2.0 ** 25]], f32), (0, 0, 0), 1.0, res)
    assert u[0, 0, 2] == res


def llff_wall_scene(H=63, W=84, focal=68.0, S=128, depth=3.0, k=400.0):
    """rays of one identity camera with LLFF's field of view (focal / W about 0.8), inverse-depth samples over [1, 0]
    as sample_depth draws them in val mode, and the analytic wall σ = softplus(k (z - depth)) -> (o, d, t, sigma_fn)"""
    v, u = np.meshgrid(np.arange(H, dtype=f32) + f32(0.5), np.arange(W, dtype=f32) + f32(0.5), indexing="ij")
    d = np.stack([(u - f32(W / 2)) / f32(focal), (v - f32(H / 2)) / f32(focal), np.ones_like(u)], -1).reshape(-1, 3)
    kk = np.arange(S, dtype=f32)
    disparity = (kk + f32(0.5)) / f32(S) * f32(-1) + f32(1)
    t = np.broadcast_to(f32(1) / (disparity + f32(1e-8)), (len(d), S)).copy()
    sigma_fn = lambda x: np.logaddexp(0, k * (x[..., 2].astype(np.float64) - depth)).astype(f32)
    return np.zeros_like(d), d.astype(f32), t, sigma_fn


@pytest.mark.parametrize("res,grid_kept,both_kept", [(128, 48, 16), (256, 45, 13)])
def test_llff_wall_scene_kept_counts(res, grid_kept, both_kept):
    """A wall at depth 3 in front of the camera, inverse depth, 128 samples; contracted grid with the camera at the
    center and radius 1.33 (the LLFF loader's near bound), thres 0.01.  Termination alone (eps 1e-4, window 16) keeps
    96 of 128 samples per ray (0.75); the grid keeps grid_kept (about 0.35) and grid + termination both_kept (about
    0.1).  Every skipped sample's σ is below thres."""
    o, d, t, sigma_fn = llff_wall_scene()
    center, radius = (0.0, 0.0, 0.0), 1.33
    bits = C.build(_axis(res), center, radius, sigma_fn, 0.01)
    keep = C.kept(bits, res, center, radius, o, d, t)
    sigma = sigma_fn(o[:, None] + d[:, None] * t[..., None])
    assert (sigma[~keep] < 0.01).all()
    term = T.evaluated(sigma, t, d, 1e-4, 16)
    both = T.evaluated(sigma, t, d, 1e-4, 16, keep)
    assert (term.sum(1) == 96).all()
    assert (keep.sum(1) == grid_kept).all(), np.unique(keep.sum(1))
    assert (both.sum(1) == both_kept).all(), np.unique(both.sum(1))
