"""Early ray termination without a GPU: properties of the NumPy restatement (tests/termination_oracle.py) that the GPU
tests hold the kernels to, its op order against a scalar restatement, and the C ABI's new entry points and workspace
sizes."""
import itertools

import numpy as np
import pytest

import occupancy_oracle as O
import termination_oracle as T

f32 = np.float32


def _scene(seed, R=200, S=40):
    """rays with sorted t, σ from empty to opaque per ray"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(R, 3)).astype(f32)
    t = np.sort(rng.uniform(1, 4, (R, S)), 1).astype(f32)
    sigma = (rng.random((R, S)) * rng.choice([0.0, 0.5, 5.0, 50.0], R)[:, None]).astype(f32)
    return sigma, t, d


def _grid_keep(seed, t, d):
    rng = np.random.default_rng(seed)
    res = 8
    o = rng.uniform(-2, 2, (t.shape[0], 3)).astype(f32)
    bits = O.pack_bits(rng.random((res,) * 3) < 0.4)
    return O.kept(bits, res, -1.0, 1.0, o, d * f32(0.2), t)


@pytest.mark.parametrize("window", [1, 7, 16, 40, 64])
def test_eps_zero_or_one_window_keeps_everything_the_grid_keeps(window):
    sigma, t, d = _scene(1)
    keep = _grid_keep(2, t, d)
    for g in (None, keep):
        want = np.ones_like(keep) if g is None else keep
        assert np.array_equal(T.evaluated(sigma, t, d, 0.0, window, g), want)
        assert np.array_equal(T.evaluated(sigma, t, d, 0.5, 40, g), want)     # window >= S: one window, no update
    # and a positive eps does terminate rays here
    assert not T.evaluated(sigma, t, d, 1e-4, 8).all()


def test_masks_are_monotone_in_eps():
    sigma, t, d = _scene(3)
    keep = _grid_keep(4, t, d)
    for window, g in itertools.product((1, 5, 16), (None, keep)):
        masks = [T.evaluated(sigma, t, d, eps, window, g) for eps in (0.0, 1e-6, 1e-4, 1e-2, 0.5)]
        for a, b in zip(masks, masks[1:]):
            assert not (b & ~a).any()                  # larger eps evaluates a subset
        assert masks[-1].sum() < masks[0].sum()


@pytest.mark.parametrize("window", [1, 6, 16])
def test_a_terminated_ray_skips_all_its_later_samples(window):
    sigma, t, d = _scene(5)
    ev = T.evaluated(sigma, t, d, 1e-3, window)
    S = t.shape[1]
    first_windows = np.arange(S) // window
    for r in range(t.shape[0]):
        dead = [w for w in range(first_windows[-1] + 1) if not ev[r, first_windows == w].any()]
        if dead:                                      # without a grid: whole windows, and every one after the first
            assert not ev[r, first_windows >= dead[0]].any()
            assert ev[r, first_windows < dead[0]].all()
    assert (~ev).any() and ev[:, :window].all()


def test_nan_sigma_keeps_the_ray_alive():
    sigma, t, d = _scene(6, R=50)
    sigma[:] = 1e4
    sigma[::2, 3] = np.nan
    ev = T.evaluated(sigma, t, d, 1e-4, 4)
    assert ev[::2].all()
    assert not ev[1::2, 4:].any()
    # a grid-skipped sample counts as σ = 0: no optical depth, so no termination from it
    keep = np.ones_like(ev)
    keep[:, :4] = False
    assert not T.evaluated(sigma, t, d, 1e-4, 4, keep)[:, :4].any()
    assert not T.evaluated(sigma, t, d, 1e-4, 4, keep)[1::2, 8:].any()


def test_update_matches_a_scalar_restatement():
    """tau += σ_k * (gap_k * len) in k order with each op rounded, len = sqrt((dx dx + dy dy) + dz dz), the last gap 1e10;
    τ > fp32(-ln eps) kills; NaN τ lives; dead rays are untouched"""
    rng = np.random.default_rng(7)
    R, S, k0, k1 = 40, 9, 3, 9
    sigma = rng.exponential(2, (R, S)).astype(f32)
    sigma[0, 5], sigma[1, 4], sigma[2, 8] = np.nan, np.inf, 1e-12
    t = np.sort(rng.uniform(0, 3, (R, S)), 1).astype(f32)
    d = rng.normal(size=(R, 3)).astype(f32)
    d[3] = 0
    tau0 = rng.uniform(0, 2, R).astype(f32)
    alive0 = (rng.random(R) < 0.8).astype(np.uint8)
    tmax = T.tau_max(1e-3)
    assert tmax == f32(6.9077554)
    tau, alive = T.update(sigma, t, d, k0, k1, tmax, tau0, alive0)
    for r in range(R):
        if not alive0[r]:
            assert tau[r] == tau0[r] and alive[r] == 0
            continue
        ln = np.sqrt(f32(f32(d[r, 0] * d[r, 0]) + f32(d[r, 1] * d[r, 1])) + f32(d[r, 2] * d[r, 2]))
        acc = tau0[r]
        for k in range(k0, k1):
            gap = f32(t[r, k + 1] - t[r, k]) if k + 1 < S else f32(1e10)
            with np.errstate(invalid="ignore", over="ignore"):
                acc = f32(acc + f32(sigma[r, k] * f32(gap * ln)))
        assert tau[r].tobytes() == acc.tobytes(), r
        assert alive[r] == (0 if acc > tmax else 1), r
    assert np.isnan(tau[0]) and alive[0] == alive0[0]
    assert T.tau_max(0.0) == np.inf


def test_compaction_selects_the_window_of_alive_rays():
    rng = np.random.default_rng(8)
    R, S = 30, 11
    o = rng.uniform(-2, 2, (R, 3)).astype(f32)
    d = rng.normal(size=(R, 3)).astype(f32)
    t = rng.uniform(0, 2, (R, S)).astype(f32)
    alive = (rng.random(R) < 0.5).astype(np.uint8)
    res = 4
    bits = O.pack_bits(rng.random((res,) * 3) < 0.5)
    keep = O.kept(bits, res, -1.0, 1.0, o, d, t)
    for k0, k1 in ((0, 11), (3, 4), (8, 11)):
        for a, g in itertools.product((None, alive), (None, (bits, res, -1.0, 1.0))):
            idx, ok, dk, tk = T.compact(o, d, t, k0, k1, a, g)
            r, k = idx // S, idx % S
            want = [(rr, kk) for rr in range(R) for kk in range(k0, k1)
                    if (a is None or a[rr]) and (g is None or keep[rr, kk])]
            assert list(zip(r.tolist(), k.tolist())) == want
            assert np.array_equal(ok, o[r]) and np.array_equal(dk, d[r]) and np.array_equal(tk[:, 0], t[r, k])


def test_abi_declares_the_termination_entry_points():
    import test_abi
    from sparf_b200 import _lib
    names = {"sparf_termination_workspace_bytes", "sparf_termination_count", "sparf_termination_emit",
             "sparf_termination_update"}
    assert names <= set(test_abi._header_functions())
    assert names <= set(_lib.exported_symbols())


def test_workspace_bytes():
    """the occupancy compaction's workspace over R x window samples"""
    from sparf_b200 import _lib
    L = _lib.lib()
    for R, W in ((1, 1), (3, 700), (131070, 32), (524293, 4096), (1 << 40, 64)):
        assert L.sparf_termination_workspace_bytes(R, W) == L.sparf_occupancy_workspace_bytes(R, W), (R, W)
        tiles = -(-R * W // 2048)
        assert L.sparf_termination_workspace_bytes(R, W) == -(-tiles * 2048 // 256) * 256 + 8 * tiles
    assert L.sparf_termination_workspace_bytes(-1, 4) == 0 and L.sparf_termination_workspace_bytes(4, 0) == 0
    assert L.sparf_termination_workspace_bytes(1 << 40, 1 << 20) == 0
