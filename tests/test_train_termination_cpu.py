"""Early ray termination in training steps without a GPU: NumPy oracles of the appending window compaction and of the
segment ray sum (used by tests/test_train_termination.py against the kernels), checked here against the per-window
compaction of termination_oracle and against float64 sums; the C ABI's new entry points; the argument checks of
Graph.set_training_termination; and the routing of the training passes."""
import numpy as np
import pytest
import torch

import common
import occupancy_oracle as O
import termination_oracle as T

f32 = np.float32


def append_oracle(origins, dirs, t, window, alive_masks, keep=None):
    """what the appending compaction writes over every window w (alive rays alive_masks[w], grid kept mask `keep` [R,S]
    or None): (ends [W+1] int64, sample_idx [K], origins_k [K,3], dirs_k [K,3], t_k [K,1]); window w's rows are
    [ends[w], ends[w+1]), in increasing r*S + k"""
    o, d, t = np.asarray(origins, f32), np.asarray(dirs, f32), np.asarray(t, f32)
    R, S = t.shape
    ends, parts = [0], []
    for w, k0 in enumerate(range(0, S, window)):
        k1 = min(k0 + window, S)
        idx, o_k, d_k, t_k = T.compact(o, d, t, k0, k1, np.asarray(alive_masks[w], np.uint8))
        if keep is not None:
            sel = np.asarray(keep, bool).reshape(-1)[idx]
            idx, o_k, d_k, t_k = idx[sel], o_k[sel], d_k[sel], t_k[sel]
        parts.append((idx, o_k, d_k, t_k))
        ends.append(ends[-1] + len(idx))
    cat = [np.concatenate([p[i] for p in parts]) if parts else np.zeros(0) for i in range(4)]
    return [np.asarray(ends, np.int64)] + cat


def segment_ray_sum_oracle(R, S, ends, idx, src):
    """dst [R, width]: per ray, the rows of each segment [ends[w], ends[w+1]) with idx // S == r, in segment order and
    increasing k within one, added sequentially in fp32 from 0"""
    src = np.asarray(src, f32)
    dst = np.zeros((R, src.shape[1]), f32)
    for w in range(len(ends) - 1):
        for k in range(int(ends[w]), int(ends[w + 1])):
            r = int(idx[k]) // S
            dst[r] = (dst[r] + src[k]).astype(f32)
    return dst


def _scene(rng, R, S):
    o = rng.normal(0, 0.4, (R, 3)).astype(f32)
    d = rng.normal(0, 1, (R, 3)).astype(f32)
    t = np.sort(rng.uniform(0.0, 2.0, (R, S)), 1).astype(f32)
    return o, d, t


@pytest.mark.parametrize("R,S,window", [(1, 1, 1), (7, 20, 6), (50, 64, 16), (50, 64, 64)])
@pytest.mark.parametrize("with_grid", [False, True])
def test_append_oracle_is_the_concatenated_windows(R, S, window, with_grid):
    """with the alive masks of termination_oracle.evaluated, the appended rows are exactly its evaluated samples, each
    window's block in increasing r*S + k, and equal to the concatenation of termination_oracle.compact per window"""
    rng = np.random.default_rng(R + S + window)
    o, d, t = _scene(rng, R, S)
    sigma = rng.exponential(3.0, (R, S)).astype(f32)
    keep = None
    grid = None
    if with_grid:
        res = 5
        bits = O.pack_bits(rng.random((res,) * 3) < 0.5)
        grid = (bits, res, -0.8, 0.8)
        keep = O.kept(*grid, o, d, t)
    ev = T.evaluated(sigma, t, d, 1e-2, window, keep)
    # the alive mask of each window, replayed with the oracle's own update
    masks, alive, tau = [], np.ones(R, np.uint8), np.zeros(R, f32)
    for k0 in range(0, S, window):
        k1 = min(k0 + window, S)
        masks.append(alive != 0)
        if k1 < S:
            tau, alive = T.update(np.where(ev, sigma, f32(0)), t, d, k0, k1, T.tau_max(1e-2), tau, alive)
    ends, idx, o_k, d_k, t_k = append_oracle(o, d, t, window, masks, keep)
    assert sorted(idx.tolist()) == np.nonzero(ev.reshape(-1))[0].tolist()
    W = len(ends) - 1
    for w in range(W):
        seg = idx[ends[w]:ends[w + 1]]
        assert (np.diff(seg) > 0).all()
        k0, k1 = w * window, min((w + 1) * window, S)
        want = T.compact(o, d, t, k0, k1, masks[w].astype(np.uint8), grid)
        for a, b in zip((seg, o_k[ends[w]:ends[w + 1]], d_k[ends[w]:ends[w + 1]], t_k[ends[w]:ends[w + 1]]), want):
            assert a.tobytes() == b.tobytes()
    assert np.array_equal(o_k, o[idx // S]) and np.array_equal(t_k[:, 0], t.reshape(-1)[idx])


def test_segment_ray_sum_oracle_is_the_per_ray_sum_in_k_order():
    """the segment order of the appended rows gives every ray its rows in increasing k, so the oracle equals the grid
    path's per-ray sequential sum over the sorted kept set; against float64 it is off by rounding only"""
    rng = np.random.default_rng(3)
    R, S, window = 30, 40, 8
    o, d, t = _scene(rng, R, S)
    masks = [rng.random(R) < p for p in (1.0, 0.8, 0.5, 0.0, 0.3)]
    ends, idx, *_ = append_oracle(o, d, t, window, masks)
    src = rng.normal(0, 1, (len(idx), 3)).astype(f32)
    got = segment_ray_sum_oracle(R, S, ends, idx, src)
    order = np.argsort(idx, kind="stable")
    want = np.zeros((R, 3), f32)
    for k in order:                               # the grid path: kept rows sorted by sample, each ray's in increasing k
        want[idx[k] // S] = (want[idx[k] // S] + src[k]).astype(f32)
    assert got.tobytes() == want.tobytes()
    exact = np.zeros((R, 3))
    np.add.at(exact, idx // S, src.astype(np.float64))
    assert np.abs(got - exact).max() < 1e-5


def test_abi_declares_the_entry_points():
    import test_abi
    from sparf_b200 import _lib
    names = {"sparf_mlp_forward_tape_span", "sparf_termination_append", "sparf_contracted_append",
             "sparf_compact_scatter_span", "sparf_compact_gather_span", "sparf_compact_ray_sum_segments"}
    assert names <= set(test_abi._header_functions())
    assert names <= set(_lib.exported_symbols())


def test_set_training_termination_checks_its_arguments():
    from sparf_b200.renderer import Graph
    net = Graph(common.make_opt(S=4, S_fine=4, fine=True), torch.device("cpu"))
    for eps, window in ((-1e-4, 16), (1.0, 16), (float("nan"), 16), ("1e-4", 16), (1e-4, 0), (1e-4, 2.5), (1e-4, True)):
        with pytest.raises(ValueError):
            net.set_training_termination(eps, window)
    net.set_training_termination(1e-4, 16)
    assert net._train_termination == (1e-4, 16)
    net.set_training_termination(0, 1)
    assert net._train_termination == (0.0, 1)
    net.set_training_termination(None)
    assert net._train_termination is None


def test_simt_engine_is_refused_before_any_work():
    from sparf_b200 import _lib, ops
    with pytest.raises(ValueError, match="simt_fp32"):
        ops.mlp_forward_terminated(ops.MLPSpec(), torch.zeros(1, 3), torch.zeros(1, 3), torch.zeros(1, 1), None, 1e-4, 16, [],
                                   engine=_lib.ENGINE_SIMT_FP32)


def test_training_termination_routes_train_and_test_optim_only(monkeypatch):
    from sparf_b200 import occupancy, termination
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=4, S_fine=4, fine=True)
    net = Graph(opt, torch.device("cpu"))
    calls = []
    monkeypatch.setattr(termination, "train_forward_samples",
                        lambda nerf, g, eps, window, *a: calls.append(("term", g, eps, window)))
    monkeypatch.setattr(occupancy, "train_forward_samples", lambda nerf, g, *a: calls.append(("grid", g)))
    for m in net.get_network_components():
        monkeypatch.setattr(m, "forward_samples", lambda *a, **k: calls.append(("dense",)))

    def route(which, mode):
        calls.clear()
        net._forward_samples(net.get_network_components()[which], which, opt, None, None, None, mode)
        return calls[0]

    g = object()
    net.set_training_occupancy(g)
    net.set_training_termination(1e-3, 8)
    assert route(0, "train") == ("term", g, 1e-3, 8)
    assert route(1, "train") == ("term", None, 1e-3, 8)      # no fine grid: termination alone on the fine pass
    assert route(0, "test-optim") == ("term", g, 1e-3, 8)
    assert route(0, "val") == ("dense",)
    net.set_training_termination(None)
    assert route(0, "train") == ("grid", g)
    assert route(1, "train") == ("dense",)
