"""Training-time occupancy grids without a GPU: the C ABI's new entry points, which pass Graph.set_training_occupancy
routes where (train and test-optim only, next to an untouched set_occupancy), and the engine gate of
ops.mlp_forward_grid."""
import pytest
import torch

import common


def test_abi_declares_the_entry_points():
    import test_abi
    from sparf_b200 import _lib
    names = {"sparf_mlp_forward_tape_rows", "sparf_mlp_backward_tape_rows", "sparf_compact_scatter", "sparf_compact_gather",
             "sparf_compact_ray_sum"}
    assert names <= set(test_abi._header_functions())
    assert names <= set(_lib.exported_symbols())


def test_simt_engine_is_refused_before_any_work():
    from sparf_b200 import _lib, ops
    with pytest.raises(ValueError, match="simt_fp32"):
        ops.mlp_forward_grid(ops.MLPSpec(), torch.zeros(1, 3), torch.zeros(1, 3), torch.zeros(1, 1), None, [],
                             engine=_lib.ENGINE_SIMT_FP32)


@pytest.fixture
def routed(monkeypatch):
    """a CPU Graph whose three sample paths only record which one ran"""
    from sparf_b200 import occupancy
    from sparf_b200.renderer import Graph
    opt = common.make_opt(S=4, S_fine=4, fine=True)
    net = Graph(opt, torch.device("cpu"))
    calls = []
    monkeypatch.setattr(occupancy, "train_forward_samples", lambda nerf, g, *a: calls.append(("train", nerf, g)))
    monkeypatch.setattr(occupancy, "forward_samples", lambda nerf, g, *a: calls.append(("inference", nerf, g)))
    for m in net.get_network_components():
        monkeypatch.setattr(m, "forward_samples", lambda *a, _m=m, **k: calls.append(("dense", _m, None)))

    def route(which, mode, grad=False):
        calls.clear()
        with torch.set_grad_enabled(grad):
            net._forward_samples(net.get_network_components()[which], which, opt, None, None, None, mode)
        return calls[0][0], calls[0][2]

    return net, route


def test_training_grids_apply_in_train_and_test_optim_only(routed):
    net, route = routed
    g, gf = object(), object()
    net.set_training_occupancy(g, gf)
    for grad in (False, True):
        assert route(0, "train", grad) == ("train", g)
        assert route(1, "train", grad) == ("train", gf)
        assert route(0, "test-optim", grad) == ("train", g)
    for mode in ("val", "eval", "test"):
        assert route(0, mode) == ("dense", None)
    net.set_training_occupancy(g)                 # no fine grid: the fine pass stays dense
    assert route(1, "train") == ("dense", None)
    net.set_training_occupancy(None)
    assert route(0, "train") == ("dense", None)


def test_inference_grids_keep_their_meaning(routed):
    net, route = routed
    g, t = object(), object()
    net.set_occupancy(g)
    assert route(0, "val") == ("inference", g)
    assert route(0, "train") == ("dense", None)
    net.set_training_occupancy(t)
    assert route(0, "val") == ("inference", g)
    assert route(0, "train") == ("train", t)
    assert route(0, "val", grad=True) == ("dense", None)
