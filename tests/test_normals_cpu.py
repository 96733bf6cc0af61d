"""CPU-side checks of the normal maps: the new C entry point is declared and bound, ops.density_gradient and
Graph.set_normals reject bad arguments before any library call, and the fp64 oracle of the GPU tests
(tests/normals_oracle.py) agrees with torch autograd."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C2F = (0.1, 0.5)
TRUNK_KEYS = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], [])


def test_density_gradient_is_declared_and_bound():
    from sparf_b200 import _lib
    src = open(os.path.join(ROOT, "include", "sparf_b200.h")).read()
    assert re.search(r"int sparf_density_gradient\(const SparfMLP\* mlp, int32_t engine, int64_t M, const float\* points, "
                     r"float\* grad_points,\s+void\* workspace, size_t workspace_bytes, sparf_stream_t stream\);", src)
    assert "sparf_density_gradient" in _lib.exported_symbols()


@pytest.fixture
def no_library(monkeypatch):
    from sparf_b200 import _lib

    def refuse():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_density_gradient_rejects_bad_arguments(no_library):
    from sparf_b200 import ops
    spec = ops.MLPSpec(barf_c2f=C2F)
    params = [torch.zeros(1)] * 16
    with pytest.raises(ValueError, match="CUDA"):
        ops.density_gradient(spec, torch.zeros(4, 3), params, progress=torch.tensor(0.3))
    with pytest.raises(ValueError, match=r"\[\.\.\., 3\]"):
        ops.density_gradient(spec, torch.zeros(4, 2), params, progress=torch.tensor(0.3))
    with pytest.raises(ValueError, match=r"\[\.\.\., 3\]"):
        ops.density_gradient(spec, [0.0, 0.0, 0.0], params, progress=torch.tensor(0.3))
    if torch.cuda.is_available():
        pts = torch.zeros(4, 3, device="cuda")
        with pytest.raises(ValueError, match="2 \\* n_trunk"):
            ops.density_gradient(spec, pts, params[:15], progress=torch.tensor(0.3))
        with pytest.raises(ValueError, match="engine"):
            ops.density_gradient(spec, pts, params, progress=torch.tensor(0.3), engine=7)
        with pytest.raises(ValueError, match="progress"):
            ops.density_gradient(spec, pts, params)


def test_set_normals_rejects_non_bool():
    import common
    from sparf_b200.renderer import Graph
    net = Graph(common.make_opt(S=4, S_fine=4, fine=True), torch.device("cpu"))
    assert not getattr(net, "_normals", False)
    for bad in (1, "yes", None, 0.5):
        with pytest.raises(ValueError):
            net.set_normals(bad)
    net.set_normals()
    assert net._normals is True
    net.set_normals(False)
    assert net._normals is False


def _net(seed):
    import common
    opt = common.make_opt(barf_c2f=C2F)
    return {k: v for k, v in common.det_weights(opt, seed, progress=0.3).items()}


def test_point_gradient_oracle_matches_autograd():
    from density_oracle import raw_density
    from normals_oracle import point_gradient
    sd = _net(5)
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(64, 3, generator=g, dtype=torch.float64) * 3 - 1.5)
    p = {k: sd[k].double() for k in TRUNK_KEYS}
    p["progress"] = sd["progress"]
    xg = x.clone().requires_grad_(True)
    raw, _ = raw_density(p, xg, barf_c2f=C2F)
    (ref,) = torch.autograd.grad(raw.sum(), xg)
    got = point_gradient({k: sd[k].numpy() for k in TRUNK_KEYS}, x.numpy(), progress=float(sd["progress"]), barf_c2f=C2F)
    assert np.abs(got - ref.numpy()).max() <= 1e-10 * np.abs(ref.numpy()).max()


def test_normal_map_oracle_matches_autograd():
    """the oracle's normal map on 6 rays of 40 samples against a torch fp64 autograd restatement"""
    import torch.nn.functional as F
    from density_oracle import raw_density
    from normals_oracle import normal_map
    from oracle import sparf_oracle as O
    sd = _net(9)
    g = torch.Generator().manual_seed(9)
    o = torch.rand(6, 3, generator=g, dtype=torch.float64) - 0.5
    d = torch.randn(6, 3, generator=g, dtype=torch.float64)
    t = torch.linspace(0.1, 2.0, 40, dtype=torch.float64).expand(6, 40).contiguous()
    got, w = normal_map({k: sd[k].numpy() for k in TRUNK_KEYS}, o.numpy(), d.numpy(), t.numpy(),
                        progress=float(sd["progress"]), barf_c2f=C2F)
    p = {k: sd[k].double() for k in TRUNK_KEYS}
    p["progress"] = sd["progress"]
    x = (o[:, None] + d[:, None] * t[..., None]).requires_grad_(True)
    raw, _ = raw_density(p, x, barf_c2f=C2F)
    (gx,) = torch.autograd.grad(raw.sum(), x)
    n = torch.where(gx.norm(dim=-1, keepdim=True) > 0, -gx / gx.norm(dim=-1, keepdim=True), torch.zeros_like(gx))
    w_ref = O.composite(d[None], F.softplus(raw.detach())[None], torch.zeros(1, 6, 40, 3, dtype=torch.float64), t[None])
    w_ref = w_ref["weights"][0, ..., 0]
    ref = (w_ref[..., None] * n).sum(1)
    assert np.abs(w - w_ref.numpy()).max() <= 1e-12
    assert np.abs(got - ref.numpy()).max() <= 1e-10
    assert (np.linalg.norm(got, axis=-1) <= w.sum(1) + 1e-12).all()     # |normal| <= opacity
