"""The fp64 reference that starts from the engines' fp32 encoding (tests/engine_oracle.py), checked on the CPU: without
rounding it is the oracle's graph; with rounding its x and band arguments are the fp32 values the encoders compute; its
straight-through gradients are those of the unrounded graph up to the rounding; the margin mask flags what it says."""
import pytest
import torch

import density_oracle as D
import engine_oracle as E
from oracle import sparf_oracle as O
from sparf_b200.ops import MLPSpec

SPECS = {
    "default": dict(),
    "w136_layerwise": dict(width=136, n_trunk=4, skip_layer=2, L_xyz=6, L_view=2, head_width=64),
    "w256_short_noskip": dict(width=256, n_trunk=3, skip_layer=-1, L_xyz=4, L_view=1),
}
C2F = (0.4, 0.7)


def _inputs(R, S, seed, dtype=torch.float32):
    return tuple(x.to(dtype) for x in E.ray_inputs(R, S, seed))


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("c2f", [None, C2F])
@pytest.mark.parametrize("name", list(SPECS))
def test_unrounded_reference_is_the_oracle_graph(name, c2f):
    spec = MLPSpec(barf_c2f=c2f, **SPECS[name])
    params = [p.double() for p in E.make_params(spec, seed=3)]
    o, d, t, noise = _inputs(5, 7, seed=1, dtype=torch.float64)
    ref = E.mlp_reference(spec, params, o, d, t, noise=noise, progress=0.6, rounded=False)
    sd = dict(zip(E.param_keys(spec), params), progress=torch.tensor(0.6))
    skip = (spec.skip_layer,) if spec.skip_layer >= 0 else ()
    pts = o[:, None] + d[:, None] * t[..., None]
    dens, rgb = O.mlp_forward(sd, pts[None], d[None], L_3D=spec.L_xyz, L_view=spec.L_view, skip=skip, barf_c2f=c2f,
                              noise=noise[None])
    assert _rel(ref["sigma"], dens[0]) < 1e-12 and _rel(ref["rgb"], rgb[0]) < 1e-12
    assert len(ref["pre"]) == spec.n_trunk + 1
    # density queries: the trunk alone at the points
    trunk = params[:2 * spec.n_trunk]
    pts = pts.reshape(-1, 3)
    dref = E.density_reference(spec, trunk, pts, progress=0.6, rounded=False)
    raw, feat = D.raw_density(sd, pts, L_3D=spec.L_xyz, skip=skip, barf_c2f=c2f)
    assert _rel(dref["raw"], raw) < 1e-12 and _rel(dref["feat"], feat) < 1e-12
    assert torch.equal(dref["raw"], ref["raw"].reshape(-1)) or _rel(dref["raw"], ref["raw"].reshape(-1)) < 1e-12


def test_rounded_inputs_are_the_encoders_fp32_values():
    """x = o + d t and arg = x * 2^j float32(pi) hold the fp32 results of those two-op / one-op products bit for bit,
    and the unit direction is the fp32 quotient."""
    spec = MLPSpec()
    params = [p.double() for p in E.make_params(spec, seed=4)]
    o, d, t, _ = _inputs(9, 11, seed=2)
    ref = E.mlp_reference(spec, params, o.double(), d.double(), t.double())
    x32 = o[:, None] + d[:, None] * t[..., None]
    f = torch.tensor([2.0 ** j * 3.14159274101257324 for j in range(spec.L_xyz)], dtype=torch.float32)
    assert torch.equal(ref["x"], x32.double())
    assert torch.equal(ref["arg"], (x32[..., None] * f).double())
    assert not torch.equal(ref["x"], o.double()[:, None] + d.double()[:, None] * t.double()[..., None])
    u32 = d / d.norm(dim=-1, keepdim=True)
    assert (ref["u"] - u32.double()).abs().max().item() <= 2 ** -23
    fv = f[:spec.L_view]
    assert torch.equal(ref["arg_view"], (ref["u"].float()[..., None] * fv).double())
    pts = x32.reshape(-1, 3)
    dref = E.density_reference(spec, params[:16], pts.double())
    assert torch.equal(dref["arg"], (pts[..., None] * f).double())


@pytest.mark.parametrize("name", list(SPECS))
def test_straight_through_gradients_are_the_unrounded_ones_up_to_the_rounding(name):
    """Autograd through the rounded reference = the fp64 gradient at the rounded point: within the rounding
    perturbation of the fp64 gradient at the exact point, for the ray inputs and every parameter."""
    spec = MLPSpec(barf_c2f=C2F, **SPECS[name])
    o, d, t, noise = _inputs(6, 9, seed=5)
    g = torch.Generator().manual_seed(9)
    gs, gc = torch.randn(6, 9, generator=g).double(), torch.randn(6, 9, 3, generator=g).double()
    res = {}
    for rounded in (False, True):
        params = [p.double().requires_grad_(True) for p in E.make_params(spec, seed=6)]
        oo, dd = o.double().requires_grad_(True), d.double().requires_grad_(True)
        ref = E.mlp_reference(spec, params, oo, dd, t.double(), noise=noise.double(), progress=0.6, rounded=rounded)
        ((ref["sigma"] * gs).sum() + (ref["rgb"] * gc).sum()).backward()
        res[rounded] = [oo.grad, dd.grad] + [p.grad for p in params]
    # x moves by <= 2^-23 relative, the top band's argument by up to 2^-23 |x| 2^(L-1) pi (|x| < 5.2 here); the
    # gradients move by that times the net's sensitivity (measured: <= 0.1 of it on these nets)
    arg_ulp = 2.0 ** -23 * 5.2 * 2 ** (spec.L_xyz - 1) * 3.15
    for i, (a, b) in enumerate(zip(res[True], res[False])):
        e = _rel(a, b)
        assert e < 2 * arg_ulp, (i, e)
    assert any(not torch.equal(a, b) for a, b in zip(res[True], res[False])), "rounding changed nothing"


def test_straight_through_point_gradient_of_the_density_reference():
    """density_reference's points enter exactly (they are fp32 already): only the band arguments are rounded."""
    spec = MLPSpec(**SPECS["w256_short_noskip"])
    params = [p.double() for p in E.make_params(spec, seed=8)][:2 * spec.n_trunk]
    pts = (torch.rand(50, 3, generator=torch.Generator().manual_seed(2)) * 3 - 1.5)
    grads = []
    for rounded in (False, True):
        x = pts.double().requires_grad_(True)
        E.density_reference(spec, params, x, rounded=rounded)["raw"].sum().backward()
        grads.append(x.grad)
    assert _rel(grads[1], grads[0]) < 1e-4


def test_margin_mask_flags_exactly_the_small_preactivations():
    z0 = torch.tensor([[1.0, -2.0, 3.0], [0.5, 1e-9, -1.0], [2.0, 2.0, 2.0], [-1.0, 1.0, -1e-6]], dtype=torch.float64)
    z1 = torch.tensor([[1.0, 1.0], [1.0, 1.0], [3e-7, 4.0], [1.0, 1.0]], dtype=torch.float64)
    rms0, rms1 = z0.pow(2).mean().sqrt().item(), z1.pow(2).mean().sqrt().item()
    mu = 2.0 ** -14
    assert 1e-6 < mu * rms0 and 3e-7 < mu * rms1 and 1e-9 < mu * rms0
    m = E.margin_mask([z0, z1], mu)
    assert m.tolist() == [False, True, True, True]
    # one layer alone; leading dimensions kept
    m0 = E.margin_mask([z0.reshape(2, 2, 3)], mu)
    assert m0.shape == (2, 2) and m0.reshape(-1).tolist() == [False, True, False, True]
    # a bound below the smallest entry flags nothing; a negative value counts by its magnitude
    assert not E.margin_mask([z0], 1e-12).any()
    assert E.margin_mask([torch.tensor([[-1e-9, 5.0]], dtype=torch.float64)], mu).tolist() == [True]
