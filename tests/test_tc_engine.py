"""Tensor-core engines: exact-integer self-tests of the wgmma GEMM kernels, then the engines against the SIMT fp32
engine (same C ABI, same inputs, on the device) and the fp64 oracle."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("K", [64, 128, 256])
def test_tcgen05_selftest_gemm_exact(K):
    """Small-integer operands are exact in bf16 and their dot products exact in fp32: a bit-exact result
    proves the shared-memory operand layout, the wgmma descriptors, K stepping and the accumulator fragment mapping."""
    from sparf_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cpu").manual_seed(K)
    A = torch.randint(-4, 5, (128, K), generator=g).float().cuda()
    B = torch.randint(-4, 5, (128, K), generator=g).float().cuda()
    packed = torch.zeros(128 * K * 2, dtype=torch.uint8, device="cuda")
    D = torch.full((128, 128), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest(_p(A), _p(B), K, _p(packed), _p(D), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest")
    torch.cuda.synchronize()
    ref = A @ B.t()
    assert torch.equal(D, ref), (D - ref).abs().max().item()


def _rand_problem(R, S, seed=0, c2f=None, peaky=True):
    import common
    from sparf_b200 import ops
    opt = common.make_opt(S=S, barf_c2f=c2f)
    sd = common.det_weights(opt, seed, peaky=peaky, sigma_bias=-3.0, progress=0.6 if c2f else None)
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
        ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]
    params = [sd[k].cuda() for k in keys]
    g = torch.Generator(device="cpu").manual_seed(seed)
    o = (torch.randn(R, 3, generator=g) * 0.5).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    d = d / d.norm(dim=-1, keepdim=True) * (1 + 0.2 * torch.rand(R, 1, generator=g).cuda())
    t = torch.sort(torch.rand(R, S, generator=g) * 4 + 1.2, dim=1).values.cuda()
    spec = ops.MLPSpec(barf_c2f=c2f)
    prog = sd["progress"].cuda()
    return spec, params, o, d, t, prog


@pytest.mark.parametrize("R,S,c2f", [(8, 128, None), (1023, 128, None), (333, 96, (0.4, 0.7)), (37, 384, None), (5, 1, None)])
def test_tc_forward_matches_simt(R, S, c2f):
    """Tensor-core forward (3-pass fp16 split) vs the fp32 SIMT engine on identical device inputs."""
    from sparf_b200 import _lib, ops
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_3X):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _rand_problem(R, S, seed=R, c2f=c2f)
    noise = torch.randn(R, S, device="cuda") * 0.5
    with torch.no_grad():
        s_ref, c_ref = ops.mlp_forward(spec, o, d, t, params, noise=noise, progress=prog, engine=_lib.ENGINE_SIMT_FP32)
        s_tc, c_tc = ops.mlp_forward(spec, o, d, t, params, noise=noise, progress=prog, engine=_lib.ENGINE_TC_3X)
    torch.cuda.synchronize()
    es = ((s_tc - s_ref).abs().max() / s_ref.abs().max()).item()
    ec = (c_tc - c_ref).abs().max().item()
    print("R=%d S=%d: sigma rel err %.2e, rgb abs err %.2e" % (R, S, es, ec))
    assert es < 3e-5 and ec < 3e-5
    if S < 2:
        return
    # composited outputs: the quantity the 1e-4 north-star bound is stated on
    a = ops.composite(s_tc, c_tc, t, d)
    b = ops.composite(s_ref, c_ref, t, d)
    for x, y in zip(a[:3], b[:3]):
        assert ((x - y).abs().max() / y.abs().max()).item() < 3e-5


def test_tc_single_pass_is_a_fast_mode_outside_the_bound():
    """TC_1X (one bf16 pass) runs and is close, but is NOT the parity engine (error ~1e-3)."""
    from sparf_b200 import _lib, ops
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_1X):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _rand_problem(256, 128, seed=3)
    with torch.no_grad():
        s_ref, c_ref = ops.mlp_forward(spec, o, d, t, params, progress=prog, engine=_lib.ENGINE_SIMT_FP32)
        s_1, c_1 = ops.mlp_forward(spec, o, d, t, params, progress=prog, engine=_lib.ENGINE_TC_1X)
    e = (c_1 - c_ref).abs().max().item()
    print("single-pass bf16 rgb abs err %.2e" % e)
    assert e < 5e-2


@pytest.mark.parametrize("rows", [64, 128])
def test_tcgen05_selftest_tn_mn_major(rows):
    """D = G^T X through the weight-gradient kernel (contraction over rows, operands read transposed)."""
    from sparf_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cpu").manual_seed(rows)
    G = torch.randint(-4, 5, (rows, 128), generator=g).float().cuda()
    X = torch.randint(-4, 5, (rows, 128), generator=g).float().cuda()
    D = torch.full((128, 128), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_tn(_p(G), _p(X), rows, _p(D), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_tn")
    torch.cuda.synchronize()
    ref = G.t() @ X
    assert torch.equal(D, ref), (D - ref).abs().max().item()


# the last three batches exceed one backward chunk (32768 rows): gradients accumulate over the chunks
@pytest.mark.parametrize("R,S,c2f", [(8, 128, None), (1023, 128, None), (100, 96, (0.4, 0.7)), (37, 384, None),
                                     (1100, 128, None), (600, 256, (0.4, 0.7)), (1400, 96, None)])
def test_tc_backward_matches_simt(R, S, c2f):
    """Tensor-core backward (recomputed fp16 3-pass forward, bf16 3-pass input and weight gradients) vs the fp32 SIMT
    engine: every parameter gradient, same upstream gradients, same device inputs."""
    from sparf_b200 import _lib, ops
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_3X):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _rand_problem(R, S, seed=R + 1, c2f=c2f)
    noise = torch.randn(R, S, device="cuda") * 0.3
    g = torch.Generator(device="cuda").manual_seed(7)
    gs = torch.randn(R, S, device="cuda", generator=g) * 1e-3
    gc = torch.randn(R, S, 3, device="cuda", generator=g) * 1e-3
    grads = {}
    for eng, tape in ((_lib.ENGINE_SIMT_FP32, True), (_lib.ENGINE_TC_3X, True), (_lib.ENGINE_TC_3X, False)):
        ops.USE_TAPE[0] = tape     # with and without a tape request (engines without a tape recompute either way)
        ps = [p.clone().requires_grad_(True) for p in params]
        s, c = ops.mlp_forward(spec, o, d, t, ps, noise=noise, progress=prog, engine=eng)
        ((s * gs).sum() + (c * gc).sum()).backward()
        torch.cuda.synchronize()
        if eng == _lib.ENGINE_TC_3X and not tape:
            grads["tc_recompute"] = [p.grad.clone() for p in ps]
        else:
            grads[eng] = [p.grad.clone() for p in ps]
    ops.USE_TAPE[0] = True
    # ground truth: the oracle's formulas in fp64 on the device (autograd)
    from oracle import sparf_oracle as O
    keys = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
        ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]
    p64 = {k: p.double().clone().requires_grad_(True) for k, p in zip(keys, params)}
    p64["progress"] = prog.double()
    pts = o.double()[None, :, None] + d.double()[None, :, None] * t.double()[None, ..., None]
    dens, rgb = O.mlp_forward(p64, pts, d.double()[None], barf_c2f=c2f, noise=noise.double()[None])
    ((dens[0] * gs.double()).sum() + (rgb[0] * gc.double()).sum()).backward()
    truth = [p64[k].grad for k in keys]
    worst_tc = worst_simt = 0.0
    for i, (a, b, tr) in enumerate(zip(grads[_lib.ENGINE_TC_3X], grads[_lib.ENGINE_SIMT_FP32], truth)):
        den = tr.abs().max().clamp_min(1e-30)
        e_tc = ((a.double() - tr).abs().max() / den).item()
        e_simt = ((b.double() - tr).abs().max() / den).item()
        worst_tc, worst_simt = max(worst_tc, e_tc), max(worst_simt, e_simt)
        # within 2e-3 of the exact gradient, or as good as the fp32 engine up to a small factor (both engines
        # see ReLU sign flips of near-zero pre-activations on these ill-conditioned random nets)
        assert e_tc < max(2e-3, 4 * e_simt), (keys[i], e_tc, e_simt)
        e_rc = ((grads["tc_recompute"][i].double() - tr).abs().max() / den).item()
        assert e_rc < max(2e-3, 4 * e_simt), (keys[i], "recompute path", e_rc, e_simt)
    print("R=%d S=%d: worst grad rel err vs fp64: tensor cores %.2e, simt fp32 %.2e" % (R, S, worst_tc, worst_simt))


@pytest.mark.parametrize("R,S,c2f", [(64, 128, None), (341, 128, (0.4, 0.7)), (50, 96, (0.1, 0.9)), (1100, 128, (0.4, 0.7))])
def test_tc_ray_gradients_match_simt(R, S, c2f):
    """dL/d origins, dL/d dirs (camera-pose optimisation) from the tensor-core path (G4.W4e + G0.W0 on tensor cores,
    encoding backward, view-direction chain) vs the fp32 SIMT engine."""
    from sparf_b200 import _lib, ops
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_3X):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _rand_problem(R, S, seed=R + 5, c2f=c2f, peaky=False)
    g = torch.Generator(device="cuda").manual_seed(3)
    gs = torch.randn(R, S, device="cuda", generator=g) * 1e-2
    gc = torch.randn(R, S, 3, device="cuda", generator=g) * 1e-2
    res = {}
    for eng in (_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_3X):
        oo, dd = o.clone().requires_grad_(True), d.clone().requires_grad_(True)
        s, c = ops.mlp_forward(spec, oo, dd, t, params, progress=prog, engine=eng)
        ((s * gs).sum() + (c * gc).sum()).backward()
        torch.cuda.synchronize()
        res[eng] = (oo.grad.clone(), dd.grad.clone())
    for a, b, nm in zip(res[_lib.ENGINE_TC_3X], res[_lib.ENGINE_SIMT_FP32], ("d_origins", "d_dirs")):
        e = ((a - b).abs().max() / b.abs().max()).item()
        print("R=%d S=%d %s rel diff tc vs simt: %.2e" % (R, S, nm, e))
        assert e < 2e-2, (nm, e)   # both sit ~1e-2 from the exact gradient on random nets (2^9 pi amplification)


@pytest.mark.parametrize("R,S,c2f", [(1023, 128, None), (300, 96, (0.4, 0.7)), (1100, 128, None)])
def test_tc_3x_w1_reduced_weight_gradient_engine(R, S, c2f):
    """SPARF_ENGINE_TC_3X_W1 (non-default): same forward and same ray gradients as TC_3X, the wide layers' weight / bias
    gradients from ONE bf16 pass over the hi halves -- close to TC_3X, but outside the parity bound."""
    from sparf_b200 import _lib, ops
    if not _lib.lib().sparf_engine_available(_lib.ENGINE_TC_3X_W1):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _rand_problem(R, S, seed=R + 9, c2f=c2f)
    g = torch.Generator(device="cuda").manual_seed(11)
    gs = torch.randn(R, S, device="cuda", generator=g) * 1e-3
    gc = torch.randn(R, S, 3, device="cuda", generator=g) * 1e-3
    res = {}
    for eng in (_lib.ENGINE_TC_3X, _lib.ENGINE_TC_3X_W1):
        ps = [p.clone().requires_grad_(True) for p in params]
        oo, dd = o.clone().requires_grad_(True), d.clone().requires_grad_(True)
        s, c = ops.mlp_forward(spec, oo, dd, t, ps, progress=prog, engine=eng)
        ((s * gs).sum() + (c * gc).sum()).backward()
        torch.cuda.synchronize()
        res[eng] = (s.detach(), c.detach(), oo.grad.clone(), dd.grad.clone(), [p.grad.clone() for p in ps])
    a, b = res[_lib.ENGINE_TC_3X], res[_lib.ENGINE_TC_3X_W1]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])                      # same forward kernels
    for x, y in zip(a[2:4], b[2:4]):                                                # same input-gradient chain (float atomics)
        assert ((x - y).abs().max() / x.abs().max()).item() < 1e-5
    worst = 0.0
    for i, (x, y) in enumerate(zip(a[4], b[4])):
        e = ((x - y).abs().max() / x.abs().max().clamp_min(1e-30)).item()
        worst = max(worst, e)
        assert e < 3e-2, (i, e)
    assert worst > 1e-6, "the reduced engine produced the 3-pass result: the single-pass path did not run"
    print("R=%d S=%d: TC_3X_W1 weight gradients within %.1e (max-normalised) of TC_3X" % (R, S, worst))
