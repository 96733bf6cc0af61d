"""Density queries at arbitrary points (sparf_density_forward / sparf_density_backward, ops.density_forward,
NeRF.compute_raw_density) on the SIMT and tensor-core engines, against the fp64 oracle, the reference's own outputs
(tests/golden/density_raw.npz) and NeRF.forward."""
import ctypes

import pytest
import torch

import make_density_golden as G

pytestmark = pytest.mark.gpu

C2F = (0.1, 0.5)
TRUNK_KEYS = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], [])


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _engine(name):
    from sparf_b200 import _lib
    e = _lib.ENGINES[name]
    if not _lib.lib().sparf_engine_available(e):
        pytest.skip("%s not available on this device" % name)
    return e


def _err(x, ref):
    """max |x - ref| / max |ref|"""
    ref = ref.double()
    return ((x.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _problem(M, seed):
    """default network with common.det_weights, BARF mask at progress 0.3, M points uniform in [-1.5, 1.5]^3"""
    import common
    from sparf_b200 import ops
    opt = common.make_opt(barf_c2f=C2F)
    sd = common.det_weights(opt, seed, progress=0.3)
    params = [sd[k].cuda() for k in TRUNK_KEYS]
    g = torch.Generator(device="cpu").manual_seed(seed)
    pts = (torch.rand(M, 3, generator=g) * 3 - 1.5).cuda()
    return ops.MLPSpec(barf_c2f=C2F), params, sd["progress"].cuda(), pts


def _oracle(params, prog, pts, dtype):
    from density_oracle import raw_density
    p = {k: v.to(dtype) for k, v in zip(TRUNK_KEYS, params)}
    p["progress"] = prog
    return raw_density(p, pts.to(dtype), barf_c2f=C2F)


# M = 65 536 + 333 spans two forward chunks
@pytest.mark.parametrize("M", [1, 333, 65536 + 333])
def test_density_forward_matches_oracle(M):
    from sparf_b200 import ops
    spec, params, prog, pts = _problem(M, seed=M % 1000 + 3)
    with torch.no_grad():
        raw64, feat64 = _oracle(params, prog, pts, torch.float64)
        raw32, feat32 = _oracle(params, prog, pts, torch.float32)
        out = {}
        for name in ("simt_fp32", "tc_3x"):
            eng = _engine(name)
            raw, feat = ops.density_forward(spec, pts, params, progress=prog, engine=eng)
            raw_only, none = ops.density_forward(spec, pts, params, progress=prog, engine=eng, features=False)
            torch.cuda.synchronize()
            assert none is None and raw.shape == (M,) and feat.shape == (M, 256)
            assert torch.equal(raw_only, raw), "features=False changed raw"
            for what, x, x64, x32 in (("raw", raw, raw64, raw32), ("feat", feat, feat64, feat32)):
                e, e32 = _err(x, x64), _err(x32, x64)
                print("M=%d %-9s %-4s err vs fp64 %.2e (fp32 oracle %.2e)" % (M, name, what, e, e32))
                assert e <= max(2e-5, 2 * e32), (name, what, e, e32)
            out[name] = (raw, feat)
        if "tc_3x" in out:
            for i, what in enumerate(("raw", "feat")):
                assert _err(out["tc_3x"][i], out["simt_fp32"][i]) <= 3e-5, what


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
@pytest.mark.parametrize("case", list(G.CASES))
def test_density_matches_reference_golden(engine, case):
    """NeRF.compute_raw_density against the reference's own compute_raw_density on the golden's [2,37,5,3] points:
    outputs, and the gradients of the golden's probe w.r.t. the points and every trunk tensor."""
    import numpy as np
    from helpers import GOLDEN_DIR, check_grads
    from sparf_b200 import ops
    from sparf_b200.frequency_nerf import NeRF
    eng = _engine(engine)
    opt, sd, pts, a, b = G.case_inputs(case)
    with np.load(GOLDEN_DIR + "/density_raw.npz") as z:
        gold = {k[len(case) + 1:]: z[k] for k in z.files if k.startswith(case + "/")}
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=False)
    pts = pts.cuda().requires_grad_(True)
    old = ops.get_engine()
    ops.set_engine(eng)
    try:
        raw, feat = nerf.compute_raw_density(opt, pts, None)
        G.probe(raw, feat, a.cuda(), b.cuda()).backward()
        torch.cuda.synchronize()
    finally:
        ops.set_engine(old)
    assert raw.shape == G.SHAPE and feat.shape == G.SHAPE + (256,)
    p64 = {k: v.double() for k, v in sd.items()}
    raw64, feat64 = _oracle([p64[k] for k in TRUNK_KEYS], p64["progress"], pts.detach().cpu(), torch.float64)
    for what, x, ref, x64 in (("raw", raw, gold["raw"], raw64), ("feat", feat, gold["feat"], feat64)):
        ref = torch.from_numpy(ref)
        e, e_ref = _err(x.detach().cpu(), ref), _err(ref, x64)
        print("%s %s %-4s err vs reference %.2e (reference vs fp64 %.2e)" % (case, engine, what, e, e_ref))
        assert e <= max(2e-5, 2 * e_ref), (what, e, e_ref)
    grads = {"grad_points": pts.grad}
    grads.update({"grad_" + k: p.grad for k, p in nerf.named_parameters() if k.startswith("mlp_feat.")})
    assert all(p.grad is None for p in nerf.mlp_rgb.parameters())
    check_grads(grads, gold, tol=2e-3)


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_softplus_of_raw_matches_nerf_forward(engine):
    """x = o + 0*d is x = p: NeRF.forward's density at the same points is the softplus of compute_raw_density's raw."""
    import common
    from sparf_b200 import ops
    from sparf_b200.frequency_nerf import NeRF
    eng = _engine(engine)
    opt = common.make_opt(barf_c2f=C2F)
    nerf = NeRF(opt).cuda()
    nerf.load_state_dict({k: v.cuda() for k, v in common.det_weights(opt, 9, progress=0.3).items()})
    g = torch.Generator(device="cpu").manual_seed(9)
    pts = (torch.rand(2, 300, 7, 3, generator=g) * 3 - 1.5).cuda()
    ray = torch.randn(2, 300, 3, generator=g).cuda()
    old = ops.get_engine()
    ops.set_engine(eng)
    try:
        with torch.no_grad():
            raw, feat = nerf.compute_raw_density(opt, pts, None)
            dens = nerf.forward(opt, pts, ray, None, None)["density_samples"]
    finally:
        ops.set_engine(old)
    assert raw.shape == (2, 300, 7) and feat.shape == (2, 300, 7, 256)
    sp = torch.nn.functional.softplus(raw)
    assert ((sp - dens).abs() / dens.abs().clamp_min(1e-30)).max().item() <= 1e-6


def _trunk_grads(spec, params, prog, pts, eng, a, b):
    """gradients of sum(a * raw) + sum(b * feat) (a or b None: that output not differentiated) w.r.t. the points and the
    trunk tensors, through ops.density_forward"""
    from sparf_b200 import ops
    ps = [p.clone().requires_grad_(True) for p in params]
    x = pts.clone().requires_grad_(True)
    raw, feat = ops.density_forward(spec, x, ps, progress=prog, engine=eng)
    loss = (raw * a).sum() if a is not None else 0
    if b is not None:
        loss = loss + (feat * b).sum()
    loss.backward()
    torch.cuda.synchronize()
    return [x.grad] + [p.grad for p in ps]


def _point_errors(x, ref):
    """per point: max over its coordinates of |x - ref|, over max |ref|"""
    ref = ref.double()
    return (x.double() - ref).abs().amax(-1) / ref.abs().max().clamp_min(1e-30)


# M = 2 x 32 768 + 5 spans three backward chunks
@pytest.mark.parametrize("probe", ["raw_and_feat", "raw_only", "feat_only"])
@pytest.mark.parametrize("M", [333, 2 * 32768 + 5])
def test_density_backward_matches_fp64(M, probe):
    """Every trunk gradient and the points' gradient of tc_3x and tc_3x_w1 against fp64 autograd, within the bound
    test_tc_narrow.py puts on the tensor-core engines: 2e-3 or 4 x the fp32 SIMT engine's own error.  raw_only is the
    normals case (d_feat = NULL); feat_only passes d_raw = NULL.

    A point with a pre-activation within rounding of 0 can take the other side of a ReLU in fp32-level arithmetic than
    in fp64.  Its own gradient is then off by O(1e-2) of the largest, and every gradient below that layer by as much
    (the random probe's sums cancel to about 1/sqrt(M) of their terms): one such point at 333 points puts layers 0-4 of
    tc_3x 2e-2 away from fp64, and a few at 65 541 points put the SIMT engine's own errors at 5e-3.  Such points (a
    point-gradient error above 1e-4 on any engine, ten times the others') are taken out of the probe (a and b zero
    there), at most 1 % of them, and the gradients are compared on the others.  tc_3x_w1 computes the weight gradients
    in one bf16 pass by design (8-bit factors, test_tc_engine.test_tc_3x_w1_reduced_weight_gradient_engine): its weight
    tensors get 1e-2."""
    from sparf_b200 import _lib
    spec, params, prog, pts = _problem(M, seed=M % 1000 + 11)
    g = torch.Generator(device="cuda").manual_seed(M)
    a = torch.randn(M, device="cuda", generator=g) if probe != "feat_only" else None
    b = torch.randn(M, 256, device="cuda", generator=g) * 0.1 if probe != "raw_only" else None
    names = ["points"] + TRUNK_KEYS
    engines = [n for n in ("simt_fp32", "tc_3x", "tc_3x_w1") if _lib.lib().sparf_engine_available(_lib.ENGINES[n])]

    def run(a, b):
        p64 = [p.double().requires_grad_(True) for p in params]
        x64 = pts.double().requires_grad_(True)
        raw, feat = _oracle(p64, prog.double(), x64, torch.float64)
        loss = (raw * a.double()).sum() if a is not None else 0
        if b is not None:
            loss = loss + (feat * b.double()).sum()
        loss.backward()
        return [x64.grad] + [p.grad for p in p64], {n: _trunk_grads(spec, params, prog, pts, _lib.ENGINES[n], a, b)
                                                     for n in engines}

    truth, got = run(a, b)
    flipped = torch.stack([_point_errors(got[n][0], truth[0]) for n in engines]).amax(0) > 1e-4
    nf = int(flipped.sum())
    print("M=%d %s: %d point(s) with a point-gradient error above 1e-4 taken out of the probe" % (M, probe, nf))
    assert nf <= max(1, M // 100), nf
    if nf:
        keep = (~flipped).float()
        a = a * keep if a is not None else None
        b = b * keep[:, None] if b is not None else None
        truth, got = run(a, b)
    e_simt = [_err(x, t) for x, t in zip(got["simt_fp32"], truth)]
    bad = []
    for name in engines[1:]:
        for k, x, t, es in zip(names, got[name], truth, e_simt):
            e = _err(x, t)
            ok = e < max(2e-3, 4 * es, 1e-2 if name == "tc_3x_w1" and k.endswith(".weight") else 0)
            print("M=%d %s %-9s %-18s err vs fp64 %.2e (simt %.2e)%s" % (M, probe, name, k, e, es, "" if ok else "  FAIL"))
            if not ok:
                bad.append((name, k, e, es))
    assert not bad, bad


@pytest.mark.parametrize("M,W,row_passes,tr_passes", [(1, 256, 3, 3), (200, 256, 3, 3), (333, 256, 3, 1),
                                                      (1000, 256, 1, 1), (77, 200, 3, 3), (4100, 72, 3, 1)])
def test_tc_feat_backward_images_bit_identical(M, W, row_passes, tr_passes):
    """The density backward's last-layer kernel writes, byte for byte, the images that masking d_feat in fp32 and packing
    it gives, with the zero padding past M and W (the buffers start as 0xFFFF); its sums of d_raw and of G's columns
    equal colsum_kernel's.  The gradients are multiples of 2^-8 below 4 in magnitude: they sum exactly in any order, and
    their bf16 splits have lo halves.  M = 1, 200, 333, 77 leave ragged row tiles and k-steps; W = 200 and 72 ragged
    column blocks."""
    from sparf_b200 import _lib
    L = _lib.lib()
    if not L.sparf_engine_available(_lib.ENGINE_TC_3X):
        pytest.skip("tensor-core engine not available")
    g = torch.Generator(device="cpu").manual_seed(M + W)
    d_raw = (torch.randint(-1024, 1024, (M,), generator=g) / 256.0).cuda()
    d_feat = (torch.randint(-1024, 1024, (M, W), generator=g) / 256.0).cuda()
    feat = torch.randn(M, W, generator=g).cuda()                # about half masked
    cd = lambda x, y: -(-x // y)
    nrow = cd(M, 128) * cd(W, 32) * 8192
    ntr = cd(W, 128) * cd(M, 32) * 8192
    img = torch.zeros(2 * (nrow + ntr), dtype=torch.int16, device="cuda")
    sums = torch.full((2, W + 1), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_featgrad(_p(d_raw), _p(d_feat), _p(feat), M, W, row_passes, tr_passes, _p(img), _p(sums),
                                            _stream()), "tc_selftest_featgrad")
    torch.cuda.synchronize()
    fused, ref = img[:nrow + ntr], img[nrow + ntr:]
    assert torch.equal(fused[:nrow], ref[:nrow]), "row image: %d elements differ" % (fused[:nrow] != ref[:nrow]).sum().item()
    assert torch.equal(fused[nrow:], ref[nrow:]), "transposed image: %d elements differ" % (fused[nrow:] != ref[nrow:]).sum().item()
    assert not (ref[:nrow] == -1).all() and not (ref[nrow:] == -1).all()
    assert torch.equal(sums[0], sums[1])
    G_ = torch.where(feat > 0, d_feat, torch.zeros_like(d_feat))
    assert torch.equal(sums[1, 1:], G_.double().sum(0).float()) and sums[1, 0].item() == d_raw.double().sum().item()


def _abi(spec, params, prog, M):
    from sparf_b200 import _lib
    m, keep = spec.fill(params, prog)
    grads = [torch.zeros_like(p) for p in params]
    return _lib.lib(), m, keep, grads, spec.grad_struct(grads)


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_density_abi_accumulates_accepts_null_head_and_empty(engine):
    """Two backward calls double the gradients (up to the fp32 atomic-order noise of the sums); the head pointers are NULL
    throughout;
    M = 0 launches nothing."""
    from sparf_b200 import _lib
    eng = _engine(engine)
    M = 40000
    spec, params, prog, pts = _problem(M, seed=4)
    L, m, keep, grads, gs = _abi(spec, params, prog, M)
    assert not any(m.head_w) and not any(m.head_b) and not any(gs.head_w) and not any(gs.head_b)
    d_raw = torch.randn(M, device="cuda")
    d_feat = torch.randn(M, 256, device="cuda") * 0.1
    d_pts = torch.zeros(M, 3, device="cuda")
    ws = torch.empty(L.sparf_density_workspace_bytes(ctypes.byref(m), M, 1, eng), dtype=torch.uint8, device="cuda")
    once = None
    for _ in range(2):
        _lib.check(L.sparf_density_backward(ctypes.byref(m), eng, M, _p(pts), _p(d_raw), _p(d_feat), ctypes.byref(gs), _p(d_pts),
                                            _p(ws), ws.numel(), _stream()), "density_backward")
        torch.cuda.synchronize()
        if once is None:
            once = [g.clone() for g in grads] + [d_pts.clone()]
    for x, x1 in zip(grads + [d_pts], once):      # relative L2: the atomic-order noise of a sum over 40 000 rows
        assert ((x - 2 * x1).norm() / (2 * x1).norm().clamp_min(1e-30)).item() <= 1e-6
    n0 = L.sparf_launch_count()
    _lib.check(L.sparf_density_forward(ctypes.byref(m), eng, 0, _p(None), _p(None), _p(None), _p(None), 0, _stream()), "fwd M=0")
    _lib.check(L.sparf_density_backward(ctypes.byref(m), eng, 0, _p(None), _p(None), _p(None), ctypes.byref(gs), _p(None),
                                        _p(None), 0, _stream()), "bwd M=0")
    assert L.sparf_launch_count() == n0
    assert L.sparf_density_workspace_bytes(ctypes.byref(m), 0, 0, eng) == 0


@pytest.mark.parametrize("engine", ["simt_fp32", "tc_3x"])
def test_density_no_sync_and_cuda_graph_replay(engine):
    """A forward + backward (normals: the gradient of raw w.r.t. the points) synchronises nothing, and replays correctly
    from a CUDA graph on new points."""
    from sparf_b200 import ops
    eng = _engine(engine)
    M = 5000
    spec, params, prog, pts = _problem(M, seed=6)
    b = torch.randn(M, 256, device="cuda") * 0.01

    def step(x):
        raw, feat = ops.density_forward(spec, x, params, progress=prog, engine=eng)
        (d,) = torch.autograd.grad(raw.sum() + (feat * b).sum(), x)
        return raw, feat, d

    x = pts.clone().requires_grad_(True)
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(x)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(x)
    new = torch.rand(M, 3, device="cuda") * 3 - 1.5
    with torch.no_grad():
        x.copy_(new)
    graph.replay()
    torch.cuda.synchronize()
    ref = step(new.clone().requires_grad_(True))
    torch.cuda.synchronize()
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
    assert ((out[2] - ref[2]).abs().max() / ref[2].abs().max()).item() <= 1e-6
