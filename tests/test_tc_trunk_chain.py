"""The fused trunk forward of the tensor-core engines (trunk_chain_kernel, width 256): every fp32 activation it writes and
the last layer's row image must be the bytes the layer-by-layer GEMMs write (sparf_tc_selftest_chain runs either on the
same inputs), and the public calls it serves must not depend on which activations they keep."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

W = 256
NETS = {"default": (8, 4, 63), "short": (5, 2, 27)}      # nt, skip, E3 (63 -> two encoding k-steps, 27 -> one)
PRECS = {"f16x3": (3, 1), "f16x1": (1, 1), "bf16x3": (3, 0)}


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _net(name, M, seed):
    nt, skip, E3 = NETS[name]
    E3p = -(-E3 // 32) * 32
    g = torch.Generator(device="cpu").manual_seed(seed)
    enc = torch.zeros(M, E3p)
    enc[:, :E3] = torch.randn(M, E3, generator=g)
    ws = []
    for l in range(nt):
        k = (E3 if l == 0 else W) + (E3 if l == skip else 0)
        ws.append((torch.randn(W, k, generator=g) * (2.0 / k) ** 0.5).reshape(-1))
    bias = torch.randn(nt, W, generator=g) * 0.1
    return nt, skip, E3, enc.cuda(), torch.cat(ws).cuda(), bias.cuda()


def _run(net, M, prec, chain, max_ctas=0, outputs=None, rows=None):
    """H [nt, M, 256] (NaN where nothing was written) and the last row image (0xFFFF likewise), as int32 / int16 bytes"""
    from sparf_b200 import _lib
    nt, skip, E3, enc, w, bias = net
    passes, f16 = PRECS[prec]
    H = torch.full((nt, M, W), float("nan"), device="cuda")
    last = torch.full((-(-M // 128) * 8 * 8192,), -1, dtype=torch.int16, device="cuda")
    cnt = torch.tensor([rows], dtype=torch.int64, device="cuda") if rows is not None else None
    outputs = (1 << nt) - 1 if outputs is None else outputs
    _lib.check(_lib.lib().sparf_tc_selftest_chain(_p(enc), M, E3, nt, skip, _p(w), _p(bias), passes, f16, max_ctas, chain,
                                                  outputs, _p(cnt), _p(H), _p(last),
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_chain")
    torch.cuda.synchronize()
    return H.view(torch.int32), last


def _same(a, b):
    assert torch.equal(a[0], b[0]), "fp32 activations differ in %d words" % (a[0] != b[0]).sum().item()
    assert torch.equal(a[1], b[1]), "last row image differs in %d elements" % (a[1] != b[1]).sum().item()


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(NETS))
@pytest.mark.parametrize("M", [1, 63, 64, 65, 129, 131072])
def test_chain_equals_layer_by_layer(M, name, prec):
    """Partial and odd 64-row tiles: rows past M are not written in fp32 and are zero in the image, whose 128-row tiles
    are written whole."""
    net = _net(name, M, 7 * M + len(name))
    ref = _run(net, M, prec, 0)
    assert not torch.isnan(ref[0].view(torch.float32)).any() and (ref[0] != 0).any()
    _same(_run(net, M, prec, 1), ref)


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("name", list(NETS))
def test_chain_few_ctas(name, max_ctas):
    """One CTA walks several tiles: the weight ring (4 stages) wraps across layers and tiles, the encoding buffer is
    refilled per tile."""
    net = _net(name, 1000, 11 + max_ctas)
    _same(_run(net, 1000, "f16x3", 1, max_ctas=max_ctas), _run(net, 1000, "f16x3", 0))


@pytest.mark.parametrize("name", list(NETS))
def test_chain_optional_outputs(name):
    """Activations that are not asked for stay on the SM: what is written is what the all-outputs run writes."""
    M = 333
    net = _net(name, M, 5)
    nt = net[0]
    Hall, last_all = _run(net, M, "f16x3", 1)
    H2, last2 = _run(net, M, "f16x3", 1, outputs=3 << (nt - 2))
    assert torch.equal(H2[nt - 2:], Hall[nt - 2:]) and torch.equal(last2, last_all)
    assert torch.isnan(H2[:nt - 2].view(torch.float32)).all()
    H1, last1 = _run(net, M, "f16x3", 1, outputs=1 << (nt - 2))      # the chain ends below the last layer
    assert torch.equal(H1[nt - 2], Hall[nt - 2])
    assert torch.isnan(H1[nt - 1].view(torch.float32)).all() and (last1 == -1).all()
    _same((H1, last1), _run(net, M, "f16x3", 0, outputs=1 << (nt - 2)))


@pytest.mark.parametrize("K", [0, 1, 63, 64, 65, 300])
def test_chain_device_row_count(K):
    """M = 300 is a capacity and K, read on the device, the rows computed: as the layer-by-layer GEMMs with the same
    count, and the live rows as a call of K rows."""
    cap = 300
    net = _net("default", cap, 3)
    got = _run(net, cap, "f16x3", 1, rows=K)
    _same(got, _run(net, cap, "f16x3", 0, rows=K))
    assert torch.isnan(got[0][:, K:].view(torch.float32)).all()
    if K:
        small = (net[0], net[1], net[2], net[3][:K].contiguous(), net[4], net[5])
        ref = _run(small, K, "f16x3", 1)
        n = ref[1].numel()
        assert torch.equal(got[0][:, :K], ref[0]) and torch.equal(got[1][:n], ref[1])


def _trunk(seed, nt=8, skip=4, L=10):
    g = torch.Generator(device="cpu").manual_seed(seed)
    E3 = 3 + 6 * L
    ps = []
    for l in range(nt):
        k = (E3 if l == 0 else W) + (E3 if l == skip else 0)
        ps += [torch.randn(W + (l == nt - 1), k, generator=g) * (2.0 / k) ** 0.5, torch.randn(W + (l == nt - 1), generator=g) * 0.1]
    return [p.cuda() for p in ps], g


@pytest.mark.parametrize("engine", ["tc_3x", "tc_1x"])
def test_density_forward_through_the_chain(engine):
    """The density calls at the default width: raw does not depend on whether the features are computed (the chain ends
    one layer earlier without them) or on which other points share a tile, and agrees with the fp32 engine."""
    from sparf_b200 import _lib, ops
    spec = ops.MLPSpec()
    params, g = _trunk(1)
    pts = (torch.rand(70001, 3, generator=g) * 2 - 1).cuda()
    eng = _lib.ENGINES[engine]
    with torch.no_grad():
        raw, feat = ops.density_forward(spec, pts, params, engine=eng)
        raw_nf, none = ops.density_forward(spec, pts, params, engine=eng, features=False)
        raw_part, feat_part = ops.density_forward(spec, pts[100:1101], params, engine=eng)
        raw32, feat32 = ops.density_forward(spec, pts, params, engine=_lib.ENGINES["simt_fp32"])
    assert none is None and torch.equal(raw, raw_nf)
    assert torch.equal(raw[100:1101], raw_part) and torch.equal(feat[100:1101], feat_part)
    tol = 1e-4 if engine == "tc_3x" else 5e-2
    assert (raw - raw32).abs().max().item() < tol * (1 + raw32.abs().max().item())
    assert (feat - feat32).abs().max().item() < tol * (1 + feat32.abs().max().item())


@pytest.mark.parametrize("engine", ["tc_3x", "tc_1x"])
@pytest.mark.parametrize("S", [128, 96])
def test_mlp_forward_through_the_chain(S, engine):
    """R = 1023 rays: the plain forward (the chain keeps the last two activations only) and the taped forward (all of
    them) give the same sigma and rgb, which agree with the fp32 engine."""
    from sparf_b200 import _lib, ops
    spec = ops.MLPSpec()
    params, g = _trunk(2)
    hw, ev = spec.head_width, 3 + 6 * spec.L_view
    params += [p.cuda() for p in (torch.randn(hw, W + ev, generator=g) * (2.0 / (W + ev)) ** 0.5, torch.randn(hw, generator=g) * 0.1,
                                  torch.randn(3, hw, generator=g) * (2.0 / hw) ** 0.5, torch.randn(3, generator=g) * 0.1)]
    R = 1023
    o = (torch.randn(R, 3, generator=g) * 0.3).cuda()
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda()
    t = torch.sort(torch.rand(R, S, generator=g) * 4 + 1.2, dim=1).values.cuda()
    eng = _lib.ENGINES[engine]
    with torch.no_grad():
        sigma, rgb = ops.mlp_forward(spec, o, d, t, params, engine=eng)
        sigma32, rgb32 = ops.mlp_forward(spec, o, d, t, params, engine=_lib.ENGINES["simt_fp32"])
    taped = [p.clone().requires_grad_(True) for p in params]
    sigma_t, rgb_t = ops.mlp_forward(spec, o, d, t, taped, engine=eng)
    assert torch.equal(sigma, sigma_t.detach()) and torch.equal(rgb, rgb_t.detach())
    tol = 1e-4 if engine == "tc_3x" else 5e-2
    assert (sigma - sigma32).abs().max().item() < tol * (1 + sigma32.abs().max().item())
    assert (rgb - rgb32).abs().max().item() < tol
