"""The fused input gradients of the trunk backward (dgrad_chain_kernel, width 256): the transposed images of G[nt-3] ...
G[0] and the row images of G[skip] and G[0] it writes must be the bytes the layer-by-layer input-gradient GEMMs write
with the same bit masks (sparf_tc_selftest_dgrad_chain runs either on the same inputs), and its column sums the same
sums up to the order of the float additions.  The fused forward's ReLU masks (sparf_tc_selftest_chain_bits) must be
H > 0 of its own fp32 activations."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

W = 256
NETS = {"default": (8, 4, 63), "short": (5, 2, 27)}      # nt, skip, E3
PRECS = {"bf16x3": (3, 3), "bf16x1": (1, 1), "bf16x3_w1": (3, 1)}     # input-gradient passes, weight-gradient passes


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _weights(nt, skip, E3, g, ints):
    ws = []
    for l in range(nt):
        k = (E3 if l == 0 else W) + (E3 if l == skip else 0)
        if ints and 1 <= l <= nt - 2:
            # a signed permutation over the first 256 columns: every gradient stays a small integer, so the products and
            # the column sums are exact in any order
            w = torch.zeros(W, k)
            w[torch.randperm(W, generator=g), torch.arange(W)] = torch.randint(0, 2, (W,), generator=g).float() * 2 - 1
        else:
            w = torch.randn(W, k, generator=g) * (2.0 / k) ** 0.5
        ws.append(w.reshape(-1))
    return torch.cat(ws)


def _inputs(name, M, seed, ints=False):
    nt, skip, E3 = NETS[name]
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randint(-3, 4, (M, W), generator=g).float() if ints else torch.randn(M, W, generator=g)
    bits = torch.randint(-2 ** 31, 2 ** 31, (nt - 2, M, 8), generator=g, dtype=torch.int64).to(torch.int32)
    return nt, skip, E3, G.cuda(), _weights(nt, skip, E3, g, ints).cuda(), bits.cuda()


def _run(inp, M, prec, chain, max_ctas=0, rows=None, row=True):
    """(transposed images, row images, column sums); images start as 0xFFFF, so bytes not written show"""
    from sparf_b200 import _lib
    nt, skip, E3, G, w, bits = inp
    dp, tp = PRECS[prec]
    ntr = 2 * -(-M // 32) * 8192
    nrow = -(-M // 128) * 8 * 8192
    tr = torch.full(((nt - 2) * ntr,), -1, dtype=torch.int16, device="cuda")
    rimg = torch.full((2 * nrow,), -1, dtype=torch.int16, device="cuda") if row else None
    db = torch.full((nt - 2, W), float("nan"), device="cuda")
    cnt = torch.tensor([rows], dtype=torch.int64, device="cuda") if rows is not None else None
    _lib.check(_lib.lib().sparf_tc_selftest_dgrad_chain(_p(G), M, E3, nt, skip, _p(w), _p(bits), dp, tp, max_ctas, chain,
                                                        _p(cnt), _p(tr), _p(rimg), _p(db), _stream()),
               "tc_selftest_dgrad_chain")
    torch.cuda.synchronize()
    return tr, rimg, db


def _same(a, b, exact_sums=False):
    assert torch.equal(a[0], b[0]), "transposed images differ in %d elements" % (a[0] != b[0]).sum().item()
    if a[1] is not None:
        assert torch.equal(a[1], b[1]), "row images differ in %d elements" % (a[1] != b[1]).sum().item()
    assert not torch.isnan(a[2]).any() and not torch.isnan(b[2]).any()
    if exact_sums:
        assert torch.equal(a[2], b[2])
    else:     # 64-row tiles against 128-row tiles: the same sums, added in another order
        scale = b[2].abs().amax(dim=1, keepdim=True) + 1e-30
        assert ((a[2] - b[2]).abs() / scale).max().item() < 1e-5


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(NETS))
@pytest.mark.parametrize("M", [1, 63, 64, 65, 129, 131072])
def test_dgrad_chain_equals_layer_by_layer(M, name, prec):
    """Partial and odd 64-row tiles: rows past M are zero in every image, and the row images' 128-row tiles are written
    whole."""
    inp = _inputs(name, M, 3 * M + len(name) + len(prec))
    ref = _run(inp, M, prec, 0)
    assert (ref[0] != -1).any() and (ref[1] != -1).any()
    _same(_run(inp, M, prec, 1), ref)


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("name", list(NETS))
def test_dgrad_chain_few_ctas(name, max_ctas):
    """One CTA walks several tiles: the weight ring wraps across layers and tiles, the input buffer is refilled per
    tile; and without row images asked for."""
    inp = _inputs(name, 1000, 17 + max_ctas)
    _same(_run(inp, 1000, "bf16x3", 1, max_ctas=max_ctas), _run(inp, 1000, "bf16x3", 0))
    _same(_run(inp, 1000, "bf16x3_w1", 1, max_ctas=max_ctas, row=False), _run(inp, 1000, "bf16x3_w1", 0, row=False))


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(NETS))
def test_dgrad_chain_column_sums_exact(name, prec):
    """Small-integer gradients through signed permutations: every product and sum is exact, so the column sums are equal
    whatever the order of their additions."""
    inp = _inputs(name, 5000, 29, ints=True)
    got, ref = _run(inp, 5000, prec, 1), _run(inp, 5000, prec, 0)
    _same(got, ref, exact_sums=True)
    assert ref[2].abs().max().item() > 0


@pytest.mark.parametrize("K", [0, 1, 63, 64, 65, 300])
def test_dgrad_chain_device_row_count(K):
    """M = 300 is a capacity and K, read on the device, the rows computed: the same bytes as the layer-by-layer GEMMs
    with the same count (nothing at all for K = 0)."""
    cap = 300
    inp = _inputs("default", cap, 5)
    got = _run(inp, cap, "bf16x3", 1, rows=K)
    ref = _run(inp, cap, "bf16x3", 0, rows=K)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    if K == 0:
        assert (got[0] == -1).all() and (got[1] == -1).all() and (got[2] == 0).all()
    else:
        scale = ref[2].abs().amax(dim=1, keepdim=True) + 1e-30
        assert ((got[2] - ref[2]).abs() / scale).max().item() < 1e-5


def _fwd_net(name, M, seed):
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


def _pack_bits(H):
    """(H > 0) as the kernels' words: bit n & 31 of word [m][n >> 5], as int32"""
    b = (H > 0).reshape(*H.shape[:-1], W // 32, 32).long() << torch.arange(32, device=H.device)
    w = b.sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


@pytest.mark.parametrize("rows", [None, 0, 65, 300])
@pytest.mark.parametrize("name", list(NETS))
@pytest.mark.parametrize("M", [1, 65, 333])
def test_forward_chain_bits(M, name, rows):
    """The fused forward's masks of H[0] ... H[nt-3] are (H > 0) of the fp32 H of the same call, at ragged M and with a
    device row count (rows past it are not written); asking for them leaves H as it is."""
    from sparf_b200 import _lib
    if rows is not None and rows > M:
        pytest.skip("row count above the capacity")
    nt, skip, E3, enc, w, bias = net = _fwd_net(name, M, 7 * M + len(name))
    cnt = torch.tensor([rows], dtype=torch.int64, device="cuda") if rows is not None else None
    H = torch.full((nt, M, W), float("nan"), device="cuda")
    bits = torch.full((nt - 2, M, W // 32), -1, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().sparf_tc_selftest_chain_bits(_p(enc), M, E3, nt, skip, _p(w), _p(bias), 3, 1, 0, _p(cnt), _p(H),
                                                       _p(bits), _stream()), "tc_selftest_chain_bits")
    H0 = torch.full((nt, M, W), float("nan"), device="cuda")
    last = torch.full((-(-M // 128) * 8 * 8192,), -1, dtype=torch.int16, device="cuda")
    _lib.check(_lib.lib().sparf_tc_selftest_chain(_p(enc), M, E3, nt, skip, _p(w), _p(bias), 3, 1, 0, 1, (1 << nt) - 1, _p(cnt),
                                                  _p(H0), _p(last), _stream()), "tc_selftest_chain")
    torch.cuda.synchronize()
    assert torch.equal(H.view(torch.int32), H0.view(torch.int32))
    K = M if rows is None else rows
    assert torch.equal(bits[:, :K], _pack_bits(H[:nt - 2, :K]))
    assert (bits[:, K:] == -1).all()
    if K:
        assert (bits[:, :K] != 0).any() and (bits[:, :K] != -1).any()
