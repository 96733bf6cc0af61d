"""The weight-gradient GEMM's B operand (X, packed as its transposed bf16 image) and the ReLU mask bits written with it
for the input-gradient GEMM (sparf_tc_selftest_wgrad).

With a one-hot G (G[m][n] = 1 for one row m = sel[n] per output row n) every output row is one row of X through the
bf16 split: hi alone (1 pass) or hi + lo 2^-11 (3 passes), each exact in fp32, so the GEMM must match a NumPy model of
the split exactly.  The bits must equal (X > 0) packed on the host, NaN and -0 included."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _bf16(x):
    """round-to-nearest-even to bf16, kept in float32 (finite and infinite values)"""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def _split_value(x, passes):
    """what the GEMM makes of x times a one-hot 1, stored by a float atomic add, which flushes a subnormal result to
    zero"""
    hi = _bf16(x)
    v = hi
    if passes == 3:
        v = hi + _bf16((x - hi) * np.float32(2.0 ** 11)) * np.float32(2.0 ** -11)
    return np.where(np.abs(v) < np.float32(2.0 ** -126), np.float32(0), v).astype(np.float32)


def _mask_bits(X, M, K, div):
    keep = X[np.arange(M) // div, :K] > 0
    kw = -(-K // 32)
    keep = np.concatenate([keep, np.zeros((M, kw * 32 - K), bool)], 1)
    return np.packbits(keep.reshape(M, kw, 32), axis=2, bitorder="little").view("<u4").reshape(M, kw)


def _run(G, X, M, N, K, Kv, ldx, div, passes, max_ctas, bits):
    from sparf_b200 import _lib
    L = _lib.lib()
    dW = torch.full((N, K), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_wgrad(_p(G), _p(X), M, N, K, Kv, ldx, div, passes, max_ctas, _p(dW), _p(bits),
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_wgrad")
    torch.cuda.synchronize()
    return dW.cpu().numpy()


def _operand(rng, rows, ldx):
    """normals over many binades, exact zeros of both signs, subnormals and large values"""
    X = (rng.standard_normal((rows, ldx)) * np.exp2(rng.integers(-20, 20, (rows, ldx)))).astype(np.float32)
    pick = rng.random((rows, ldx))
    X[pick < 0.05] = 0.0
    X[(pick >= 0.05) & (pick < 0.08)] = -0.0
    sub = (pick >= 0.08) & (pick < 0.11)
    X[sub] = (rng.standard_normal(sub.sum()) * 1e-39).astype(np.float32)
    big = (pick >= 0.11) & (pick < 0.13)
    X[big] = (rng.standard_normal(big.sum()) * 1e30).astype(np.float32)
    return X


@pytest.mark.parametrize("max_ctas", [1, 3, 0])          # 0: one CTA per SM, as the engines run
@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("div", [1, 8])
@pytest.mark.parametrize("K,Kv", [(64, 63), (128, 128), (256, 256)])
def test_wgrad_operand_exact(K, Kv, div, passes, max_ctas):
    """M = 3001 rows (94 k-steps, the last one ragged) into N = 300 output rows (3 A row tiles): with 1 or 3 CTAs each
    CTA walks several units and its ring wraps across them, with one CTA per SM the rows split into short k-ranges."""
    M, N = 3001, 300
    rng = np.random.default_rng(K * 1000 + div * 100 + passes * 10 + max_ctas)
    ldx = K + (4 if div == 1 else 1)        # 16-byte aligned rows (L2 prefetch) and odd rows (none)
    rows = -(-M // div)
    X = _operand(rng, rows, ldx)
    sel = rng.choice(M, N, replace=False)
    sel[:3] = [M - 1, 0, 32 * (M // 32)]    # last row, first row, first row of the ragged k-step
    G = np.zeros((M, N), np.float32)
    G[sel, np.arange(N)] = 1.0
    bits = torch.full((M, -(-K // 32)), 0x55555555, dtype=torch.int32, device="cuda")
    dW = _run(torch.from_numpy(G).cuda(), torch.from_numpy(X).cuda(), M, N, K, Kv, ldx, div, passes, max_ctas, bits)
    want = _split_value(X[sel // div, :K], passes)
    want[:, Kv:] = 0.0
    bad = ~((dW == want) | (np.isnan(dW) & np.isnan(want)))
    assert not bad.any(), (np.argwhere(bad)[:5], dW[bad][:5], want[bad][:5])
    got_bits = bits.cpu().numpy().view(np.uint32)
    assert np.array_equal(got_bits, _mask_bits(X, M, K, div))


@pytest.mark.parametrize("div", [1, 3])
@pytest.mark.parametrize("M", [1, 77, 1000])
@pytest.mark.parametrize("K", [64, 96, 128, 256])
def test_wgrad_mask_bits(K, M, div):
    """Every word of the bit buffer equals the host's packing of X > 0: NaN, -0, +0 and -inf masked, +inf kept.  The
    words are written by the pack of the weight gradient's B operand, one block per 32 rows and 128 columns of X, each
    word by one warp ballot, before the GEMM runs; K = 96 leaves that block's last word outside K, M = 77 and 1000 end
    in a partial block of rows."""
    N = 8
    rng = np.random.default_rng(K * 7919 + M * 31 + div * 3)
    rows = -(-M // div)
    X = rng.standard_normal((rows, K)).astype(np.float32)
    pick = rng.random((rows, K))
    X[pick < 0.1] = np.nan
    X[(pick >= 0.1) & (pick < 0.2)] = -0.0
    X[(pick >= 0.2) & (pick < 0.3)] = 0.0
    X[(pick >= 0.3) & (pick < 0.32)] = np.inf
    X[(pick >= 0.32) & (pick < 0.34)] = -np.inf
    bits = torch.full((M, -(-K // 32)), 0x55555555, dtype=torch.int32, device="cuda")   # a word left unwritten shows
    G = torch.zeros((M, N), device="cuda")
    _run(G, torch.from_numpy(X).cuda(), M, N, K, K, K, div, 3, 0, bits)
    got = bits.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, _mask_bits(X, M, K, div))


def _image_values(img, rows, cols):
    """hi + lo 2^-11 of a 3-pass bf16 image of a [rows x cols] matrix (tiles of 128 rows x 32 columns, hi and lo halves
    adjacent, each in wgmma's no-swizzle K-major layout)"""
    r = np.arange(128)[:, None]
    k = np.arange(32)[None, :]
    off = (((r >> 3) * 4 + (k >> 3)) << 6) + ((r & 7) << 3) + (k & 7)
    rt, ks = -(-rows // 128), -(-cols // 32)
    t = img[: rt * ks * 2 * 4096].reshape(rt, ks, 2, 4096)[..., off]          # [rt, ks, half, 128, 32]
    f = (t.astype(np.uint32) << 16).view(np.float32)
    v = f[:, :, 0] + f[:, :, 1] * np.float32(2.0 ** -11)
    return v.transpose(0, 2, 1, 3).reshape(rt * 128, ks * 32)[:rows, :cols]


@pytest.mark.parametrize("max_ctas", [2, 0])
@pytest.mark.parametrize("K", [96, 256])
@pytest.mark.parametrize("M", [77, 1000])
def test_input_grad_bit_mask_matches_fp32_mask(M, K, max_ctas):
    """The input-gradient GEMM (row and transposed images, the epilogue of the trunk layers) gives bit-identical images
    whether its ReLU mask is the fp32 layer input or the bits the weight-gradient GEMM wrote of it: every column of a
    tile maps to the right bit of the right word, partial word tiles (K = 96) and partial row tiles included.  The
    images also hold (X > 0) * (G W) to fp32 accuracy, so the comparison is not between two empty outputs."""
    from sparf_b200 import _lib
    L = _lib.lib()
    N = 128
    rng = np.random.default_rng(M * 131 + K * 7 + max_ctas)
    G = rng.standard_normal((M, N)).astype(np.float32)
    W = rng.standard_normal((N, K)).astype(np.float32)
    X = rng.standard_normal((M, K)).astype(np.float32)
    pick = rng.random((M, K))
    X[pick < 0.05] = np.nan
    X[(pick >= 0.05) & (pick < 0.1)] = -0.0
    X[(pick >= 0.1) & (pick < 0.15)] = 0.0
    nrow = -(-M // 128) * -(-K // 32) * 8192
    ntr = -(-K // 128) * -(-M // 32) * 8192
    img = torch.empty(2 * (nrow + ntr), dtype=torch.int16, device="cuda")
    g, w, x = (torch.from_numpy(a).cuda() for a in (G, W, X))
    _lib.check(L.sparf_tc_selftest_mask_bits(_p(g), _p(w), _p(x), M, N, K, max_ctas, _p(img),
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_mask_bits")
    torch.cuda.synchronize()
    im = img.cpu().numpy().view(np.uint16)
    fp32_run, bit_run = im[: nrow + ntr], im[nrow + ntr:]
    assert np.array_equal(fp32_run, bit_run), np.argwhere(fp32_run != bit_run)[:5]
    want = np.where(X > 0, G.astype(np.float64) @ W.astype(np.float64), 0.0)
    got = _image_values(fp32_run[:nrow], M, K)
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()
    got_t = _image_values(fp32_run[nrow:], K, M)
    assert np.array_equal(got_t, got.T)
