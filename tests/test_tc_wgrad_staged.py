"""The weight-gradient GEMM that reads its B operand X as fp32 and splits it inside the GEMM (16-byte aligned X, ldx and
K multiples of 4 floats: every engine call), through sparf_tc_selftest_wgrad.

Checked exactly, either against the one-hot NumPy model of test_tc_wgrad_operand or against the pack path on the same
values (X copied to rows of K + 1 floats, which no bulk copy can read): with one CTA the atomics run in one order and the
two must be bit-identical.  X sits inside a larger buffer filled with NaN, so a row past M or a column past K that
reached an MMA or a mask word would show."""
import numpy as np
import pytest
import torch

from test_tc_wgrad_operand import _mask_bits, _operand, _run, _split_value

pytestmark = pytest.mark.gpu


def _embedded(X, ldx, col0=0, pad_rows=3):
    """X [rows x K] at column col0 of a NaN-filled [rows + pad_rows x ldx] buffer: the device view and its rows' start"""
    rows, K = X.shape
    buf = torch.full((rows + pad_rows, ldx), float("nan"), device="cuda")
    buf[:rows, col0:col0 + K] = torch.from_numpy(X).cuda()
    return buf[:, col0:]


def _bits(M, K):
    return torch.full((M, -(-K // 32)), 0x55555555, dtype=torch.int32, device="cuda")   # a word left unwritten shows


@pytest.mark.parametrize("max_ctas", [1, 3, 0])
@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("div", [1, 3, 128])
def test_staged_per_ray_rows(div, passes, max_ctas):
    """K = 32 with ldx = 32 and one row per `div` rows m, as the direction encoding of the colour head (div = samples
    per ray): each lane's bulk copy reads 128 bytes, and rows of one ray are copied once per row m"""
    M, N, K = 3001, 300, 32
    rng = np.random.default_rng(div * 100 + passes * 10 + max_ctas)
    rows = -(-M // div)
    X = _operand(rng, rows, K)
    sel = rng.choice(M, N, replace=False)
    sel[:3] = [M - 1, 0, 32 * (M // 32)]
    G = np.zeros((M, N), np.float32)
    G[sel, np.arange(N)] = 1.0
    bits = _bits(M, K)
    dW = _run(torch.from_numpy(G).cuda(), _embedded(X, K), M, N, K, K, K, div, passes, max_ctas, bits)
    want = _split_value(X[sel // div], passes)
    bad = ~((dW == want) | (np.isnan(dW) & np.isnan(want)))
    assert not bad.any(), (np.argwhere(bad)[:5], dW[bad][:5], want[bad][:5])
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), _mask_bits(X, M, K, div))


@pytest.mark.parametrize("max_ctas", [1, 3, 0])
@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("K,Kv,ldx,col0", [(256, 256, 320, 64), (64, 63, 96, 4), (96, 96, 100, 0)])
def test_staged_offset_source(K, Kv, ldx, col0, passes, max_ctas):
    """X at an offset inside a larger NaN-filled buffer with ldx > K, as a chunk of the tape; K = 96 leaves the last row
    tile's copies 384 bytes and its last mask word outside K, Kv < K drops a column of dW"""
    M, N = 2501, 200
    rng = np.random.default_rng(K * 1000 + ldx * 10 + passes + max_ctas)
    X = _operand(rng, M, K)
    sel = rng.choice(M, N, replace=False)
    sel[:2] = [M - 1, 32 * (M // 32)]
    G = np.zeros((M, N), np.float32)
    G[sel, np.arange(N)] = 1.0
    bits = _bits(M, K)
    dW = _run(torch.from_numpy(G).cuda(), _embedded(X, ldx, col0), M, N, K, Kv, ldx, 1, passes, max_ctas, bits)
    want = _split_value(X[sel], passes)
    want[:, Kv:] = 0.0
    bad = ~((dW == want) | (np.isnan(dW) & np.isnan(want)))
    assert not bad.any(), (np.argwhere(bad)[:5], dW[bad][:5], want[bad][:5])
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), _mask_bits(X, M, K, 1))


@pytest.mark.parametrize("passes", [1, 3])
def test_staged_special_values_match_pack_path(passes):
    """Values near the fp32 limit (whose lo half overflows), infinities and NaN split to the same bytes as in the pack
    kernel: with one CTA, dW is bit-identical, NaN payloads included"""
    M, N, K = 3001, 64, 128
    rng = np.random.default_rng(passes)
    X = _operand(rng, M, K)
    pick = rng.random((M, K))
    X[pick < 0.002] = np.nan
    X[(pick >= 0.002) & (pick < 0.004)] = np.inf
    X[(pick >= 0.004) & (pick < 0.006)] = -np.inf
    X[(pick >= 0.006) & (pick < 0.02)] = 3.3e38 * np.sign(rng.standard_normal(((pick >= 0.006) & (pick < 0.02)).sum()))
    G = torch.from_numpy((rng.random((M, N)) < 0.01).astype(np.float32)).cuda()
    got = [_run(G, _embedded(X, ld), M, N, K, K, ld, 1, passes, 1, None) for ld in (K, K + 1)]
    assert np.array_equal(got[0].view(np.uint32), got[1].view(np.uint32))


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("M", [131072, 131072 - 37])
def test_staged_matches_pack_path_large(M, passes):
    """4096 k-steps of random operands (a c2 chunk), each output tile over several k-ranges: with one CTA the staged GEMM
    and the pack path give bit-identical dW and bits; with one CTA per SM (the same k-ranges, their atomics in any
    order) they agree to the rounding of those few adds, a small fraction of sum_m |G[m][n] X[m][k]|"""
    N, K = 256, 256
    rng = np.random.default_rng(M + passes)
    G = torch.from_numpy(rng.standard_normal((M, N)).astype(np.float32)).cuda()
    X = rng.standard_normal((M, K)).astype(np.float32)
    staged_x = _embedded(X, K)
    packed_x = _embedded(X, K + 1)          # rows of 257 floats: the pack path
    out = {}
    for name, x, ld in (("staged", staged_x, K), ("packed", packed_x, K + 1)):
        for ctas in (1, 0):
            bits = _bits(M, K)
            out[name, ctas] = _run(G, x, M, N, K, K, ld, 1, passes, ctas, bits), bits.cpu().numpy()
    assert np.array_equal(out["staged", 1][0], out["packed", 1][0])
    bound = (G.abs().T @ torch.from_numpy(np.abs(X)).cuda()).cpu().numpy()
    assert (np.abs(out["staged", 0][0] - out["packed", 0][0]) <= 2.0 ** -16 * bound).all()
    want_bits = _mask_bits(X, M, K, 1)
    for key in out:
        assert np.array_equal(out[key][1].view(np.uint32), want_bits), key
