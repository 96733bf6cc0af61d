"""The staged weight-gradient GEMM's epilogue, which sums a CTA's consecutive units of one output tile (its k-ranges) in
shared memory and adds the sum to dW once (sparf_tc_selftest_wgrad and sparf_tc_selftest_wgrad_rows).

Small-integer operands are exact in bf16 and every partial sum stays an integer below 2^24, so any order of the adds
gives the same fp32 value: there dW must equal the fp64 product exactly, whatever the grid.  A lost, repeated or
misplaced partial shows as a wrong integer.  Random operands over a c2 chunk are checked against fp64 within the bound
of test_tc_wgrad_staged, 2^-16 sum_m |G[m][n] X[m][k]|."""
import ctypes

import numpy as np
import pytest
import torch

from test_tc_wgrad_operand import _bf16, _mask_bits, _p, _run
from test_tc_wgrad_staged import _bits, _embedded

pytestmark = pytest.mark.gpu


def _tiles(N, K):
    return -(-N // 128) * -(-K // 128)


def _int_operands(rng, rows, cols):
    return rng.integers(-2, 3, (rows, cols)).astype(np.float32)


def _exact(G, X, Kv):
    want = (torch.from_numpy(G).cuda().double().T @ torch.from_numpy(X).cuda().double()).cpu().numpy()
    want[:, Kv:] = 0.0
    return want


# max_ctas = the tile count: every CTA sums all k-ranges of one tile before its one flush; 2 x tiles: two CTAs per tile;
# 3 with 4 tiles: consecutive units of a CTA change tile, so each unit flushes its own partial
@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("N,K,Kv,ctas", [(256, 256, 256, 4), (256, 256, 256, 8), (256, 256, 256, 3), (200, 252, 250, 4),
                                         (100, 64, 64, 1), (100, 64, 64, 3)])
def test_presum_exact_on_integers(N, K, Kv, ctas, passes):
    """M = 100 003 rows (3126 k-steps, 4 k-ranges per tile at max_ctas = tiles): N = 200 and K = 252 leave partial row
    tiles on both sides of dW and Kv < K drops its last columns"""
    M = 100003
    rng = np.random.default_rng(N * 7 + K * 3 + ctas + passes)
    G = _int_operands(rng, M, N)
    X = _int_operands(rng, M, K)
    bits = _bits(M, K)
    dW = _run(torch.from_numpy(G).cuda(), _embedded(X, K), M, N, K, Kv, K, 1, passes, ctas, bits)
    want = _exact(G, X, Kv)
    assert np.array_equal(dW, want), (np.argwhere(dW != want)[:5], _tiles(N, K))
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), _mask_bits(X, M, K, 1))


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("max_ctas", [4, 0])       # the tile count; one CTA per SM, as the engines run
@pytest.mark.parametrize("M", [131072, 131072 - 37])
def test_presum_random_against_fp64(M, max_ctas, passes):
    """random operands over a c2 chunk at the trunk's shape (N = K = 256, 4 tiles)"""
    N = K = 256
    rng = np.random.default_rng(M + 10 * max_ctas + passes)
    G = rng.standard_normal((M, N)).astype(np.float32)
    X = rng.standard_normal((M, K)).astype(np.float32)
    dW = _run(torch.from_numpy(G).cuda(), _embedded(X, K), M, N, K, K, K, 1, passes, max_ctas, None)
    g, x = (G, X) if passes == 3 else (_bf16(G), _bf16(X))      # one pass: the products of the hi halves
    want = _exact(g, x, K)
    bound = (torch.from_numpy(np.abs(G)).cuda().double().T @ torch.from_numpy(np.abs(X)).cuda().double()).cpu().numpy()
    assert (np.abs(dW - want) <= 2.0 ** -16 * bound).all()


@pytest.mark.parametrize("passes", [1, 3])
@pytest.mark.parametrize("max_ctas", [4, 0])
@pytest.mark.parametrize("live", [100003, 131072, 0])
def test_presum_device_row_count(live, max_ctas, passes):
    """capacity 131 072 rows of which *rows are summed: the k-ranges are those of the live rows, computed on the device.
    X is NaN past them (never copied, zero in the split operand) and the mask words of those rows stay unwritten.  G is
    zero past them, as the images the engines write are (the last k-step's products with X's zeros must stay 0)."""
    C, N, K = 131072, 256, 256
    rng = np.random.default_rng(live + max_ctas + passes)
    G = _int_operands(rng, C, N)
    X = _int_operands(rng, C, K)
    G[live:] = 0.0
    X[live:] = np.nan
    rows = torch.tensor(live, dtype=torch.int64, device="cuda")
    bits = _bits(C, K)
    from sparf_b200 import _lib
    L = _lib.lib()
    dW = torch.full((N, K), -777.0, device="cuda")
    g, x = torch.from_numpy(G).cuda(), _embedded(X, K)
    _lib.check(L.sparf_tc_selftest_wgrad_rows(_p(g), _p(x), C, N, K, K, K, 1, passes, max_ctas, _p(rows), _p(dW),
                                              _p(bits), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_wgrad_rows")
    torch.cuda.synchronize()
    want = _exact(G[:live], X[:live], K)
    assert np.array_equal(dW.cpu().numpy(), want)
    got_bits = bits.cpu().numpy().view(np.uint32)
    assert np.array_equal(got_bits[:live], _mask_bits(X[:live], live, K, 1))
    assert (got_bits[live:] == 0x55555555).all()
