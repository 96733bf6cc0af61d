"""The persistent GEMM kernel's work loop: the three-GEMM exact-integer chain of test_tc_images.py with the grids capped
at a few CTAs, so that each CTA walks several output tiles (and, in the weight-gradient GEMM, uneven k-ranges) and its
copy ring wraps across them.  Bit-exact against torch."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("max_ctas", [1, 3, 0])     # 0: one CTA per SM, as the engines run
@pytest.mark.parametrize("M", [200, 333, 1000])
def test_tc_selftest_persistent_exact(M, max_ctas):
    """Small integers keep every product and sum exact in the 3-pass bf16 split.  With 1 or 3 CTAs the NN and NT GEMMs
    (up to 8 output tiles, 4 and 5 k-steps per tile) run several tiles per CTA through one 6-stage ring, and the
    weight-gradient GEMM splits its ceil(M / 32) k-steps into 1 or 3 ranges of unequal length.  The image buffers start
    as NaN, so a stage that is read before its copy lands, or a stale stage, shows as a mismatch."""
    from sparf_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cpu").manual_seed(1000 * M + max_ctas)
    X = torch.randint(-2, 3, (M, 128), generator=g).float().cuda()
    W1 = torch.randint(-2, 3, (128, 96), generator=g).float().cuda()
    E = torch.randint(-2, 3, (M, 40), generator=g).float().cuda()
    W2 = torch.randint(-2, 3, (128, 136), generator=g).float().cuda()
    Y = torch.full((M, 128), -777.0, device="cuda")
    Z = torch.full((96, 128), -777.0, device="cuda")
    db = torch.full((96,), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_persistent(_p(X), _p(W1), _p(E), _p(W2), M, _p(Y), _p(Z), _p(db), max_ctas,
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "tc_selftest_persistent")
    torch.cuda.synchronize()
    D = X @ W1
    assert torch.equal(db, D.sum(0)), (db - D.sum(0)).abs().max().item()
    y_ref = torch.cat([D, E], 1) @ W2.t()
    assert torch.equal(Y, y_ref), (Y - y_ref).abs().max().item()
    z_ref = D.t() @ X
    assert torch.equal(Z, z_ref), (Z - z_ref).abs().max().item()
