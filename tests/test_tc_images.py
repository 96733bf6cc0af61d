"""Operand images written by the tensor-core GEMM epilogues: exact-integer chain of three GEMMs (row image into a
two-segment NT operand, transposed image into the weight-gradient GEMM, column sums), bit-exact against torch."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("M", [128, 200, 333])
def test_tc_selftest_epilogue_images_exact(M):
    """Small integers keep every product and sum exact in the 3-pass bf16 split, so any layout, transpose, segment or
    padding error shows as a mismatch.  M = 200 and 333 leave ragged k-steps in the transposed image: they must read as
    zeros (the image buffers start as NaN)."""
    from sparf_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cpu").manual_seed(M)
    X = torch.randint(-2, 3, (M, 128), generator=g).float().cuda()
    W1 = torch.randint(-2, 3, (128, 96), generator=g).float().cuda()
    E = torch.randint(-2, 3, (M, 40), generator=g).float().cuda()
    W2 = torch.randint(-2, 3, (128, 136), generator=g).float().cuda()
    Y = torch.full((M, 128), -777.0, device="cuda")
    Z = torch.full((96, 128), -777.0, device="cuda")
    db = torch.full((96,), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_images(_p(X), _p(W1), _p(E), _p(W2), M, _p(Y), _p(Z), _p(db),
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "tc_selftest_images")
    torch.cuda.synchronize()
    D = X @ W1
    assert torch.equal(db, D.sum(0)), (db - D.sum(0)).abs().max().item()
    y_ref = torch.cat([D, E], 1) @ W2.t()
    assert torch.equal(Y, y_ref), (Y - y_ref).abs().max().item()
    z_ref = D.t() @ X
    assert torch.equal(Z, z_ref), (Z - z_ref).abs().max().item()
