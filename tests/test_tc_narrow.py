"""The narrow layers' backward on the tensor-core engines: the fused colour-head kernel (Ghid written straight into its
operand images, the head's and the density row's small gradients reduced per CTA) and the density row's weight
gradient summed in the last trunk layer's input-gradient epilogue."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

KEYS = sum([["mlp_feat.%d.weight" % i, "mlp_feat.%d.bias" % i] for i in range(8)], []) + \
    ["mlp_rgb.0.weight", "mlp_rgb.0.bias", "mlp_rgb.1.weight", "mlp_rgb.1.bias"]


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _cdiv(a, b):
    return -(-a // b)


@pytest.mark.parametrize("M,HW,row_passes,tr_passes", [(1, 128, 3, 3), (200, 128, 3, 3), (333, 128, 3, 1),
                                                       (1000, 128, 1, 1), (77, 200, 3, 3), (4100, 72, 3, 1)])
def test_tc_head_backward_images_bit_identical(M, HW, row_passes, tr_passes):
    """The fused kernel's Ghid images are byte for byte what the old path (fp32 Ghid, then the pack kernels) made of the
    same inputs, graw is bit-identical, and the zero padding past M and HW is written (the buffers start as 0xFFFF).
    M = 1, 200, 333, 77 leave ragged row tiles and k-steps; HW = 200 and 72 leave ragged column blocks."""
    from sparf_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cpu").manual_seed(M + HW)
    d_rgb = torch.randn(M, 3, generator=g).cuda()
    rgb = torch.rand(M, 3, generator=g).cuda()
    d_sigma = torch.randn(M, generator=g).cuda()
    raw = (torch.randn(M, generator=g) * 8).cuda()
    hid = torch.randn(M, HW, generator=g).cuda()            # about half masked
    W9 = torch.randn(3, HW, generator=g).cuda()
    nrow = _cdiv(M, 128) * _cdiv(HW, 32) * 8192
    ntr = _cdiv(HW, 128) * _cdiv(M, 32) * 8192
    img = torch.zeros(2 * (nrow + ntr), dtype=torch.int16, device="cuda")
    graw = torch.full((2, M), -777.0, device="cuda")
    _lib.check(L.sparf_tc_selftest_head(_p(d_rgb), _p(rgb), _p(d_sigma), _p(raw), _p(hid), _p(W9), M, HW, row_passes,
                                        tr_passes, _p(img), _p(graw),
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "tc_selftest_head")
    torch.cuda.synchronize()
    fused, ref = img[:nrow + ntr], img[nrow + ntr:]
    assert torch.equal(fused[:nrow], ref[:nrow]), "row image: %d elements differ" % (fused[:nrow] != ref[:nrow]).sum().item()
    assert torch.equal(fused[nrow:], ref[nrow:]), "transposed image: %d elements differ" % (fused[nrow:] != ref[nrow:]).sum().item()
    assert not (ref[:nrow] == -1).all() and not (ref[nrow:] == -1).all()
    assert torch.equal(graw[0], graw[1])


def _problem(R, S, seed):
    import common
    from sparf_b200 import ops
    opt = common.make_opt(S=S)
    sd = common.det_weights(opt, seed, peaky=True, sigma_bias=-3.0)
    params = [sd[k].cuda() for k in KEYS]
    g = torch.Generator(device="cpu").manual_seed(seed)
    o = (torch.randn(R, 3, generator=g) * 0.5).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    d = d / d.norm(dim=-1, keepdim=True) * (1 + 0.2 * torch.rand(R, 1, generator=g).cuda())
    t = torch.sort(torch.rand(R, S, generator=g) * 4 + 1.2, dim=1).values.cuda()
    return ops.MLPSpec(), params, o, d, t, sd["progress"].cuda()


def _narrow_grads(ps):
    """head_w[1], head_b[1], head_b[0], the density row of trunk_w[7] and its bias"""
    return {"head_w[1]": ps[18].grad, "head_b[1]": ps[19].grad, "head_b[0]": ps[17].grad,
            "trunk_w[7][0]": ps[14].grad[0], "trunk_b[7][0]": ps[15].grad[:1]}


# 333 x 96 rows are not a multiple of 128; 1023 x 128 is the c2 batch; 1100 x 128 takes two taped chunks of 131072 rows
@pytest.mark.parametrize("engine", ["tc_3x", "tc_3x_w1"])
@pytest.mark.parametrize("R,S", [(333, 96), (1023, 128), (1100, 128)])
def test_tc_narrow_gradients_match_oracle_and_simt(engine, R, S):
    """The narrow gradients of a tensor-core engine, taped and recomputed, against the fp64 oracle, within the bound
    test_tc_backward_matches_simt puts on every gradient: 2e-3 or 4 x the fp32 SIMT engine's own error."""
    from sparf_b200 import _lib, ops
    eng_id = {"tc_3x": _lib.ENGINE_TC_3X, "tc_3x_w1": _lib.ENGINE_TC_3X_W1}[engine]
    if not _lib.lib().sparf_engine_available(eng_id):
        pytest.skip("tensor-core engine not available")
    spec, params, o, d, t, prog = _problem(R, S, seed=R + 2)
    noise = torch.randn(R, S, device="cuda") * 0.3
    g = torch.Generator(device="cuda").manual_seed(5)
    gs = torch.randn(R, S, device="cuda", generator=g) * 1e-3
    gc = torch.randn(R, S, 3, device="cuda", generator=g) * 1e-3
    grads = {}
    for name, eng, tape in (("simt", _lib.ENGINE_SIMT_FP32, True), ("tc", eng_id, True), ("tc_recompute", eng_id, False)):
        ops.USE_TAPE[0] = tape
        try:
            ps = [p.clone().requires_grad_(True) for p in params]
            s, c = ops.mlp_forward(spec, o, d, t, ps, noise=noise, progress=prog, engine=eng)
            ((s * gs).sum() + (c * gc).sum()).backward()
            torch.cuda.synchronize()
        finally:
            ops.USE_TAPE[0] = True
        grads[name] = _narrow_grads(ps)
    from oracle import sparf_oracle as O
    p64 = {k: p.double().clone().requires_grad_(True) for k, p in zip(KEYS, params)}
    p64["progress"] = prog.double()
    pts = o.double()[None, :, None] + d.double()[None, :, None] * t.double()[None, ..., None]
    dens, rgb = O.mlp_forward(p64, pts, d.double()[None], noise=noise.double()[None])
    ((dens[0] * gs.double()).sum() + (rgb[0] * gc.double()).sum()).backward()
    truth = _narrow_grads([p64[k] for k in KEYS])
    for k, tr in truth.items():
        den = tr.abs().max().clamp_min(1e-30)
        e_simt = ((grads["simt"][k].double() - tr).abs().max() / den).item()
        for name in ("tc", "tc_recompute"):
            e = ((grads[name][k].double() - tr).abs().max() / den).item()
            vs_simt = ((grads[name][k] - grads["simt"][k]).abs().max() / grads["simt"][k].abs().max().clamp_min(1e-30)).item()
            print("%s R=%d S=%d %-14s %-13s err vs fp64 %.2e (simt %.2e), vs simt %.2e" % (engine, R, S, k, name, e, e_simt,
                                                                                       vs_simt))
            assert e < max(2e-3, 4 * e_simt), (k, name, e, e_simt)
