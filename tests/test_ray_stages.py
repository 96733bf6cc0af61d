"""The stages around the MLP (csrc/elementwise.cu) against the oracle (oracle/sparf_oracle.py) evaluated in fp64, at the
shapes where these kernels go wrong: partial warp chunks, block-reduction edges, non-power-of-two sorts, the composite
backward's large-shared-memory path, grid-stride loops longer than one stride, NULL gradient inputs.

Yardstick (as in test_cuda_parity.py::_error_vs_fp64): a kernel output's distance from the fp64 oracle is gated against
the distance of the SAME oracle evaluated in fp32 on the same inputs,  err_kernel <= C * err_oracle_fp32 + floor,
with C = 4 (the kernels sum in a different order than torch: a few times the fp32 oracle's own rounding, never a
systematic error) and a floor of a few fp32 ulps at the output's natural scale, stated at each use.  Distances are
max|x - exact| / scale.  Depth sampling is bit-exact against the fp32 oracle instead.
"""
import itertools

import pytest
import torch
import torch.nn.functional as F

from oracle import sparf_oracle as O

pytestmark = pytest.mark.gpu

C = 4.0
ULP = 2.0 ** -24        # half an fp32 ulp of 1: unit round-off


def _dist(x, exact, scale=None):
    """max|x - exact| / scale (scale defaults to max|exact|)."""
    x, exact = x.detach().double(), exact.detach().double()
    s = exact.abs().max().item() if scale is None else float(scale)
    return (x - exact).abs().max().item() / max(s, 1e-30)


def _gate(what, got, exact, fp32, floor, scale=None):
    ek, eo = _dist(got, exact, scale), _dist(fp32, exact, scale)
    assert ek <= C * eo + floor, "%s: kernel %.2e vs fp32 oracle %.2e (bound %.2e)" % (what, ek, eo, C * eo + floor)


def _lib():
    from sparf_b200 import _lib
    return _lib.lib()


# ------------------------------------------------------------------------------------------------ ray generation
def _cameras(B, H, W, seed):
    """Random rigid w2c poses [B,3,4] (rotation from a QR, translation ~ 3) and pinhole intrinsics [B,3,3] for an HxW
    image, fp64 on the GPU."""
    g = torch.Generator().manual_seed(seed)
    q, r = torch.linalg.qr(torch.randn(B, 3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r, dim1=-2, dim2=-1))[:, None, :]
    t = torch.randn(B, 3, 1, generator=g, dtype=torch.float64) * 3
    pose = torch.cat([q, t], dim=-1)
    f = 0.8 * max(H, W) * (1 + 0.1 * torch.rand(B, generator=g, dtype=torch.float64))
    K = torch.zeros(B, 3, 3, dtype=torch.float64)
    K[:, 0, 0], K[:, 1, 1] = f, f * 1.05
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = W / 2 + 3.25, H / 2 - 1.5, 1.0
    # round to fp32 first: kernel, fp32 oracle and fp64 oracle then see the same numbers
    return pose.float().double().cuda(), K.float().double().cuda()


def _ray_idx(shape, H, W, seed):
    """Random flat pixel indices with the image's last pixels (H*W - 1, the start of the last row, ...) at the end."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, H * W, shape, generator=g)
    edge = torch.tensor([H * W - 1, H * W - 2, (H - 1) * W, W - 1, 0])
    k = min(len(edge), shape[-1])
    idx[..., shape[-1] - k:] = edge[:k]
    return idx.cuda()


def _centres(idx, W):
    """The pixel centres (x + 0.5, y + 0.5) of flat indices y*W + x (camera.py:363-368), fp64 [..., 2]."""
    idx = idx.long()
    return torch.stack([(idx % W).double() + 0.5, (idx // W).double() + 0.5], dim=-1)


RAY_B = [1, 3, 9]
RAY_N = [1, 127, 128, 129, 255, 256, 257, 4099]     # forward block 128 threads, backward block 256 + 12x8 reduction
SOURCES = ["idx_shared", "idx_per_image", "px_shared", "px_per_image"]


def _raygen_case(pose64, K_arg64, W, src, uv64, idx, g_o, g_d):
    """Kernel and oracle (fp64, fp32) rays and gradients for one pixel source: origins, dirs, d_pose, d_pixels (None for
    indices).  The oracle sees the pixel centres of the indices; g_o / g_d None leave that output out of the loss."""
    from sparf_b200 import ops
    res = []
    for dt in (None, torch.float64, torch.float32):
        pose = pose64.to(dt or torch.float32, copy=True).requires_grad_(True)
        px = uv64.to(dt or torch.float32, copy=True).requires_grad_(True) if idx is None else None
        if dt is None:
            kw = dict(pixels=px) if idx is None else dict(ray_idx=idx)
            o, d = ops.raygen(pose, K_arg64.float(), W, **kw)
        else:
            uv = px if idx is None else uv64.to(dt)
            if uv.dim() == 3 and uv.shape[0] == 1:     # the oracle takes a shared list as [n,2] or expanded to [B,n,2]
                uv = uv.expand(pose.shape[0], -1, -1)
            o, d = O.rays_at_pixels(pose, K_arg64.to(dt), uv)
        loss = 0
        if g_o is not None:
            loss = loss + (o * g_o.to(o.dtype)).sum()
        if g_d is not None:
            loss = loss + (d * g_d.to(d.dtype)).sum()
        loss.backward()
        res.append((o, d, pose.grad, None if px is None else px.grad))
    return res


def _gate_rays(tag, res, grads=True):
    """Floors: 8 unit round-offs of the tensor's largest entry for origins and directions (a few fp32 products and sums
    per entry); 64 for the gradients, which are sums over up to 4099 rays (and B images for a shared pixel list)."""
    (o, d, gp, gx), (o64, d64, gp64, gx64), (o32, d32, gp32, gx32) = res
    assert o.shape == d.shape == o64.shape, (tag, o.shape, o64.shape)
    _gate(tag + " origins", o, o64, o32, 8 * ULP)
    _gate(tag + " dirs", d, d64, d32, 8 * ULP)
    if grads:
        _gate(tag + " d_pose", gp, gp64, gp32, 64 * ULP)
        if gx64 is not None:
            assert gx.shape == gx64.shape
            _gate(tag + " d_pixels", gx, gx64, gx32, 64 * ULP)


@pytest.mark.parametrize("n", RAY_N)
@pytest.mark.parametrize("B", RAY_B)
def test_raygen_vs_fp64(B, n):
    """ops.raygen forward and backward for shared / per-image ray indices into a 3000x4000 image (the last pixels
    included) and shared / per-image float pixels, against fp64 autograd through O.rays_at_pixels: origins and
    directions, the pose gradient with g_o only, g_d only and both, and the pixel gradient (per image, or summed over
    the B images by atomics for a shared list)."""
    H, W = 3000, 4000
    pose64, K64 = _cameras(B, H, W, seed=B * 1000 + n)
    g = torch.Generator(device="cuda").manual_seed(n)
    g_o = torch.randn(B, n, 3, device="cuda", generator=g)
    g_d = torch.randn(B, n, 3, device="cuda", generator=g)
    for src in SOURCES:
        if src.startswith("idx"):
            idx = _ray_idx((n,) if src == "idx_shared" else (B, n), H, W, seed=n + B)
            uv64 = _centres(idx, W)
        else:
            idx = None
            shape = (n, 2) if src == "px_shared" else (B, n, 2)
            scale = torch.tensor([W, H], device="cuda", dtype=torch.float64)
            uv64 = (torch.rand(shape, device="cuda", generator=g, dtype=torch.float64) * scale).float().double()
        for go, gd in ((g_o, None), (None, g_d), (g_o, g_d)):
            tag = "B=%d n=%d %s g_o=%d g_d=%d" % (B, n, src, go is not None, gd is not None)
            _gate_rays(tag, _raygen_case(pose64, K64, W, src, uv64, idx, go, gd))


def test_raygen_small_image_matches_oracle_indexing():
    """Indices into a small odd-sized image against the oracle's full-grid-then-gather path (O.rays_from_ray_idx), which
    pins the idx = y*W + x, +0.5 convention for shared and per-image indices."""
    from sparf_b200 import ops
    B, H, W = 3, 17, 23
    pose64, K64 = _cameras(B, H, W, seed=5)
    for idx in (_ray_idx((131,), H, W, 1), _ray_idx((B, 131), H, W, 2)):
        o, d = ops.raygen(pose64.float(), K64.float(), W, ray_idx=idx)
        o64, d64 = O.rays_from_ray_idx(pose64, K64, H, W, idx)
        o32, d32 = O.rays_from_ray_idx(pose64.float(), K64.float(), H, W, idx)
        _gate("origins", o, o64, o32, 8 * ULP)
        _gate("dirs", d, d64, d32, 8 * ULP)


# intrinsics as passed ([B,3,3], [1,3,3] or [3,3]) and pixel source as passed
BROADCAST = {"intr_1": ("K1", "px_b"), "intr_2d": ("K2d", "px_shared"), "pixels_1": ("KB", "px_1"),
             "ray_idx_1": ("KB", "idx_1"), "intr_1_pixels_1": ("K1", "px_1")}


@pytest.mark.parametrize("form", list(BROADCAST))
def test_raygen_broadcast_shapes(form):
    """Intrinsics [1,3,3] / [3,3] shared by B poses, pixels [1,n,2] and indices [1,n] shared by the B images: the rays
    and gradients the oracle's broadcasting gives (a pixel gradient of the caller's shape, summed over the images)."""
    B, n, H, W = 3, 300, 48, 64
    pose64, K64 = _cameras(B, H, W, seed=11)
    kform, src = BROADCAST[form]
    K_arg = {"K1": K64[:1], "K2d": K64[0], "KB": K64[:1].expand(B, 3, 3).contiguous()}[kform]
    g = torch.Generator(device="cuda").manual_seed(3)
    g_o = torch.randn(B, n, 3, device="cuda", generator=g)
    g_d = torch.randn(B, n, 3, device="cuda", generator=g)
    if src == "idx_1":
        from sparf_b200 import ops
        idx = _ray_idx((1, n), H, W, 4)
        o, d = ops.raygen(pose64.float(), K_arg.float(), W, ray_idx=idx)
        o64, d64 = O.rays_from_ray_idx(pose64, K_arg, H, W, idx)       # [B,1,n,3]: the same rays as a shared [n] list
        o32, d32 = O.rays_from_ray_idx(pose64.float(), K_arg.float(), H, W, idx)
        _gate(form + " origins", o, o64.reshape(B, n, 3), o32.reshape(B, n, 3), 8 * ULP)
        _gate(form + " dirs", d, d64.reshape(B, n, 3), d32.reshape(B, n, 3), 8 * ULP)
        return
    shape = {"px_b": (B, n, 2), "px_shared": (n, 2), "px_1": (1, n, 2)}[src]
    uv64 = (torch.rand(shape, device="cuda", generator=g, dtype=torch.float64) * 60).float().double()
    _gate_rays(form, _raygen_case(pose64, K_arg, W, src, uv64, None, g_o, g_d))


@pytest.mark.parametrize("case", ["pose_2d", "pose_4x4", "intr_b", "intr_4x4", "pixels_b", "pixels_3col", "pixels_1d",
                                  "ray_idx_b", "ray_idx_3d", "both", "neither"])
def test_raygen_rejects_bad_shapes(case):
    """Shapes the kernel would index out of bounds (or silently misread) raise ValueError before any launch: a 2-D pose,
    intrinsics or pixels for a different number of images, ray indices [B',n] with B' not in {1, B}."""
    from sparf_b200 import ops
    B, n, W = 3, 64, 40
    pose = torch.eye(3, 4, device="cuda").expand(B, 3, 4).contiguous()
    K = torch.tensor([[50.0, 0, 20], [0, 50.0, 15], [0, 0, 1]], device="cuda").expand(B, 3, 3).contiguous()
    px = torch.rand(n, 2, device="cuda") * 30
    idx = torch.arange(n, device="cuda")
    args = {
        "pose_2d": (pose[0], K[:1], dict(pixels=px)),
        "pose_4x4": (torch.eye(4, device="cuda").expand(B, 4, 4), K, dict(pixels=px)),
        "intr_b": (pose, K[:2], dict(pixels=px)),
        "intr_4x4": (pose, torch.eye(4, device="cuda").expand(B, 4, 4), dict(pixels=px)),
        "pixels_b": (pose, K, dict(pixels=px.expand(2, n, 2))),
        "pixels_3col": (pose, K, dict(pixels=torch.rand(n, 3, device="cuda"))),
        "pixels_1d": (pose, K, dict(pixels=px.reshape(-1))),
        "ray_idx_b": (pose, K, dict(ray_idx=idx.expand(2, n))),
        "ray_idx_3d": (pose, K, dict(ray_idx=idx.reshape(1, n, 1).expand(B, n, 1))),
        "both": (pose, K, dict(ray_idx=idx, pixels=px)),
        "neither": (pose, K, dict()),
    }[case]
    torch.cuda.synchronize()
    n0 = _lib().sparf_launch_count()
    with pytest.raises(ValueError):
        ops.raygen(args[0], args[1], W, **args[2])
    assert _lib().sparf_launch_count() == n0


# ------------------------------------------------------------------------------------------------ depth sampling
@pytest.mark.parametrize("S", [1, 7, 64, 129])
@pytest.mark.parametrize("R", [1, 37, 1001])
def test_sample_depth_bit_exact_vs_oracle(R, S):
    """Metric and inverse depth, each with and without stratification, and the per-ray far bound: bit for bit the fp32
    oracle (the kernel follows torch's op order and rounding), at S = 1 and R*S not a multiple of the 256-thread block."""
    from sparf_b200 import ops
    g = torch.Generator().manual_seed(R * 131 + S)
    rng32 = torch.tensor([0.35, 6.2])
    rand = torch.rand(R, S, generator=g)
    for param, with_rand in itertools.product(("metric", "inverse"), (False, True)):
        near, far = rng32[0], rng32[1]
        t = ops.sample_depth(R, S, float(near), float(far - near), inverse=param == "inverse",
                             rand=rand.cuda() if with_rand else None, device="cuda")
        ref = O.sample_depth(1, R, S, rng32, param=param, rand=rand if with_rand else None)[0]
        assert torch.equal(t.cpu(), ref), (param, with_rand, (t.cpu() - ref).abs().max().item())
    far_r = torch.rand(R, generator=g) * 5 + 0.5
    t = ops.sample_depth(R, S, float(rng32[0]), 0.0, far_per_ray=far_r.cuda())
    ref = O.sample_depth_to_max(far_r, S, rng32[0])
    assert torch.equal(t.cpu(), ref), (t.cpu() - ref).abs().max().item()


# ------------------------------------------------------------------------------------------------ resampling + merge
PDF_SIZES = [(1, 1), (33, 31), (64, 128), (5, 250), (2048, 2048), (4095, 1)]
PDF_WEIGHTS = ["random", "zero", "onehot_first", "onehot_last", "zero_runs"]


def _pdf_weights(kind, R, S, g):
    w = torch.rand(R, S, generator=g, dtype=torch.float64)
    if kind == "zero":
        w.zero_()
    elif kind == "onehot_first":
        w = torch.zeros_like(w); w[:, 0] = 0.5 + w[:, 0]
    elif kind == "onehot_last":
        w = torch.zeros_like(w); w[:, -1] = 0.5 + w[:, -1]
    elif kind == "zero_runs":    # leading and trailing zero runs of different lengths per ray, a zero run in between
        for r in range(R):
            a, b = int(torch.randint(0, S, (1,), generator=g)), int(torch.randint(0, S, (1,), generator=g))
            w[r, : min(a, b)] = 0
            w[r, max(a, b) + 1:] = 0
            w[r, (a + b) // 2: (a + b) // 2 + S // 8] = 0
    return w.float()


def _pdf_u(Sf, g, cdf32):
    """Uniform u after three edge values: 0 (against a zero prefix searchsorted must take the right side), a value of the
    fp32 cdf itself (a tie, on a plateau where the weights have zeros) and 1.  Returns (u, number of edge values)."""
    u = torch.rand(Sf, generator=g)
    special = [0.0, float(cdf32[0, cdf32.shape[1] // 2]), 1.0][:Sf]
    u[: len(special)] = torch.tensor(special)
    return u, len(special)


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("S,Sf", PDF_SIZES)
def test_sample_pdf_merge_vs_fp64(S, Sf, descending):
    """t_fine against the fp64 oracle (u given directly) for random, all-zero, one-hot-first/-last and zero-run weights,
    ascending and descending bins; t_all is cat(t_coarse, t_fine) sorted, bit for bit.  u within a margin of an fp64 cdf
    value is masked (there a last-bit change of the cdf legitimately moves a sample across a plateau): the margin is 4x
    the fp32 oracle cdf's own distance from fp64 plus 4 unit round-offs, and at most 5% of the samples may be masked.
    Floor: 8 unit round-offs of max |t| (one interpolation, a handful of roundings)."""
    from sparf_b200 import ops
    near, far = (4.0, 0.5) if descending else (0.5, 6.0)
    R = 37 if S + Sf <= 512 else 3
    g = torch.Generator().manual_seed(S * 7 + Sf)
    t_c = torch.sort(torch.rand(R, S, generator=g) * abs(far - near) + min(near, far), dim=1,
                     descending=descending).values.cuda()
    for kind in PDF_WEIGHTS:
        w = _pdf_weights(kind, R, S, g).cuda()
        pdf32 = w / (w.sum(-1, keepdim=True) + 1e-6)
        cdf32 = torch.cat([torch.zeros_like(pdf32[:, :1]), pdf32.cumsum(-1)], dim=-1)
        u, n_edge = _pdf_u(Sf, g, cdf32)
        u = u.cuda()
        t_f, t_all = ops.sample_pdf_merge(w, t_c, u, near, far)
        assert torch.equal(t_all, torch.cat([t_c, t_f], dim=1).sort(dim=1).values), kind
        ref64 = O.sample_pdf(w.double(), S, Sf, (near, far), u=u.double())
        ref32 = O.sample_pdf(w, S, Sf, (near, far), u=u)
        if kind == "zero":       # denominator 1e-6 alone: the cdf is 0 everywhere and every sample lands on far
            assert (t_f == far).all()
            continue
        w64 = w.double()
        cdf64 = torch.cat([torch.zeros_like(w64[:, :1]), (w64 / (w64.sum(-1, keepdim=True) + 1e-6)).cumsum(-1)], dim=-1)
        margin = 4 * (cdf32.double() - cdf64).abs().max().item() + 4 * ULP
        pos = torch.searchsorted(cdf64, u.double().expand(R, Sf).contiguous())
        nb = torch.minimum((cdf64.gather(1, pos.clamp(max=S)) - u.double()).abs(),
                           (cdf64.gather(1, (pos - 1).clamp(min=0)) - u.double()).abs())
        keep = nb > margin
        if Sf > n_edge:
            assert keep[:, n_edge:].double().mean().item() >= 0.95, (kind, keep[:, n_edge:].double().mean().item())
        scale = max(abs(near), abs(far))
        # u = 0 is an exact tie with the zero prefix of every cdf, in fp32 and in the kernel alike: never masked
        assert _dist(t_f[:, 0], ref32[:, 0], scale) <= 8 * ULP, (kind, "u = 0")
        ek = ((t_f.double() - ref64).abs() * keep).max().item() / scale
        eo = ((ref32.double() - ref64).abs() * keep).max().item() / scale
        assert ek <= C * eo + 8 * ULP, (kind, ek, eo)
    # ties: u equal to a plateau value of the fp32 cdf (bit for bit the kernel's: one nonzero weight then zeros) takes the
    # bin AFTER the plateau (searchsorted right=True), exactly as the fp32 oracle does
    if S >= 4 and Sf >= 2:
        w = torch.zeros(R, S, device="cuda"); w[:, 0] = 0.25; w[:, S // 2] = 0.5
        c = (w[:, :1] / (w.sum(-1, keepdim=True) + 1e-6))[0]
        u = torch.full((Sf,), float(c), device="cuda"); u[0] = 0.0
        t_f, _ = ops.sample_pdf_merge(w, t_c, u, near, far)
        ref32 = O.sample_pdf(w, S, Sf, (near, far), u=u)
        assert _dist(t_f, ref32, max(abs(near), abs(far))) <= 8 * ULP
        step = (far - near) / S
        assert abs(float(t_f[0, -1]) - (near + step * (S // 2))) <= 1e-5 * abs(far)
        assert abs(float(t_f[0, 0]) - near) <= 1e-6 * abs(far)      # u = 0 before the first (nonzero) weight's bin


def test_sample_pdf_merge_limit():
    """S + S_fine = 4096 runs; 4097 raises an error naming the limit, before any launch."""
    from sparf_b200 import ops
    w = torch.rand(2, 4095, device="cuda")
    t_c = torch.sort(torch.rand(2, 4095, device="cuda"), dim=1).values
    ops.sample_pdf_merge(w, t_c, torch.rand(1, device="cuda"), 0.0, 1.0)
    torch.cuda.synchronize()
    n0 = _lib().sparf_launch_count()
    with pytest.raises(RuntimeError, match="S \\+ S_fine <= 4096"):
        ops.sample_pdf_merge(w, t_c, torch.rand(2, device="cuda"), 0.0, 1.0)
    assert _lib().sparf_launch_count() == n0


# ------------------------------------------------------------------------------------------------ compositing
COMP_S = [2, 3, 31, 32, 33, 95, 257, 1536, 1537, 4096]     # backward: 8*S floats of smem per block, > 48 KB above 1536
REGIMES = ["random", "transparent", "opaque", "zero_runs", "short_dirs", "descending"]
OUTS = ["rgb", "depth", "opacity", "weights", "depth_var", "rgb_var", "all_cumulated"]


def _comp_cases():
    for S in COMP_S:
        for R in (1, 5, 4097):
            if R * S <= 4097 * 257 or R == 1 or R == 5:     # fp64 autograd stays at a few hundred MB
                yield R, S


def _composite_inputs(R, S, regime, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.sort(torch.rand(R, S, device="cuda", generator=g) * 4 + 1, dim=1, descending=regime == "descending").values
    dirs = torch.randn(R, 3, device="cuda", generator=g)
    if regime == "short_dirs":   # non-unit and very short rays
        lens = torch.tensor([1e-4, 1e-2, 1.0, 30.0], device="cuda")[torch.arange(R, device="cuda") % 4]
        dirs = dirs / dirs.norm(dim=-1, keepdim=True) * lens[:, None]
    rgb = torch.rand(R, S, 3, device="cuda", generator=g)
    sigma = torch.rand(R, S, device="cuda", generator=g) * (0.5 if regime == "descending" else 3.0)
    gaps = torch.cat([t[:, 1:] - t[:, :-1], torch.ones_like(t[:, :1])], dim=1).abs().clamp_min(1e-6) * dirs.norm(dim=-1,
                                                                                                             keepdim=True)
    if regime == "transparent":     # sigma * delta ~ 1e-4 (the last sample's 1e10 gap still makes it opaque)
        sigma = 1e-4 / gaps * (0.5 + torch.rand(R, S, device="cuda", generator=g))
    elif regime == "opaque":        # optical depth ~ 200 by the middle of the ray: T underflows to 0 halfway
        sigma = (400.0 / S) / gaps * (0.5 + torch.rand(R, S, device="cuda", generator=g))
    elif regime == "zero_runs":     # sigma = 0 runs (empty space, as the occupancy-grid passes feed it), last sample too
        keep = torch.rand(R, S // 8 + 1, device="cuda", generator=g) < 0.5
        sigma = sigma * keep.repeat_interleave(8, dim=1)[:, :S]
        sigma[:, -1] = 0
        sigma[::3] = 0               # whole rays of empty space
    return sigma, rgb, t, dirs


def _oracle_composite(sigma, rgb, t, dirs, white_bg, dt, need_dirs):
    s = sigma.detach().to(dt).requires_grad_(True)
    c = rgb.detach().to(dt).requires_grad_(True)
    d = dirs.detach().to(dt).requires_grad_(need_dirs)
    out = O.composite(d[None], s[None], c[None], t.to(dt)[None], white_bg=white_bg)
    res = dict(rgb=out["rgb"][0], depth=out["depth"][0, :, 0], opacity=out["opacity"][0, :, 0],
               weights=out["weights"][0, :, :, 0], depth_var=out["depth_var"][0, :, 0], rgb_var=out["rgb_var"][0, :, 0],
               all_cumulated=out["all_cumulated"][0])
    return res, (s, c, d)


def _out_scale(k, t, exact):
    """Natural scale of an output, so that a floor in unit round-offs means the same for every output: colours, opacity,
    weights and transmittance are O(1) (larger with descending t, where T grows); depth O(max t); depth_var O(max t^2)."""
    tm = t.abs().max().item()
    return max({"depth": tm, "depth_var": tm * tm}.get(k, 1.0), exact.abs().max().item())


@pytest.mark.parametrize("white_bg", [False, True])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("R,S", list(_comp_cases()))
def test_composite_vs_fp64(R, S, regime, white_bg):
    """ops.composite forward (all seven outputs) and backward for every non-empty subset of {rgb, depth, opacity,
    weights} used downstream (the unused ones reach the kernel as NULL), with and without a gradient for dirs.
    Distances are per tensor, at the output's natural scale (forward), or for a gradient relative to its largest exact
    entry or, if larger, that of the same tensor's gradient with all four outputs used: a subset whose exact gradient
    cancels to almost nothing (opacity alone is 1 - T_S, and T_S = 0 whenever the last sample is dense: d opacity /
    d sigma is 0 up to rounding) leaves only the rounding noise of the terms that cancelled, at that scale.
    Floors: 64 unit round-offs forward, 256 for gradients: the kernel's 32-lane chunked scans and sums run over up to
    4096 samples (up to 128 sequential fp32 additions per lane), torch's over a tree."""
    from sparf_b200 import ops
    sigma, rgb, t, dirs = _composite_inputs(R, S, regime, seed=R * 10007 + S * 13 + REGIMES.index(regime))
    exact, leaves64 = _oracle_composite(sigma, rgb, t, dirs, white_bg, torch.float64, True)
    f32, leaves32 = _oracle_composite(sigma, rgb, t, dirs, white_bg, torch.float32, True)
    for need_dirs in (True, False):
        s_k, c_k, d_k = sigma.clone().requires_grad_(True), rgb.clone().requires_grad_(True), dirs.clone().requires_grad_(need_dirs)
        outs = dict(zip(OUTS[:4] + ["depth_var", "rgb_var", "all_cumulated"], ops.composite(s_k, c_k, t, d_k, white_bg)))
        if need_dirs:
            for k in OUTS:
                _gate("%s fwd %s" % (regime, k), outs[k], exact[k], f32[k], 64 * ULP, _out_scale(k, t, exact[k]))
        gen = torch.Generator(device="cuda").manual_seed(S)
        ups = {k: torch.randn(exact[k].shape, device="cuda", generator=gen) for k in OUTS[:4]}
        grad_scale = {}
        for m in range(15, 0, -1):      # all four outputs first: their gradients set the scale of each tensor
            used = [k for i, k in enumerate(OUTS[:4]) if m >> i & 1]
            ins_k = [s_k, c_k] + ([d_k] if need_dirs else [])
            got = torch.autograd.grad([outs[k] for k in used], ins_k, [ups[k] for k in used], retain_graph=True,
                                      allow_unused=True)
            refs = []
            for res, leaves in ((exact, leaves64), (f32, leaves32)):
                ins = list(leaves[:2]) + ([leaves[2]] if need_dirs else [])
                refs.append(torch.autograd.grad([res[k] for k in used], ins, [ups[k].to(res[k].dtype) for k in used],
                                                retain_graph=True, allow_unused=True))
            for name, gk, g64, g32 in zip(("d_sigma", "d_rgb", "d_dirs"), got, refs[0], refs[1]):
                if g64 is None:     # no dependence (d_rgb when only opacity / weights are used): the kernel writes zeros
                    assert gk is None or gk.abs().max().item() == 0, (used, name)
                    continue
                scale = max(g64.abs().max().item(), grad_scale.setdefault(name, g64.abs().max().item()))
                if scale == 0:
                    continue
                _gate("%s bwd %s %s" % (regime, used, name), gk, g64, g32, 256 * ULP, scale)


def test_composite_zero_rays():
    from sparf_b200 import ops
    sigma = torch.zeros(0, 40, device="cuda", requires_grad=True)
    rgb = torch.zeros(0, 40, 3, device="cuda", requires_grad=True)
    dirs = torch.zeros(0, 3, device="cuda", requires_grad=True)
    outs = ops.composite(sigma, rgb, torch.zeros(0, 40, device="cuda"), dirs, True)
    assert [o.shape[0] for o in outs] == [0] * 7
    (outs[0].sum() + outs[3].sum()).backward()
    assert sigma.grad.shape == (0, 40) and rgb.grad.shape == (0, 40, 3) and dirs.grad.shape == (0, 3)


def test_composite_backward_limit():
    """The forward has no upper limit on S; the backward keeps 2*S floats per ray in shared memory and raises an error
    naming its S <= 4096 limit, before any launch."""
    from sparf_b200 import ops
    R, S = 2, 4097
    sigma, rgb, t, dirs = _composite_inputs(R, S, "random", seed=0)
    sigma.requires_grad_(True)
    out = ops.composite(sigma, rgb, t, dirs)
    assert torch.isfinite(out[0]).all()
    torch.cuda.synchronize()
    n0 = _lib().sparf_launch_count()
    with pytest.raises(RuntimeError, match="S <= 4096"):
        out[0].sum().backward()
    assert _lib().sparf_launch_count() == n0


# ------------------------------------------------------------------------------------------------ Huber loss
HUBER_N = [1, 3, 255, 256, 257, 262143, 262144, 262145, 3 * 2 ** 20]   # grid-stride loop: 1024 x 256 threads per stride


@pytest.mark.parametrize("n", HUBER_N)
def test_huber2_vs_fp64(n):
    """ops.huber2 loss and gradient against 2 * F.huber_loss(delta=0.5) in fp64, with residuals of exactly +-0.5 (the
    branch point) and large |z|, for a full target and a broadcast one.  Floors: loss 64 unit round-offs (a sum over the
    grid-stride loop and warps, then up to 1024 block sums added by fp32 atomics in arbitrary order: a random walk of
    up to 1024 roundings, measured 20 unit round-offs at n = 262143 on an H100); gradient 4 unit round-offs per element
    (norm * z: two roundings)."""
    from sparf_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    pred = torch.randn(n, device="cuda", generator=g)
    target = torch.randn(n, device="cuda", generator=g) * 0.3
    k = min(n, 8)
    pred[:k] = torch.tensor([0.5, -0.5, 1e3, -1e3, 0.25, 0.0, 5e4, 0.5 + 2 ** -23], device="cuda")[:k]
    target[:k] = 0
    for tgt in (target, torch.zeros(1, device="cuda") + 0.125):     # full, and a broadcast (expand_as) target
        p = pred.clone().requires_grad_(True)
        loss = ops.huber2(p, tgt)
        loss.backward()
        res = []
        for dt in (torch.float64, torch.float32):
            p_r = pred.to(dt, copy=True).requires_grad_(True)
            l_r = 2 * F.huber_loss(p_r, tgt.to(dt).expand_as(p_r), delta=0.5)
            l_r.backward()
            res.append((l_r, p_r.grad))
        (l64, g64), (l32, g32) = res
        _gate("n=%d loss" % n, loss, l64, l32, 64 * ULP)
        ek = ((p.grad.double() - g64).abs() / g64.abs().clamp_min(1e-300)).max().item()
        eo = ((g32.double() - g64).abs() / g64.abs().clamp_min(1e-300)).max().item()
        nz = g64 != 0
        assert torch.equal(p.grad[~nz], torch.zeros_like(p.grad[~nz]))
        assert ek <= C * eo + 4 * ULP, ("n=%d grad" % n, ek, eo)


def test_huber2_nan_inf_like_torch():
    """A NaN prediction gives a NaN loss and a NaN gradient entry (the optimiser's invalid-gradient check relies on it);
    +-inf give an infinite loss and a gradient of +-delta * norm, as torch does."""
    from sparf_b200 import ops
    for vals in ([float("nan"), 0.5, -0.5, 0.7, float("inf")], [0.2, float("inf"), -0.7, float("-inf"), 0.1],
                 [float("-inf"), float("nan"), 0.0]):
        pred = torch.tensor(vals, device="cuda")
        p = pred.clone().requires_grad_(True)
        loss = ops.huber2(p, torch.zeros_like(pred))
        loss.backward()
        p_r = pred.clone().requires_grad_(True)
        l_r = 2 * F.huber_loss(p_r, torch.zeros_like(pred), delta=0.5)
        l_r.backward()
        torch.testing.assert_close(loss, l_r, equal_nan=True)
        torch.testing.assert_close(p.grad, p_r.grad, equal_nan=True)
