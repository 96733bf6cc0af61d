"""The MLP engines and the density queries against fp64 arithmetic from their own fp32 encoding (tests/engine_oracle.py),
with bounds tight enough to see one operand of one GEMM lose its lo half.

The reference rounds x = o + t d, the band arguments and the unit direction as the encoders do, and runs everything
after in fp64; its gradients are taken at that point.  Samples with a ReLU pre-activation within MU * rms(layer) of 0
(the reference's, never an engine's) get zero upstream gradient, so a ReLU branch that rounding may flip feeds no
gradient; forward outputs are compared on every sample (a flip is continuous there).

Metric: max |x - ref| / max |ref| per tensor.  Gates: TAU_FWD on sigma, rgb, raw, feat; TAU_BWD on every parameter
gradient, the ray gradients (d_origins, d_dirs) and the point gradients (d_points, and density_gradient on the
unflagged points).  From the error model: the forward's 3-pass fp16 split leaves ~2^-22 per product and the backward's
3-pass bf16 split ~2^-17, plus sqrt(K) 2^-24 of fp32 accumulation.  simt_fp32 and tc_3x pass every gate; tc_3x_w1 the
forward and the ray / point gradients.  Controls: tc_1x's forward (one bf16 pass) and tc_3x_w1's trunk weight gradients
(one bf16 pass over the hi halves) must miss their gates by >= 10x, or the gates could not see a lost lo half (2^-9 ...
2^-11 on one operand's contribution).

Measured on an H100 80GB HBM3 (700 W power limit), worst error / gate over every case of this module:

    engine      forward   parameter grads   ray / point grads   (worst case)
    simt_fp32   0.27      0.03              0.02                fwd: rgb, 1023x128
    tc_3x       0.40      0.20              0.49                fwd: sigma, 5x13 c2f; grads: d_origins, 1x64
    tc_3x_w1    0.40      (not gated)       0.49                the same kernels as tc_3x there
    controls:   tc_1x forward >= 100x TAU_FWD; tc_3x_w1 worst trunk weight gradient >= 25x TAU_BWD

The forward's floor is fp32 itself, not the split: at 32k+ rows simt_fp32 is at 0.6e-6 ... 2.7e-6 and tc_3x at
1.1e-6 ... 3.7e-6 (fp32 activations between layers, fp32 sinf / cosf in the encoding), above the model's 2^-22 per
product.  The backward's 3-pass error, ~1e-5 (median 9e-6), is what the model gives.  The margin mask flags 3 ... 17 %
of the samples (~10 % at 64k+ rows).  Both non-default networks run on every engine (none refuses them).

Sensitivity to the error class itself: a build whose fused input-gradient chain packs trunk layer 3's weight at one
bf16 pass (its lo half zeroed) puts 1.2e-3 ... 2.2e-3 on d_origins, d_dirs and trunk layers 0-2's gradients (12 ... 22x
TAU_BWD) and fails every default-network gradient case here, while tests/test_tc_engine.py passes with it.

Runtime: the fp64 references run on the device; the module's 28 tests take ~15 s on that H100.
"""
import pytest
import torch

import engine_oracle as E

pytestmark = pytest.mark.gpu

TAU_FWD = 1e-5
TAU_BWD = 1e-4
MU = 2.0 ** -14          # margin of the ReLU mask, relative to the rms of a layer's pre-activations
FLAG_CAP = 0.25          # most samples the margin mask may drop
CONTROL = 10.0           # how far the single-pass controls must miss their gates
C2F, PROGRESS = (0.4, 0.7), 0.6     # at 0.6 one band of each encoding has a fractional weight

SPECS = {
    "default": dict(),
    # not the fused chain: the layer-by-layer tensor-core path, N and K not multiples of the tile
    "w136": dict(width=136, n_trunk=4, skip_layer=2, L_xyz=6, L_view=2, head_width=64),
    # the fused chain at its shortest, without a skip layer
    "w256_nt3": dict(width=256, n_trunk=3, skip_layer=-1, L_xyz=4, L_view=1),
}
PARITY = ("simt_fp32", "tc_3x")


def _err(x, ref):
    ref = ref.detach().double()
    return ((x.detach().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _engine(name):
    from sparf_b200 import _lib
    e = _lib.ENGINES[name]
    return e if _lib.lib().sparf_engine_available(e) else None


def _param_names(spec, head=True):
    names = sum([["trunk%d.w" % i, "trunk%d.b" % i] for i in range(spec.n_trunk)], [])
    return names + (["head0.w", "head0.b", "head1.w", "head1.b"] if head else [])


class _Table:
    """Prints one line per (case, engine, tensor) and collects the gates an engine misses."""

    def __init__(self, case):
        self.case, self.misses, self.worst = case, [], {}

    def row(self, eng, what, err, gate, must=True):
        ratio = err / gate
        print("%-34s %-9s %-10s err %.2e  gate %.0e  ratio %7.3f%s" % (self.case, eng, what, err, gate, ratio,
                                                                       "" if must else "  (not gated)"))
        if must:
            self.worst[eng] = max(self.worst.get(eng, 0.0), ratio)
            if not err <= gate:
                self.misses.append("%s %s %s: %.2e > %.0e" % (self.case, eng, what, err, gate))
        return ratio

    def fail(self, msg):
        print("%-34s %s" % (self.case, msg))
        self.misses.append("%s: %s" % (self.case, msg))

    def done(self):
        print("%-34s worst ratio per gated engine: %s" % (self.case, ", ".join("%s %.3f" % kv for kv in self.worst.items())))
        assert not self.misses, "\n".join(self.misses)


def _flagged(table, flag):
    frac = flag.float().mean().item()
    print("%-34s flagged %.2f%% of %d samples (margin 2^-14 rms)" % (table.case, 100 * frac, flag.numel()))
    assert frac < FLAG_CAP, (table.case, frac)


# ----------------------------------------------------------------------------------------------
# the MLP: ops.mlp_forward and its backward
# ----------------------------------------------------------------------------------------------
def _run_mlp(spec_name, R, S, *, seed, noise, c2f, mode):
    """mode: 'tape' (taped forward + backward), 'recompute' (ops.USE_TAPE off), 'no_grad' (inference forward)"""
    from sparf_b200 import ops
    spec = ops.MLPSpec(barf_c2f=C2F if c2f else None, **SPECS[spec_name])
    params = [p.cuda() for p in E.make_params(spec, seed)]
    o, d, t, nz = (x.cuda() for x in E.ray_inputs(R, S, seed))
    nz = nz if noise else None
    prog = torch.tensor(PROGRESS, device="cuda") if c2f else None
    grad = mode != "no_grad"
    case = "%s R=%d S=%d %s%s%s" % (spec_name, R, S, mode, " noise" if noise else "", " c2f" if c2f else "")
    table = _Table(case)
    names = ["d_origins", "d_dirs"] + _param_names(spec)

    p64 = [p.double().requires_grad_(grad) for p in params]
    o64, d64 = o.double().requires_grad_(grad), d.double().requires_grad_(grad)
    with torch.set_grad_enabled(grad):
        ref = E.mlp_reference(spec, p64, o64, d64, t.double(), noise=nz, progress=PROGRESS if c2f else None)
    flag = E.margin_mask(ref["pre"], MU)
    _flagged(table, flag)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    keep = (~flag).float()
    gs = torch.randn(R, S, device="cuda", generator=g) * keep
    gc = torch.randn(R, S, 3, device="cuda", generator=g) * keep[..., None]
    fwd_ref = dict(sigma=ref["sigma"].detach(), rgb=ref["rgb"].detach())
    truth = None
    if grad and not keep.any():
        print("%-34s every sample flagged: forward only" % case)
        grad = False
    if grad:
        ((ref["sigma"] * gs.double()).sum() + (ref["rgb"] * gc.double()).sum()).backward()
        truth = [o64.grad, d64.grad] + [p.grad for p in p64]
    del ref, p64

    for eng_name in ("simt_fp32", "tc_3x", "tc_3x_w1", "tc_1x"):
        eng = _engine(eng_name)
        if eng is None:
            print("%-34s %-9s not available on this device" % (case, eng_name))
            continue
        with_grad = grad and eng_name != "tc_1x"
        ops.USE_TAPE[0] = mode != "recompute"
        try:
            ps = [p.clone().requires_grad_(with_grad) for p in params]
            oo, dd = o.clone().requires_grad_(with_grad), d.clone().requires_grad_(with_grad)
            with torch.set_grad_enabled(with_grad):
                s, c = ops.mlp_forward(spec, oo, dd, t, ps, noise=nz, progress=prog, engine=eng)
                if with_grad:
                    ((s * gs).sum() + (c * gc).sum()).backward()
            torch.cuda.synchronize()
        except RuntimeError as e:
            if spec_name == "default":
                raise
            print("%-34s %-9s refused: %s" % (case, eng_name, e))
            continue
        finally:
            ops.USE_TAPE[0] = True
        parity = eng_name in PARITY
        e_fwd = max(table.row(eng_name, "sigma", _err(s, fwd_ref["sigma"]), TAU_FWD, eng_name != "tc_1x"),
                    table.row(eng_name, "rgb", _err(c, fwd_ref["rgb"]), TAU_FWD, eng_name != "tc_1x"))
        if eng_name == "tc_1x" and e_fwd < CONTROL:
            table.fail("control: tc_1x forward within %.1fx of the forward gate" % e_fwd)
        if not with_grad:
            continue
        got = [oo.grad, dd.grad] + [p.grad for p in ps]
        worst_trunk_w = 0.0
        for nm, x, ref_g in zip(names, got, truth):
            ratio = table.row(eng_name, nm, _err(x, ref_g), TAU_BWD, parity or nm.startswith("d_"))
            if nm.startswith("trunk") and nm.endswith(".w"):
                worst_trunk_w = max(worst_trunk_w, ratio)
        if eng_name == "tc_3x_w1" and worst_trunk_w < CONTROL:
            table.fail("control: tc_3x_w1 trunk weight gradients within %.1fx of the gradient gate" % worst_trunk_w)
    table.done()


# (rows R*S at the GEMM tile edges) and the chunk edges: one taped chunk holds 131 072 rows, a recompute chunk 32 768,
# an inference chunk 65 536
MLP_CASES = [
    ("default", 1, 1, dict(noise=False, c2f=False, mode="tape")),
    ("default", 7, 9, dict(noise=True, c2f=True, mode="tape")),        # 63
    ("default", 1, 64, dict(noise=True, c2f=False, mode="tape")),
    ("default", 5, 13, dict(noise=False, c2f=True, mode="tape")),      # 65
    ("default", 127, 1, dict(noise=True, c2f=True, mode="tape")),
    ("default", 3, 43, dict(noise=False, c2f=False, mode="tape")),     # 129
    ("default", 1023, 128, dict(noise=True, c2f=False, mode="tape")),      # one taped chunk
    ("default", 1025, 128, dict(noise=False, c2f=True, mode="tape")),      # two taped chunks
    ("default", 257, 128, dict(noise=True, c2f=True, mode="recompute")),   # two recompute chunks
    ("default", 513, 128, dict(noise=True, c2f=False, mode="no_grad")),    # two inference chunks
    ("w136", 129, 64, dict(noise=True, c2f=True, mode="tape")),
    ("w136", 65, 64, dict(noise=False, c2f=False, mode="recompute")),
    ("w256_nt3", 129, 64, dict(noise=True, c2f=True, mode="tape")),
    ("w256_nt3", 65, 64, dict(noise=False, c2f=False, mode="recompute")),
]


@pytest.mark.parametrize("spec_name,R,S,kw", MLP_CASES,
                         ids=["%s-%dx%d-%s" % (c[0], c[1], c[2], c[3]["mode"]) for c in MLP_CASES])
def test_mlp_engines_against_fp64_from_their_encoding(spec_name, R, S, kw):
    _run_mlp(spec_name, R, S, seed=R * 1000 + S, **kw)


# ----------------------------------------------------------------------------------------------
# density queries: ops.density_forward with its backward, ops.density_gradient
# ----------------------------------------------------------------------------------------------
def _run_density(spec_name, M, probe, *, seed, c2f):
    """probe: which outputs carry an upstream gradient -- 'raw+feat', 'raw' (features=False) or 'feat'"""
    from sparf_b200 import ops
    spec = ops.MLPSpec(barf_c2f=C2F if c2f else None, **SPECS[spec_name])
    params = [p.cuda() for p in E.make_params(spec, seed)[:2 * spec.n_trunk]]
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(M, 3, generator=g) * 3 - 1.5).cuda()
    prog = torch.tensor(PROGRESS, device="cuda") if c2f else None
    want_raw, want_feat = "raw" in probe, "feat" in probe
    table = _Table("%s density M=%d %s%s" % (spec_name, M, probe, " c2f" if c2f else ""))
    names = ["d_points"] + _param_names(spec, head=False)

    p64 = [p.double().requires_grad_(True) for p in params]
    x64 = pts.double().requires_grad_(True)
    ref = E.density_reference(spec, p64, x64, progress=PROGRESS if c2f else None)
    flag = E.margin_mask(ref["pre"], MU)
    _flagged(table, flag)
    gg = torch.Generator(device="cuda").manual_seed(seed + 1)
    keep = (~flag).float()
    a = torch.randn(M, device="cuda", generator=gg) * keep
    b = torch.randn(M, spec.width, device="cuda", generator=gg) * keep[:, None]
    grad_pts_raw = None
    if probe == "raw+feat":     # d raw.sum() / d points: density_gradient's truth, on the unflagged points
        grad_pts_raw = torch.autograd.grad(ref["raw"].sum(), x64, retain_graph=True)[0]
    loss = (ref["raw"] * a.double()).sum() if want_raw else 0.0
    if want_feat:
        loss = loss + (ref["feat"] * b.double()).sum()
    loss.backward()
    truth = [x64.grad] + [p.grad for p in p64]
    fwd_ref = dict(raw=ref["raw"].detach(), feat=ref["feat"].detach())
    del ref, p64

    for eng_name in ("simt_fp32", "tc_3x", "tc_3x_w1"):
        eng = _engine(eng_name)
        if eng is None:
            print("%-34s %-9s not available on this device" % (table.case, eng_name))
            continue
        try:
            ps = [p.clone().requires_grad_(True) for p in params]
            x = pts.clone().requires_grad_(True)
            raw, feat = ops.density_forward(spec, x, ps, progress=prog, engine=eng, features=want_feat)
            loss = (raw * a).sum() if want_raw else 0.0
            if want_feat:
                loss = loss + (feat * b).sum()
            loss.backward()
            dg = ops.density_gradient(spec, pts, params, progress=prog, engine=eng) if grad_pts_raw is not None else None
            torch.cuda.synchronize()
        except RuntimeError as e:
            if spec_name == "default":
                raise
            print("%-34s %-9s refused: %s" % (table.case, eng_name, e))
            continue
        parity = eng_name in PARITY
        table.row(eng_name, "raw", _err(raw, fwd_ref["raw"]), TAU_FWD)
        if want_feat:
            table.row(eng_name, "feat", _err(feat, fwd_ref["feat"]), TAU_FWD)
        got = [x.grad] + [p.grad for p in ps]
        worst_trunk_w = 0.0
        for nm, y, ref_g in zip(names, got, truth):
            ratio = table.row(eng_name, nm, _err(y, ref_g), TAU_BWD, parity or nm == "d_points")
            if nm.endswith(".w"):
                worst_trunk_w = max(worst_trunk_w, ratio)
        if eng_name == "tc_3x_w1" and worst_trunk_w < CONTROL:
            table.fail("control: tc_3x_w1 trunk weight gradients within %.1fx of the gradient gate" % worst_trunk_w)
        if dg is not None:
            table.row(eng_name, "gradient", _err(dg[~flag], grad_pts_raw[~flag]), TAU_BWD)
    table.done()


# one point; a partial row tile; three backward chunks of 32 768 (the last of 5 points); two forward chunks of 65 536
DENSITY_M = [(1, False), (65, True), (2 * 32768 + 5, False), (65536 + 333, True)]


@pytest.mark.parametrize("probe", ["raw+feat", "raw", "feat"])
@pytest.mark.parametrize("M,c2f", DENSITY_M, ids=["M%d" % m for m, _ in DENSITY_M])
def test_density_engines_against_fp64_from_their_encoding(M, c2f, probe):
    _run_density("default", M, probe, seed=M % 997 + 11, c2f=c2f)


@pytest.mark.parametrize("spec_name", ["w136", "w256_nt3"])
def test_density_non_default_networks(spec_name):
    _run_density(spec_name, 4097, "raw+feat", seed=29, c2f=True)
