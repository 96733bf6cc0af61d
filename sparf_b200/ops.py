"""torch.autograd adapters over the C ABI (include/sparf_b200.h).

PyTorch is plumbing here: it owns device memory, the stream and the autograd tape; every number is
produced by the kernels in csrc/.  All functions take / return fp32 CUDA tensors and raise if the
native library is unavailable (no fallback).
"""
from __future__ import annotations

import ctypes
import numbers
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import SparfMLP, SparfMLPGrad, check

_ENGINE = [_lib.ENGINE_AUTO]
# keep the training forward's activations for the backward when offered (sparf_mlp_tape_bytes > 0); False = always recompute
USE_TAPE = [True]
# Opt-in: let the MLP backward accumulate straight into existing `param.grad` storage (the C ABI accumulates, +=)
# instead of returning fresh gradient tensors for autograd to add.  Saves ~20 tiny kernels and a 2 MB memset per
# render pass.  Only valid for plain `loss.backward()` training loops (no torch.autograd.grad / grad hooks / DDP
# hooks on these parameters).  Per parameter set: sparf_b200.distributed.FlatGradients marks its parameters
# (`p._sparf_inplace_grad`); the global switch forces it for every model of the process.
ACCUMULATE_INTO_PARAM_GRAD = [False]

# optional device-side timing of the MLP kernels (bench.py roofline): CUDA events on the launching stream
PROFILE_ON = [False]
PROFILE = []
# MLP sample-evaluations issued through this module (forward calls, backward calls): bench.py's FLOP accounting
EVALS = {"fwd": 0, "bwd": 0}


class _timed:
    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        if PROFILE_ON[0]:
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if PROFILE_ON[0]:
            self.e1.record()
            PROFILE.append((self.tag, self.e0, self.e1))


def profile_total_ms(tag_prefix="mlp"):
    """Sum of the recorded intervals (call after torch.cuda.synchronize())."""
    torch.cuda.synchronize()
    return sum(e0.elapsed_time(e1) for tag, e0, e1 in PROFILE if tag.startswith(tag_prefix))


def set_engine(name_or_id) -> None:
    """Select the MLP engine: 'auto' | 'simt_fp32' | 'tc_3x' | 'tc_1x'."""
    _ENGINE[0] = _lib.ENGINES[name_or_id] if isinstance(name_or_id, str) else int(name_or_id)


def get_engine() -> int:
    return _ENGINE[0]


def _stream() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_tensor_device(fn):
    """Run an op body with the CUDA device of its first tensor argument current: the kernels launch on the current
    device's current stream, so a Graph on cuda:1 works without a global torch.cuda.set_device (one process driving
    several devices)."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        dev = None
        for a in args:
            if torch.is_tensor(a) and a.is_cuda:
                dev = a.device
                break
            saved = getattr(a, "saved_tensors", None) if not torch.is_tensor(a) and hasattr(a, "needs_input_grad") else None
            if saved:
                cand = [t for t in saved if torch.is_tensor(t) and t.is_cuda]
                if cand:
                    dev = cand[0].device
                    break
        if dev is None:
            for a in kwargs.values():
                if torch.is_tensor(a) and a.is_cuda:
                    dev = a.device
                    break
        if dev is None and kwargs.get("device") is not None:
            dev = torch.device(kwargs["device"])
        if dev is None or (torch.cuda.current_device() == (dev.index if dev.index is not None else torch.cuda.current_device())):
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapper


def _ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _row_ptr(t: torch.Tensor, i: int) -> ctypes.c_void_p:
    """a pointer to element i of a contiguous tensor (a device address; nothing is read)"""
    return ctypes.c_void_p(t.data_ptr() + i * t.element_size())


def _f32c(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda, "sparf_b200 ops need CUDA tensors (there is no CPU path)"
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
# MLP description
# ------------------------------------------------------------------------------------------------
class MLPSpec:
    """Static description of one NeRF network (shapes + c2f schedule), independent of the tensors."""

    def __init__(self, n_trunk=8, width=256, head_width=128, skip_layer=4, L_xyz=10, L_view=4, barf_c2f=None):
        self.n_trunk, self.width, self.head_width, self.skip_layer = n_trunk, width, head_width, skip_layer
        self.L_xyz, self.L_view = L_xyz, L_view
        self.barf_c2f = tuple(barf_c2f) if barf_c2f is not None else None

    def n_params(self) -> int:
        return 2 * self.n_trunk + 4

    def fill(self, params: Sequence[torch.Tensor], progress: Optional[torch.Tensor]) -> Tuple[SparfMLP, list]:
        """params = [trunk_w0, trunk_b0, ..., head_w0, head_b0, head_w1, head_b1] (nn.Linear tensors); the trunk's 2 n_trunk
        alone leave the head pointers NULL (density calls)."""
        keep = [_f32c(p.detach()) for p in params]
        m = SparfMLP()
        m.n_trunk, m.width, m.head_width, m.skip_layer = self.n_trunk, self.width, self.head_width, self.skip_layer
        m.L_xyz, m.L_view = self.L_xyz, self.L_view
        m.use_c2f = 1 if self.barf_c2f is not None else 0
        if self.barf_c2f is not None:
            start, end = self.barf_c2f
            m.c2f_start = float(start)
            m.c2f_range = float(end - start)  # python-double subtraction, like the reference
            assert progress is not None
            prog = _f32c(progress.detach()).reshape(1)
            keep.append(prog)
            m.progress = prog.data_ptr()
        else:
            m.progress = 0
        for i in range(self.n_trunk):
            m.trunk_w[i] = keep[2 * i].data_ptr()
            m.trunk_b[i] = keep[2 * i + 1].data_ptr()
        o = 2 * self.n_trunk
        if len(params) > o:
            m.head_w[0], m.head_b[0] = keep[o].data_ptr(), keep[o + 1].data_ptr()
            m.head_w[1], m.head_b[1] = keep[o + 2].data_ptr(), keep[o + 3].data_ptr()
        return m, keep

    def grad_struct(self, grads: Sequence[torch.Tensor]) -> SparfMLPGrad:
        g = SparfMLPGrad()
        for i in range(self.n_trunk):
            g.trunk_w[i] = grads[2 * i].data_ptr()
            g.trunk_b[i] = grads[2 * i + 1].data_ptr()
        o = 2 * self.n_trunk
        if len(grads) > o:
            g.head_w[0], g.head_b[0] = grads[o].data_ptr(), grads[o + 1].data_ptr()
            g.head_w[1], g.head_b[1] = grads[o + 2].data_ptr(), grads[o + 3].data_ptr()
        return g


_WS = {}
_WS_RETIRED = []   # outgrown buffers stay alive: a captured CUDA graph may have their addresses baked into its kernels


def _workspace(nbytes: int, device) -> torch.Tensor:
    """Grow-only per-(device, stream) scratch buffer.  Reuse is stream-ordered, so one buffer per stream is safe; a
    buffer that is outgrown is retired, never freed (CUDA graphs captured earlier keep replaying into it)."""
    dev = device.index if device.index is not None else torch.cuda.current_device()
    key = (dev, torch.cuda.current_stream(dev).cuda_stream)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _WS_RETIRED.append(buf)
            nbytes = max(nbytes, int(1.5 * buf.numel()))   # geometric growth bounds the retired bytes
        buf = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
        _WS[key] = buf
    return buf


def _inplace_refs(params):
    """The parameters whose `.grad` a backward may accumulate into (ACCUMULATE_INTO_PARAM_GRAD, or every parameter of
    the call marked `_sparf_inplace_grad`), else None."""
    if ACCUMULATE_INTO_PARAM_GRAD[0] or all(getattr(p, "_sparf_inplace_grad", False) for p in params):
        return params
    return None


def _grad_targets(ctx, params, device):
    """A backward's view of the network and the destinations of its parameter gradients -> (SparfMLP, the tensors it
    points at, SparfMLPGrad, parameter gradients to return).  The destinations are the parameters' own `.grad` when the
    forward opted in (ctx.param_refs) and every one exists (autograd then gets None), else fresh zeroed tensors in one
    flat buffer."""
    m, keep = ctx.spec.fill(params, ctx.progress)
    refs = ctx.param_refs
    if refs is not None and all(p.grad is not None and p.grad.is_contiguous() and p.grad.dtype == torch.float32 for p in refs):
        grads, ret = [p.grad for p in refs], [None] * len(params)
    else:
        sizes = [p.numel() for p in params]
        flat = torch.zeros(sum(sizes), device=device, dtype=torch.float32)
        grads, o = [], 0
        for p, n in zip(params, sizes):
            grads.append(flat[o:o + n].view(p.shape))
            o += n
        ret = grads
    return m, keep, ctx.spec.grad_struct(grads), ret


# ------------------------------------------------------------------------------------------------
# MLP: sigma, rgb = NeRF.forward_samples(o, d, t)
# ------------------------------------------------------------------------------------------------
# The MLP functions' arguments: (spec, engine, how, origins, dirs, t, noise, progress, *params), where `how` is what
# differs by pass: grad_mode (dense), grid (grid) or (grid, tau_max, window) (terminated).
_ORIGINS, _DIRS, _PARAMS = 3, 4, 8


def _mlp_grads(d_o, d_d, param_grads):
    """A backward's return value in the MLP functions' argument layout."""
    ret = [None] * _PARAMS + list(param_grads)
    ret[_ORIGINS], ret[_DIRS] = d_o, d_d
    return tuple(ret)


class MLPFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, spec: MLPSpec, engine: int, grad_mode: bool, origins, dirs, t, noise, progress, *params):
        L = _lib.lib()
        origins, dirs, t = _f32c(origins), _f32c(dirs), _f32c(t)
        R, S = t.shape
        assert origins.shape == (R, 3) and dirs.shape == (R, 3)
        noise_c = _f32c(noise) if noise is not None else None
        m, keep = spec.fill(params, progress)
        sigma = torch.empty(R, S, device=t.device, dtype=torch.float32)
        rgb = torch.empty(R, S, 3, device=t.device, dtype=torch.float32)
        nbytes = L.sparf_mlp_workspace_bytes(ctypes.byref(m), R, S, 0, engine)
        ws = _workspace(nbytes, t.device)
        # Training forward: when a gradient will be asked for and the engine offers it, keep a "tape" (the
        # fp32 encodings and activations) so that the backward skips the forward recompute.
        # (grad_mode: autograd is recording at the call site -- under torch.no_grad() nothing is kept)
        EVALS["fwd"] += R * S
        needs = ctx.needs_input_grad
        wants_grad = grad_mode and (needs[_ORIGINS] or needs[_DIRS] or any(needs[_PARAMS:]))
        tape_bytes = L.sparf_mlp_tape_bytes(ctypes.byref(m), engine, R, S) if (wants_grad and USE_TAPE[0]) else 0
        ctx.tape = None
        with _timed("mlp_forward"):
            if tape_bytes:
                ctx.tape = torch.empty(tape_bytes, dtype=torch.uint8, device=t.device)
                check(L.sparf_mlp_forward_tape(ctypes.byref(m), engine, R, S, _ptr(origins), _ptr(dirs), _ptr(t),
                                               _ptr(noise_c), _ptr(sigma), _ptr(rgb), _ptr(ctx.tape), tape_bytes, _ptr(ws),
                                               ws.numel(), _stream()), "mlp_forward_tape")
            else:
                check(L.sparf_mlp_forward(ctypes.byref(m), engine, R, S, _ptr(origins), _ptr(dirs), _ptr(t), _ptr(noise_c),
                                          _ptr(sigma), _ptr(rgb), _ptr(ws), ws.numel(), _stream()), "mlp_forward")
        ctx.spec, ctx.engine = spec, engine
        ctx.noise = noise_c
        ctx.progress = progress
        ctx.param_refs = _inplace_refs(params)
        if ctx.tape is not None:
            ctx.save_for_backward(origins, dirs, t, sigma, rgb, *params)
        else:
            ctx.save_for_backward(origins, dirs, t, *params)
        return sigma, rgb

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g_sigma, g_rgb):
        L = _lib.lib()
        if ctx.tape is not None:
            origins, dirs, t, sigma_f, rgb_f, *params = ctx.saved_tensors
        else:
            origins, dirs, t, *params = ctx.saved_tensors
        R, S = t.shape
        EVALS["bwd"] += R * S
        g_sigma = _f32c(g_sigma) if g_sigma is not None else torch.zeros(R, S, device=t.device)
        g_rgb = _f32c(g_rgb) if g_rgb is not None else torch.zeros(R, S, 3, device=t.device)
        m, keep, gs, ret = _grad_targets(ctx, params, t.device)
        need_o, need_d = ctx.needs_input_grad[_ORIGINS], ctx.needs_input_grad[_DIRS]
        d_o = torch.zeros_like(origins) if (need_o or need_d) else None
        d_d = torch.zeros_like(dirs) if (need_o or need_d) else None
        nbytes = L.sparf_mlp_workspace_bytes(ctypes.byref(m), R, S, 2 if ctx.tape is not None else 1, ctx.engine)
        ws = _workspace(nbytes, t.device)
        with _timed("mlp_backward"):
            if ctx.tape is not None:
                check(L.sparf_mlp_backward_tape(ctypes.byref(m), ctx.engine, R, S, _ptr(origins), _ptr(dirs), _ptr(t),
                                                _ptr(sigma_f), _ptr(rgb_f), _ptr(g_sigma), _ptr(g_rgb), ctypes.byref(gs),
                                                _ptr(d_o), _ptr(d_d), _ptr(ctx.tape), ctx.tape.numel(), _ptr(ws), ws.numel(),
                                                _stream()), "mlp_backward_tape")
                ctx.tape = None
            else:
                check(L.sparf_mlp_backward(ctypes.byref(m), ctx.engine, R, S, _ptr(origins), _ptr(dirs), _ptr(t),
                                           _ptr(ctx.noise), _ptr(g_sigma), _ptr(g_rgb), ctypes.byref(gs), _ptr(d_o),
                                           _ptr(d_d), _ptr(ws), ws.numel(), _stream()), "mlp_backward")
        return _mlp_grads(d_o if need_o else None, d_d if need_d else None, ret)


def mlp_forward(spec: MLPSpec, origins, dirs, t, params: Sequence[torch.Tensor], *, noise=None, progress=None,
                engine: Optional[int] = None):
    """origins/dirs [R,3], t [R,S] -> (sigma [R,S], rgb [R,S,3]); differentiable w.r.t. origins, dirs, params."""
    eng = get_engine() if engine is None else engine
    return MLPFunction.apply(spec, eng, torch.is_grad_enabled(), origins, dirs, t, noise, progress, *params)


def _grid_compact(grid, o, d, t, K, idx, o_k, d_k, t_k):
    """The samples of o, d [R,3], t [R,S] that `grid` (occupancy.OccupancyGrid, box or contracted) keeps, into the
    capacity-R*S buffers idx, o_k, d_k, t_k; their count into the device scalar K.  The host never reads K."""
    L = _lib.lib()
    R, S = t.shape
    if grid.contraction is None:
        ws = _workspace(L.sparf_occupancy_workspace_bytes(R, S), t.device)
        args = (R, S, _ptr(o), _ptr(d), _ptr(t), _ptr(grid.bits), int(grid.res), float(grid.range[0]), float(grid.range[1]))
        check(L.sparf_occupancy_count(*args, _ptr(K), _ptr(ws), ws.numel(), _stream()), "occupancy_count")
        check(L.sparf_occupancy_emit(*args, _ptr(idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(), _stream()),
              "occupancy_emit")
    else:
        center, radius = grid.contraction
        c = (ctypes.c_float * 3)(*center)
        ws = _workspace(L.sparf_termination_workspace_bytes(R, S), t.device)
        args = (R, S, 0, S, _ptr(o), _ptr(d), _ptr(t), None, _ptr(grid.bits), int(grid.res), c, float(radius))
        check(L.sparf_contracted_count(*args, _ptr(K), _ptr(ws), ws.numel(), _stream()), "contracted_count")
        check(L.sparf_contracted_emit(*args, _ptr(idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(), _stream()),
              "contracted_emit")


class _CompactedMLPFunction(torch.autograd.Function):
    """The backward of the passes over a compacted sample set (grid, terminated): the output gradients gathered at the
    kept rows, one taped backward over them and the per-ray sums of the origin and direction gradients, every row count
    read on the device.  The forward sets ctx.C = R*S and, unless C = 0, saves (count, idx, o_k, d_k, t_k, sigma_k,
    rgb_k, *params) and sets ctx.shape, ctx.tape, ctx.rows_at (the kept-row count is count[rows_at]) and
    ctx.ray_sum(count, idx, src, dst), the ray sum of its layout."""

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g_sigma, g_rgb):
        if ctx.C == 0 or ctx.tape is None:
            return _mlp_grads(None, None, [None] * (len(ctx.needs_input_grad) - _PARAMS))
        L = _lib.lib()
        count, idx, o_k, d_k, t_k, sigma_k, rgb_k, *params = ctx.saved_tensors
        (R, S), C, dev = ctx.shape, ctx.C, t_k.device
        rows = _row_ptr(count, ctx.rows_at)
        g_sigma_k, g_rgb_k = torch.empty(C, 1, device=dev), torch.empty(C, 1, 3, device=dev)
        check(L.sparf_compact_gather(C, rows, _ptr(idx), 1, _ptr(_f32c(g_sigma)), _ptr(g_sigma_k), _stream()), "compact_gather")
        check(L.sparf_compact_gather(C, rows, _ptr(idx), 3, _ptr(_f32c(g_rgb)), _ptr(g_rgb_k), _stream()), "compact_gather")
        m, keep, gs, ret = _grad_targets(ctx, params, dev)
        need_o, need_d = ctx.needs_input_grad[_ORIGINS], ctx.needs_input_grad[_DIRS]
        d_o_k = torch.zeros(C, 3, device=dev) if (need_o or need_d) else None
        d_d_k = torch.zeros(C, 3, device=dev) if (need_o or need_d) else None
        ws = _workspace(L.sparf_mlp_workspace_bytes(ctypes.byref(m), C, 1, 2, ctx.engine), dev)
        with _timed("mlp_backward"):
            check(L.sparf_mlp_backward_tape_rows(ctypes.byref(m), ctx.engine, C, 1, rows, _ptr(o_k), _ptr(d_k), _ptr(t_k),
                                                 _ptr(sigma_k), _ptr(rgb_k), _ptr(g_sigma_k), _ptr(g_rgb_k), ctypes.byref(gs),
                                                 _ptr(d_o_k), _ptr(d_d_k), _ptr(ctx.tape), ctx.tape.numel(), _ptr(ws),
                                                 ws.numel(), _stream()), "mlp_backward_tape_rows")
        ctx.tape = None
        d_o = d_d = None
        if need_o:
            d_o = torch.empty(R, 3, device=dev)
            ctx.ray_sum(count, idx, d_o_k, d_o)
        if need_d:
            d_d = torch.empty(R, 3, device=dev)
            ctx.ray_sum(count, idx, d_d_k, d_d)
        return _mlp_grads(d_o, d_d, ret)


class GridMLPFunction(_CompactedMLPFunction):
    """mlp_forward over the samples an occupancy grid keeps, with gradients and without a host round trip: the
    compaction writes the kept count K to device memory, the taped MLP pair with a device row count evaluates the K
    kept samples out of a capacity of R*S, and scatter / gather / ray-sum kernels move rows between the dense and the
    compacted layouts, all reading K on the device.  So the op is capturable into a CUDA graph."""

    @staticmethod
    @_on_tensor_device
    def forward(ctx, spec: MLPSpec, engine: int, grid, origins, dirs, t, noise, progress, *params):
        L = _lib.lib()
        o, d, tt = _f32c(origins), _f32c(dirs), _f32c(t)
        R, S = tt.shape
        assert o.shape == (R, 3) and d.shape == (R, 3)
        C, dev = R * S, tt.device
        sigma = torch.zeros(R, S, device=dev)
        rgb = torch.zeros(R, S, 3, device=dev)
        ctx.C = C
        if C == 0:
            return sigma, rgb
        K = torch.empty((), dtype=torch.int64, device=dev)
        idx = torch.empty(C, dtype=torch.int64, device=dev)
        o_k, d_k, t_k = torch.empty(C, 3, device=dev), torch.empty(C, 3, device=dev), torch.empty(C, 1, device=dev)
        _grid_compact(grid, o, d, tt, K, idx, o_k, d_k, t_k)
        noise_k = None
        if noise is not None:         # drawn dense by the caller (the RNG stream of the dense pass), taken at the kept samples
            noise_k = torch.empty(C, 1, device=dev)
            check(L.sparf_compact_gather(C, _ptr(K), _ptr(idx), 1, _ptr(_f32c(noise)), _ptr(noise_k), _stream()),
                  "compact_gather")
        m, keep = spec.fill(params, progress)
        tape_bytes = L.sparf_mlp_tape_bytes(ctypes.byref(m), engine, C, 1)
        if not tape_bytes:
            raise RuntimeError("mlp_forward_grid: no tape for %d samples (a tape above 16 GB); use smaller batches" % C)
        tape = torch.empty(tape_bytes, dtype=torch.uint8, device=dev)
        ws = _workspace(L.sparf_mlp_workspace_bytes(ctypes.byref(m), C, 1, 0, engine), dev)
        sigma_k, rgb_k = torch.empty(C, 1, device=dev), torch.empty(C, 1, 3, device=dev)
        with _timed("mlp_forward"):
            check(L.sparf_mlp_forward_tape_rows(ctypes.byref(m), engine, C, 1, _ptr(K), _ptr(o_k), _ptr(d_k), _ptr(t_k),
                                                _ptr(noise_k), _ptr(sigma_k), _ptr(rgb_k), _ptr(tape), tape_bytes, _ptr(ws),
                                                ws.numel(), _stream()), "mlp_forward_tape_rows")
        check(L.sparf_compact_scatter(C, _ptr(K), _ptr(idx), 1, _ptr(sigma_k), _ptr(sigma), _stream()), "compact_scatter")
        check(L.sparf_compact_scatter(C, _ptr(K), _ptr(idx), 3, _ptr(rgb_k), _ptr(rgb), _stream()), "compact_scatter")
        ctx.spec, ctx.engine, ctx.progress, ctx.tape = spec, engine, progress, tape
        ctx.shape, ctx.rows_at = (R, S), 0
        ctx.ray_sum = lambda K_, idx_, src, dst: check(
            L.sparf_compact_ray_sum(R, S, C, _ptr(K_), _ptr(idx_), 3, _ptr(src), _ptr(dst), _stream()), "compact_ray_sum")
        ctx.param_refs = _inplace_refs(params)
        ctx.save_for_backward(K, idx, o_k, d_k, t_k, sigma_k, rgb_k, *params)
        return sigma, rgb


def mlp_forward_grid(spec: MLPSpec, origins, dirs, t, grid, params: Sequence[torch.Tensor], *, noise=None, progress=None,
                     engine: Optional[int] = None):
    """mlp_forward (origins/dirs [R,3], t [R,S] -> sigma [R,S], rgb [R,S,3]) with the samples that `grid`
    (occupancy.OccupancyGrid, box or contracted) skips set to sigma = 0, rgb = 0 and given no gradient.  The kept
    samples are evaluated exactly as mlp_forward evaluates them, and the call never synchronises with the host, so a
    training step that uses it can be captured into a CUDA graph.  noise [R,S] (density noise) is drawn dense by the
    caller and applied at the kept samples.  Differentiable w.r.t. origins, dirs, params; tensor-core engines only.
    (K stays on the device: EVALS does not count these passes.)"""
    eng = get_engine() if engine is None else engine
    if eng == _lib.ENGINE_SIMT_FP32:
        raise ValueError("mlp_forward_grid: the simt_fp32 engine has no device-side row count; use tc_3x, tc_1x or tc_3x_w1")
    return GridMLPFunction.apply(spec, eng, grid, origins, dirs, t, noise, progress, *params)


def _window_append(grid, o, d, t, k0, k1, alive, ends, w, idx, o_k, d_k, t_k):
    """Window w = samples [k0, k1) of the alive rays of o, d [R,3], t [R,S] that `grid` (box, contracted or None) keeps,
    appended to rows [ends[w], ends[w+1]) of the capacity-R*S buffers idx, o_k, d_k, t_k; ends[w+1] is written on the
    device.  The host never reads it."""
    L = _lib.lib()
    R, S = t.shape
    ws = _workspace(L.sparf_termination_workspace_bytes(R, k1 - k0), t.device)
    head = (R, S, int(k0), int(k1), _ptr(o), _ptr(d), _ptr(t), _ptr(alive))
    tail = (_ptr(ends), int(w), _ptr(idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(), _stream())
    if grid is not None and grid.contraction is not None:
        center, radius = grid.contraction
        c = (ctypes.c_float * 3)(*center)
        check(L.sparf_contracted_append(*head, _ptr(grid.bits), int(grid.res), c, float(radius), *tail), "contracted_append")
    elif grid is not None:
        check(L.sparf_termination_append(*head, _ptr(grid.bits), int(grid.res), float(grid.range[0]), float(grid.range[1]),
                                         *tail), "termination_append")
    else:
        check(L.sparf_termination_append(*head, None, 0, 0.0, 1.0, *tail), "termination_append")


class TerminatedMLPFunction(_CompactedMLPFunction):
    """mlp_forward with early ray termination in windows, on top of an optional occupancy grid, with gradients and
    without a host round trip.  Each window appends its kept samples (alive rays, grid-kept samples) to one compacted
    set per pass, rows [ends[w], ends[w+1]), and runs the taped forward over that device-side span into one tape; the
    backward is one taped backward over rows [0, ends[W]).  Only W = ceil(S / window) is known on the host, so the op
    is capturable into a CUDA graph."""

    @staticmethod
    @_on_tensor_device
    def forward(ctx, spec: MLPSpec, engine: int, how, origins, dirs, t, noise, progress, *params):
        L = _lib.lib()
        grid, tau_max, window = how
        o, d, tt = _f32c(origins), _f32c(dirs), _f32c(t)
        R, S = tt.shape
        assert o.shape == (R, 3) and d.shape == (R, 3)
        C, dev = R * S, tt.device
        ctx.C = C
        m, keep = spec.fill(params, progress)
        tape_bytes = L.sparf_mlp_tape_bytes(ctypes.byref(m), engine, C, 1) if C else 0
        if C and not tape_bytes:
            raise RuntimeError("mlp_forward_terminated: no tape for %d samples (a tape above 16 GB); use smaller batches" % C)
        sigma = torch.zeros(R, S, device=dev)
        rgb = torch.zeros(R, S, 3, device=dev)
        if C == 0:
            return sigma, rgb
        W = -(-S // window)
        cap = R * min(window, S)
        ends = torch.zeros(W + 1, dtype=torch.int64, device=dev)
        alive = torch.ones(R, dtype=torch.uint8, device=dev)
        tau = torch.zeros(R, device=dev)
        idx = torch.empty(C, dtype=torch.int64, device=dev)
        o_k, d_k, t_k = torch.empty(C, 3, device=dev), torch.empty(C, 3, device=dev), torch.empty(C, 1, device=dev)
        noise_c = _f32c(noise) if noise is not None else None     # drawn dense by the caller, taken at the kept samples
        noise_k = torch.empty(C, 1, device=dev) if noise is not None else None
        sigma_k, rgb_k = torch.empty(C, 1, device=dev), torch.empty(C, 1, 3, device=dev)
        tape = torch.empty(tape_bytes, dtype=torch.uint8, device=dev)
        for w in range(W):
            k0, k1 = w * window, min((w + 1) * window, S)
            cw = R * (k1 - k0)
            _window_append(grid, o, d, tt, k0, k1, alive, ends, w, idx, o_k, d_k, t_k)
            if noise is not None:
                check(L.sparf_compact_gather_span(cw, _ptr(ends), w, _ptr(idx), 1, _ptr(noise_c), _ptr(noise_k), _stream()),
                      "compact_gather_span")
            ws = _workspace(L.sparf_mlp_workspace_bytes(ctypes.byref(m), cap, 1, 0, engine), dev)
            with _timed("mlp_forward"):
                check(L.sparf_mlp_forward_tape_span(ctypes.byref(m), engine, C, cw, _row_ptr(ends, w), _row_ptr(ends, w + 1),
                                                    _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(noise_k), _ptr(sigma_k), _ptr(rgb_k),
                                                    _ptr(tape), tape_bytes, _ptr(ws), ws.numel(), _stream()),
                      "mlp_forward_tape_span")
            check(L.sparf_compact_scatter_span(cw, _ptr(ends), w, _ptr(idx), 1, _ptr(sigma_k), _ptr(sigma), _stream()),
                  "compact_scatter_span")
            check(L.sparf_compact_scatter_span(cw, _ptr(ends), w, _ptr(idx), 3, _ptr(rgb_k), _ptr(rgb), _stream()),
                  "compact_scatter_span")
            if k1 < S:
                check(L.sparf_termination_update(R, S, k0, k1, _ptr(sigma), _ptr(tt), _ptr(d), float(tau_max), _ptr(tau),
                                                 _ptr(alive), _stream()), "termination_update")
        ctx.spec, ctx.engine, ctx.progress, ctx.tape = spec, engine, progress, tape
        ctx.shape, ctx.rows_at = (R, S), W          # every window's rows: [0, ends[W])
        ctx.ray_sum = lambda ends_, idx_, src, dst: check(
            L.sparf_compact_ray_sum_segments(R, S, W, _ptr(ends_), _ptr(idx_), 3, _ptr(src), _ptr(dst), _stream()),
            "compact_ray_sum_segments")
        ctx.param_refs = _inplace_refs(params)
        ctx.save_for_backward(ends, idx, o_k, d_k, t_k, sigma_k, rgb_k, *params)
        return sigma, rgb


def mlp_forward_terminated(spec: MLPSpec, origins, dirs, t, grid, eps: float, window: int, params: Sequence[torch.Tensor], *,
                           noise=None, progress=None, engine: Optional[int] = None):
    """mlp_forward (origins/dirs [R,3], t [R,S] -> sigma [R,S], rgb [R,S,3]) with early ray termination: the samples of
    [k0, k0 + window) are evaluated for the rays still alive, and a ray dies once its optical depth exceeds fp32(-ln eps)
    (the rule of the inference termination, termination.forward_samples, on this pass's own sigma, density noise
    included); with `grid` (occupancy.OccupancyGrid, box or contracted; or None) only the samples it keeps are evaluated.
    Every other sample gets sigma = 0, rgb = 0 and no gradient; the kept ones the bits of mlp_forward.  noise [R,S] is
    drawn dense by the caller.  The call never synchronises with the host, so a training step that uses it can be
    captured into a CUDA graph.  Differentiable w.r.t. origins, dirs, params; tensor-core engines only."""
    eng = get_engine() if engine is None else engine
    if eng == _lib.ENGINE_SIMT_FP32:
        raise ValueError("mlp_forward_terminated: the simt_fp32 engine has no device-side row count; use tc_3x, tc_1x or "
                         "tc_3x_w1")
    if not (0 <= eps < 1) or int(window) != window or window < 1:
        raise ValueError("mlp_forward_terminated: eps %r (0 <= eps < 1), window %r (an integer >= 1)" % (eps, window))
    from .termination import tau_max
    return TerminatedMLPFunction.apply(spec, eng, (grid, tau_max(eps), int(window)), origins, dirs, t, noise, progress,
                                       *params)


# ------------------------------------------------------------------------------------------------
# density queries: raw, feat = NeRF.compute_raw_density(points)
# ------------------------------------------------------------------------------------------------
class DensityFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, spec: MLPSpec, engine: int, grad_mode: bool, features: bool, points, progress, *trunk_params):
        L = _lib.lib()
        pts = _f32c(points).reshape(-1, 3)
        M = pts.shape[0]
        m, keep = spec.fill(trunk_params, progress)
        raw = torch.empty(M, device=pts.device, dtype=torch.float32)
        feat = torch.empty(M, spec.width, device=pts.device, dtype=torch.float32) if features else None
        ws = _workspace(L.sparf_density_workspace_bytes(ctypes.byref(m), M, 0, engine), pts.device)
        EVALS["fwd"] += M
        with _timed("density_forward"):
            check(L.sparf_density_forward(ctypes.byref(m), engine, M, _ptr(pts), _ptr(raw), _ptr(feat), _ptr(ws), ws.numel(),
                                          _stream()), "density_forward")
        ctx.set_materialize_grads(False)     # an output nobody differentiated arrives as None and goes to the ABI as NULL
        ctx.spec, ctx.engine, ctx.progress = spec, engine, progress
        ctx.points_shape = points.shape
        ctx.saved = grad_mode and (ctx.needs_input_grad[4] or any(ctx.needs_input_grad[6:]))
        if ctx.saved:
            ctx.param_refs = _inplace_refs(trunk_params)
            ctx.save_for_backward(pts, *trunk_params)
        return raw, feat

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g_raw, g_feat):
        if not ctx.saved or (g_raw is None and g_feat is None):    # (only `progress` asked for a gradient)
            return (None,) * (6 + 2 * ctx.spec.n_trunk)
        L = _lib.lib()
        pts, *params = ctx.saved_tensors
        M = pts.shape[0]
        EVALS["bwd"] += M
        g_raw = _f32c(g_raw) if g_raw is not None else None
        g_feat = _f32c(g_feat) if g_feat is not None else None
        m, keep, gs, ret = _grad_targets(ctx, params, pts.device)
        d_pts = torch.zeros_like(pts) if ctx.needs_input_grad[4] else None
        ws = _workspace(L.sparf_density_workspace_bytes(ctypes.byref(m), M, 1, ctx.engine), pts.device)
        with _timed("density_backward"):
            check(L.sparf_density_backward(ctypes.byref(m), ctx.engine, M, _ptr(pts), _ptr(g_raw), _ptr(g_feat), ctypes.byref(gs),
                                           _ptr(d_pts), _ptr(ws), ws.numel(), _stream()), "density_backward")
        d_pts = d_pts.view(ctx.points_shape) if d_pts is not None else None
        ret = [g if need else None for g, need in zip(ret, ctx.needs_input_grad[6:])]
        return (None, None, None, None, d_pts, None, *ret)


def density_forward(spec: MLPSpec, points, trunk_params: Sequence[torch.Tensor], progress=None, engine: Optional[int] = None,
                    features: bool = True):
    """The trunk alone at points [..., 3] (NeRF.compute_raw_density, frequency_nerf.py:149-170) -> (raw [M], feat [M, width]),
    M = points.numel() / 3: raw = the density row before the softplus (no noise), feat = relu of the last layer's features;
    features=False returns feat = None and skips the feature GEMM of the last layer (density grids).  trunk_params =
    [trunk_w0, trunk_b0, ...] (2 n_trunk tensors).  Differentiable w.r.t. the points and trunk_params."""
    eng = get_engine() if engine is None else engine
    assert len(trunk_params) == 2 * spec.n_trunk, "density_forward takes the trunk's 2 * n_trunk tensors"
    return DensityFunction.apply(spec, eng, torch.is_grad_enabled(), bool(features), points, progress, *trunk_params)


@torch.no_grad()
def density_gradient(spec: MLPSpec, points, trunk_params: Sequence[torch.Tensor], progress=None, engine: Optional[int] = None):
    """d raw / d x at points [..., 3] -> [..., 3], raw as density_forward computes it (no noise, the BARF mask at
    progress): sparf_density_gradient, the density backward's input gradients without its weight gradients.  Bit for bit
    the points' gradient of density_forward(...)[0].sum() on every engine.  No autograd; counted in EVALS["bwd"]."""
    eng = get_engine() if engine is None else int(engine)
    if not torch.is_tensor(points) or points.dim() < 1 or points.shape[-1] != 3:
        raise ValueError("density_gradient: points must be a tensor [..., 3], got %s"
                         % ((tuple(points.shape),) if torch.is_tensor(points) else type(points).__name__))
    if not points.is_cuda:
        raise ValueError("density_gradient: points must be a CUDA tensor")
    if len(trunk_params) != 2 * spec.n_trunk:
        raise ValueError("density_gradient takes the trunk's 2 * n_trunk = %d tensors, got %d"
                         % (2 * spec.n_trunk, len(trunk_params)))
    if eng not in _lib.ENGINES.values():
        raise ValueError("density_gradient: unknown engine %r" % (engine,))
    if spec.barf_c2f is not None and progress is None:
        raise ValueError("density_gradient: a BARF coarse-to-fine spec needs progress")
    return _density_gradient(spec, eng, points, progress, trunk_params)


@_on_tensor_device
def _density_gradient(spec, eng, points, progress, trunk_params):
    L = _lib.lib()
    pts = _f32c(points).reshape(-1, 3)
    M = pts.shape[0]
    out = torch.empty_like(pts)
    if M == 0:
        return out.view(points.shape)
    m, keep = spec.fill(trunk_params, progress)
    ws = _workspace(L.sparf_density_workspace_bytes(ctypes.byref(m), M, 2, eng), pts.device)
    EVALS["bwd"] += M
    with _timed("density_gradient"):
        check(L.sparf_density_gradient(ctypes.byref(m), eng, M, _ptr(pts), _ptr(out), _ptr(ws), ws.numel(), _stream()),
              "density_gradient")
    return out.view(points.shape)


# ------------------------------------------------------------------------------------------------
# marching cubes (no gradient)
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
@_on_tensor_device
def marching_cubes(vol, iso: float):
    """Iso-surface of a dense volume vol [nx, ny, nz] (inside: vol >= iso) -> (verts [V, 3] fp32 in index space, faces
    [F, 3] int64), on vol's device; the semantics of mcubes.marching_cubes, specified in include/sparf_b200.h.  One
    device-to-host copy: the two totals that size the outputs.  Not differentiable."""
    L = _lib.lib()
    return _marching_cubes(vol, iso, L.sparf_mcubes_count, L.sparf_mcubes_emit, "mcubes")


@torch.no_grad()
@_on_tensor_device
def marching_cubes_masked(vol, iso: float):
    """marching_cubes for a volume whose unobserved points are NaN: a cell with a non-finite corner emits no triangle,
    and only the vertices the remaining triangles use are kept, renumbered in the dense order (sparf_mcubes_count_masked
    / _emit_masked).  On a volume without NaN or infinity the output is marching_cubes's, byte for byte."""
    L = _lib.lib()
    return _marching_cubes(vol, iso, L.sparf_mcubes_count_masked, L.sparf_mcubes_emit_masked, "mcubes_masked")


def _marching_cubes(vol, iso, count, emit, what):
    v = _f32c(vol)
    assert v.dim() == 3, "marching_cubes takes a 3-D volume"
    nx, ny, nz = v.shape
    ws = torch.empty(max(_lib.lib().sparf_mcubes_workspace_bytes(nx, ny, nz), 1), dtype=torch.uint8, device=v.device)
    totals = torch.empty(2, dtype=torch.int64, device=v.device)
    check(count(_ptr(v), nx, ny, nz, float(iso), _ptr(totals), _ptr(ws), ws.numel(), _stream()), what + "_count")
    n_verts, n_faces = totals.tolist()
    verts = torch.empty(n_verts, 3, device=v.device, dtype=torch.float32)
    faces = torch.empty(n_faces, 3, device=v.device, dtype=torch.int64)
    check(emit(_ptr(v), nx, ny, nz, float(iso), _ptr(verts), _ptr(faces), _ptr(ws), ws.numel(), _stream()), what + "_emit")
    return verts, faces


@torch.no_grad()
@_on_tensor_device
def mcubes_sparse_classify(coarse, iso: float):
    """Coarse density [nb+1]^3 (the lattice points at multiples of SPARF_MCUBES_BLOCK) -> (slots [nb^3] int32, -1 or
    the block's rank; block_ids [n_active] int64, the active blocks in linear order).  A block is active iff its
    coarse window (indices [b-1, b+2] per axis, clipped) holds a NaN or values on both sides of iso (include/sparf_b200.h).
    One device-to-host copy: the active count."""
    L = _lib.lib()
    c = _f32c(coarse)
    assert c.dim() == 3 and c.shape[0] == c.shape[1] == c.shape[2] >= 2, "mcubes_sparse_classify takes an [nb+1]^3 lattice"
    res = (c.shape[0] - 1) * _lib.MCUBES_BLOCK
    ws = torch.empty(max(L.sparf_mcubes_sparse_workspace_bytes(res, 0, 0), 1), dtype=torch.uint8, device=c.device)
    slots = torch.empty((res // _lib.MCUBES_BLOCK) ** 3, dtype=torch.int32, device=c.device)
    n_active = torch.empty(1, dtype=torch.int64, device=c.device)
    check(L.sparf_mcubes_sparse_classify(_ptr(c), res, float(iso), _ptr(slots), _ptr(n_active), _ptr(ws), ws.numel(),
                                         _stream()), "mcubes_sparse_classify")
    block_ids = torch.empty(int(n_active.item()), dtype=torch.int64, device=c.device)
    if block_ids.numel():       # no active block: nothing to list (and an empty tensor has no storage to pass)
        check(L.sparf_mcubes_sparse_blocks(_ptr(slots), res, _ptr(block_ids), _stream()), "mcubes_sparse_blocks")
    return slots, block_ids


@torch.no_grad()
@_on_tensor_device
def mcubes_sparse_points(axis, block_ids, b0: int, n_blocks: int):
    """The lattice points [n_blocks * 729, 3] of the active blocks block_ids[b0 : b0 + n_blocks] over the lattice axis
    [res+1] (on the device): per block its (B+1)^3 points, k fastest."""
    L = _lib.lib()
    t = _f32c(axis)
    res = t.numel() - 1
    ids = block_ids.contiguous()
    assert ids.dtype == torch.int64 and 0 <= b0 and b0 + n_blocks <= ids.numel()
    pts = torch.empty(n_blocks * (_lib.MCUBES_BLOCK + 1) ** 3, 3, device=t.device, dtype=torch.float32)
    check(L.sparf_mcubes_sparse_points(_ptr(t), res, _ptr(ids), int(b0), int(n_blocks), _ptr(pts), _stream()),
          "mcubes_sparse_points")
    return pts


@torch.no_grad()
@_on_tensor_device
def marching_cubes_sparse(sigma_blocks, res: int, slots, block_ids, iso: float):
    """Marching cubes over the active blocks only: sigma_blocks [n_active, 9, 9, 9] (the density at the points of
    block_ids, as mcubes_sparse_points lays them out), slots / block_ids of mcubes_sparse_classify -> (verts [V, 3] fp32 in
    index space, faces [F, 3] int64): the dense mesh of the [res+1]^3 lattice restricted to the cells of active blocks
    (include/sparf_b200.h).  One device-to-host copy: the two totals that size the outputs.  Not differentiable."""
    L = _lib.lib()
    s = _f32c(sigma_blocks)
    P = _lib.MCUBES_BLOCK + 1
    n = block_ids.numel()
    assert s.shape == (n, P, P, P), "marching_cubes_sparse takes sigma_blocks [n_active, 9, 9, 9]"
    assert slots.dtype == torch.int32 and block_ids.dtype == torch.int64
    assert res % _lib.MCUBES_BLOCK == 0 and slots.numel() == (res // _lib.MCUBES_BLOCK) ** 3, \
        "marching_cubes_sparse: slots [%d] is not the block table of res %d" % (slots.numel(), res)
    sl, ids = slots.contiguous(), block_ids.contiguous()
    dev = s.device
    ws = torch.empty(max(L.sparf_mcubes_sparse_workspace_bytes(res, n, 0), 1), dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    check(L.sparf_mcubes_sparse_count(_ptr(s), res, _ptr(sl), _ptr(ids), n, float(iso), _ptr(totals), _ptr(ws),
                                      ws.numel(), _stream()), "mcubes_sparse_count")
    n_verts, n_faces = totals.tolist()
    verts = torch.empty(n_verts, 3, device=dev, dtype=torch.float32)
    faces = torch.empty(n_faces, 3, device=dev, dtype=torch.int64)
    del ws
    ws = torch.empty(max(L.sparf_mcubes_sparse_workspace_bytes(res, n, n_verts), 1), dtype=torch.uint8, device=dev)
    check(L.sparf_mcubes_sparse_emit(_ptr(s), res, _ptr(sl), _ptr(ids), n, float(iso), n_verts, n_faces, _ptr(verts),
                                     _ptr(faces), _ptr(ws), ws.numel(), _stream()), "mcubes_sparse_emit")
    return verts, faces


# ------------------------------------------------------------------------------------------------
# mesh components (no gradient)
# ------------------------------------------------------------------------------------------------
MAX_MESH_ELEMENTS = 2 ** 31 - 1     # INT32_MAX: the most vertices and faces sparf_mesh_components takes


def _check_faces(faces, n_verts, what):
    """int(n_verts); ValueError unless faces is a CUDA int64 [F, 3] tensor and 0 <= n_verts, F <= INT32_MAX (no device
    access)"""
    if not torch.is_tensor(faces) or faces.dtype != torch.int64 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("%s: faces must be an int64 tensor [F, 3]" % what)
    integral = isinstance(n_verts, numbers.Integral) and not isinstance(n_verts, bool)
    if not integral or not 0 <= n_verts <= MAX_MESH_ELEMENTS:
        raise ValueError("%s: n_verts must be an int in [0, 2^31 - 1] (got %r)" % (what, n_verts))
    if faces.shape[0] > MAX_MESH_ELEMENTS or (n_verts == 0 and faces.shape[0]):
        raise ValueError("%s: %d faces over %d vertices" % (what, faces.shape[0], n_verts))
    if not faces.is_cuda:
        raise ValueError("%s: faces must be a CUDA tensor" % what)
    return int(n_verts)


def _check_ids(faces, n_verts, what):
    """ValueError unless every face id is in [0, n_verts) (one device-to-host copy)"""
    if faces.numel():
        lo, hi = torch.aminmax(faces)
        if lo.item() < 0 or hi.item() >= n_verts:
            raise ValueError("%s: face ids must lie in [0, %d)" % (what, n_verts))


@torch.no_grad()
@_on_tensor_device
def mesh_components(faces, n_verts: int):
    """Connected components of a triangle mesh with faces [F, 3] (int64, CUDA) over n_verts vertices -> (labels
    [n_verts] int32, face_counts [C] int64), on faces' device (include/sparf_b200.h).  Two vertices are connected when a
    face holds both; a component's label is the rank of its smallest vertex id, so labels run 0 .. C-1 in order of first
    vertex; a vertex no face uses is a component with 0 faces.  face_counts counts each face under the label of its first
    vertex.  Deterministic.  Bad arguments raise ValueError before any library call (one device-to-host copy checks
    the ids); one more copy reads C."""
    n_verts = _check_faces(faces, n_verts, "mesh_components")
    _check_ids(faces, n_verts, "mesh_components")
    L = _lib.lib()
    f = faces.contiguous()
    dev, F = f.device, f.shape[0]
    labels = torch.empty(n_verts, dtype=torch.int32, device=dev)
    n_comp = torch.empty(1, dtype=torch.int64, device=dev)
    ws = torch.empty(max(L.sparf_mesh_components_workspace_bytes(n_verts, F), 1), dtype=torch.uint8, device=dev)
    check(L.sparf_mesh_components(_ptr(f), F, n_verts, _ptr(labels), _ptr(n_comp), _ptr(ws), ws.numel(), _stream()),
          "mesh_components")
    C = int(n_comp.item())
    counts = torch.empty(C, dtype=torch.int64, device=dev)
    check(L.sparf_mesh_component_faces(_ptr(f), F, n_verts, _ptr(labels), C, _ptr(counts), _stream()),
          "mesh_component_faces")
    return labels, counts


@torch.no_grad()
@_on_tensor_device
def mesh_select(faces, n_verts: int, labels, keep):
    """The mesh of the kept components: faces [F, 3] and labels [n_verts] (int32) of mesh_components, keep [C] (bool or
    uint8, nonzero = kept) -> (vert_ids [V'] int64, the old id of each kept vertex, increasing; faces [F', 3] int64, the
    kept faces in their original order with renumbered ids).  Gather per-vertex data with vert_ids.  Bad arguments raise
    ValueError before any library call (device-to-host copies check the ids and labels); one more copy reads V', F'."""
    what = "mesh_select"
    n_verts = _check_faces(faces, n_verts, what)
    if not torch.is_tensor(labels) or labels.dtype != torch.int32 or labels.shape != (n_verts,):
        raise ValueError("%s: labels must be an int32 tensor [%d]" % (what, n_verts))
    if not torch.is_tensor(keep) or keep.dtype not in (torch.uint8, torch.bool) or keep.dim() != 1:
        raise ValueError("%s: keep must be a uint8 or bool tensor [C]" % what)
    if keep.numel() > max(n_verts, 0) or (n_verts and not keep.numel()):
        raise ValueError("%s: keep [%d] cannot be a component mask of %d vertices" % (what, keep.numel(), n_verts))
    if labels.device != faces.device or keep.device != faces.device:
        raise ValueError("%s: faces, labels and keep must be on one CUDA device" % what)
    _check_ids(faces, n_verts, what)
    if n_verts:
        lo, hi = torch.aminmax(labels)
        if lo.item() < 0 or hi.item() >= keep.numel():
            raise ValueError("%s: labels must lie in [0, %d)" % (what, keep.numel()))
    L = _lib.lib()
    f, lab, k = faces.contiguous(), labels.contiguous(), keep.contiguous().view(torch.uint8)
    dev, F, C = f.device, f.shape[0], k.numel()
    ws = torch.empty(max(L.sparf_mesh_components_workspace_bytes(n_verts, F), 1), dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    args = (_ptr(f), F, n_verts, _ptr(lab), _ptr(k), C)
    check(L.sparf_mesh_select_count(*args, _ptr(totals), _ptr(ws), ws.numel(), _stream()), "mesh_select_count")
    n_v, n_f = totals.tolist()
    vert_ids = torch.empty(n_v, dtype=torch.int64, device=dev)
    faces_out = torch.empty(n_f, 3, dtype=torch.int64, device=dev)
    check(L.sparf_mesh_select_emit(*args, _ptr(vert_ids), _ptr(faces_out), _ptr(ws), ws.numel(), _stream()),
          "mesh_select_emit")
    return vert_ids, faces_out


MAX_SIMPLIFY_FACES = MAX_MESH_ELEMENTS // 3     # sparf_mesh_simplify counts 3 half-edge entries per face in int32


@torch.no_grad()
@_on_tensor_device
def mesh_simplify(vertices, faces, target_faces: int, attrs=None, stats=None):
    """Quadric-error edge collapses (include/sparf_b200.h, mesh simplification) of the mesh vertices [V, 3] (fp32, CUDA),
    faces [F, 3] (int64) with optional per-vertex attrs [V, A] (fp32, interpolated along the collapses) until at most
    target_faces faces are left or no edge can collapse -> (vertices [V', 3], faces [F', 3] int64, vert_ids [V'] int64,
    the original id of each kept vertex, increasing; attrs [V', A] or None).  Deterministic; target_faces >= F returns
    the input's bytes.  Bad arguments raise ValueError before any library call (one device-to-host copy checks the ids);
    each round reads {F_live, collapses} back.  stats: an optional dict that receives rounds and collapses."""
    what = "mesh_simplify"
    if not torch.is_tensor(vertices) or vertices.dtype != torch.float32 or vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError("%s: vertices must be a float32 tensor [V, 3]" % what)
    n_verts = vertices.shape[0]
    _check_faces(faces, n_verts, what)
    if faces.shape[0] > MAX_SIMPLIFY_FACES:
        raise ValueError("%s: %d faces (at most %d)" % (what, faces.shape[0], MAX_SIMPLIFY_FACES))
    if isinstance(target_faces, bool) or not isinstance(target_faces, numbers.Integral) or target_faces < 0:
        raise ValueError("%s: target_faces must be an int >= 0 (got %r)" % (what, target_faces))
    if attrs is not None and (not torch.is_tensor(attrs) or attrs.dtype != torch.float32 or attrs.dim() != 2
                              or attrs.shape[0] != n_verts):
        raise ValueError("%s: attrs must be None or a float32 tensor [%d, A]" % (what, n_verts))
    if vertices.device != faces.device or (attrs is not None and attrs.device != faces.device):
        raise ValueError("%s: vertices, faces and attrs must be on one CUDA device" % what)
    _check_ids(faces, n_verts, what)
    L = _lib.lib()
    v, f = vertices.contiguous(), faces.contiguous()
    a = attrs.contiguous() if attrs is not None else None
    dev, F, A = f.device, f.shape[0], 0 if a is None else a.shape[1]
    ws = torch.empty(max(L.sparf_mesh_simplify_workspace_bytes(n_verts, F, A), 1), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    check(L.sparf_mesh_simplify_init(_ptr(v), _ptr(f), _ptr(a), n_verts, F, A, _ptr(counts), _ptr(ws), ws.numel(),
                                     _stream()), "mesh_simplify_init")
    n_live, rounds, collapses = F, 0, 0
    while n_live > target_faces:
        k = (n_live - target_faces + 1) // 2
        check(L.sparf_mesh_simplify_round(n_verts, F, A, n_live, k, _ptr(counts), _ptr(ws), ws.numel(), _stream()),
              "mesh_simplify_round")
        n_live, winners = counts.tolist()
        rounds += 1
        collapses += winners
        if winners == 0:
            break
    n_out = n_verts - collapses
    v_out = torch.empty(n_out, 3, dtype=torch.float32, device=dev)
    a_out = torch.empty(n_out, A, dtype=torch.float32, device=dev) if a is not None else None
    vert_ids = torch.empty(n_out, dtype=torch.int64, device=dev)
    f_out = torch.empty(n_live, 3, dtype=torch.int64, device=dev)
    check(L.sparf_mesh_simplify_emit(n_verts, F, A, n_live, _ptr(v_out), _ptr(a_out), _ptr(vert_ids), _ptr(f_out),
                                     _ptr(ws), ws.numel(), _stream()), "mesh_simplify_emit")
    if stats is not None:
        stats.update(rounds=rounds, collapses=collapses)
    return v_out, f_out, vert_ids, a_out


# ------------------------------------------------------------------------------------------------
# mesh distance (no gradient)
# ------------------------------------------------------------------------------------------------
GRID_BYTES = 40                 # sizeof(SparfDistanceGrid)
MAX_GRID_CELLS = 1 << 24


class DistanceGrid:
    """A uniform grid over a target surface (distance_grid; include/sparf_b200.h, mesh distance): the target (vertices
    [V, 3] fp32, faces [F, 3] int64 or None for a point cloud), the device grid description (params, the 40 bytes of
    SparfDistanceGrid), the CSR lists cell_start [n_cells + 1] and prims [entries] (int32), and on the host the cells
    per axis (dims) and the entry count.  Build it once, query it with closest_points as often as needed."""

    def __init__(self, vertices, faces, params, cell_start, prims, dims, entries):
        self.vertices, self.faces, self.params = vertices, faces, params
        self.cell_start, self.prims, self.dims, self.entries = cell_start, prims, dims, entries

    @property
    def n_prims(self) -> int:
        return self.vertices.shape[0] if self.faces is None else self.faces.shape[0]

    def _target(self):
        F = -1 if self.faces is None else self.faces.shape[0]
        return (_ptr(self.vertices), self.vertices.shape[0], _ptr(self.faces), F)


def _check_cells(cells_per_axis, what):
    """(cx, cy, cz): (0, 0, 0) for None (automatic), else the given int or three ints, each >= 1, at most 2^24 cells"""
    if cells_per_axis is None:
        return (0, 0, 0)
    if isinstance(cells_per_axis, numbers.Integral):
        c = (cells_per_axis,) * 3
    elif isinstance(cells_per_axis, (tuple, list)):
        c = tuple(cells_per_axis)
    else:
        c = ()
    if (len(c) != 3 or any(isinstance(x, bool) or not isinstance(x, numbers.Integral) or x < 1 for x in c)
            or c[0] * c[1] * c[2] > MAX_GRID_CELLS):
        raise ValueError("%s: cells_per_axis must be None, an int or three ints, each >= 1, with at most 2^24 cells "
                         "(got %r)" % (what, cells_per_axis))
    return tuple(int(x) for x in c)


@torch.no_grad()
@_on_tensor_device
def distance_grid(vertices, faces=None, cells_per_axis=None) -> DistanceGrid:
    """The uniform grid of closest_points over a triangle mesh (vertices [V, 3] fp32, faces [F, 3] int64, CUDA) or, with
    faces None, over the point cloud vertices (include/sparf_b200.h, mesh distance).  cells_per_axis: None (automatic:
    about min(2^24, P^1.5) cells for P primitives), an int or three ints; the query results do not depend on it.  Bad
    arguments raise ValueError before any library call (with faces, one device-to-host copy checks the ids); one more
    copy reads the entry and cell counts."""
    what = "distance_grid"
    if not torch.is_tensor(vertices) or vertices.dtype != torch.float32 or vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError("%s: vertices must be a float32 tensor [V, 3]" % what)
    n_verts = vertices.shape[0]
    if n_verts > MAX_MESH_ELEMENTS:
        raise ValueError("%s: %d vertices (at most 2^31 - 1)" % (what, n_verts))
    cells = _check_cells(cells_per_axis, what)
    if faces is not None:
        _check_faces(faces, n_verts, what)
        if faces.device != vertices.device:
            raise ValueError("%s: vertices and faces must be on one CUDA device" % what)
    if not vertices.is_cuda:
        raise ValueError("%s: vertices must be a CUDA tensor" % what)
    if faces is not None:
        _check_ids(faces, n_verts, what)
    L = _lib.lib()
    v = vertices.contiguous()
    f = faces.contiguous() if faces is not None else None
    dev = v.device
    P = n_verts if f is None else f.shape[0]
    target = (_ptr(v), n_verts, _ptr(f), -1 if f is None else f.shape[0])
    params = torch.empty(GRID_BYTES, dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    ws = torch.empty(max(L.sparf_distance_grid_workspace_bytes(P, 0), 1), dtype=torch.uint8, device=dev)
    check(L.sparf_distance_grid_count(*target, *cells, _ptr(params), _ptr(totals), _ptr(ws), ws.numel(), _stream()),
          "distance_grid_count")
    entries, n_cells, *dims = torch.cat([totals, params.view(torch.int32)[6:9].long()]).tolist()
    if entries > MAX_MESH_ELEMENTS:
        raise RuntimeError("%s: %d grid entries (at most 2^31 - 1): give fewer cells_per_axis" % (what, entries))
    ws = torch.empty(max(L.sparf_distance_grid_workspace_bytes(P, entries), 1), dtype=torch.uint8, device=dev)
    cell_start = torch.empty(n_cells + 1, dtype=torch.int32, device=dev)
    prims = torch.empty(entries, dtype=torch.int32, device=dev)
    check(L.sparf_distance_grid_fill(*target, _ptr(params), n_cells, entries, _ptr(cell_start), _ptr(prims), _ptr(ws),
                                     ws.numel(), _stream()), "distance_grid_fill")
    return DistanceGrid(v, f, params, cell_start, prims, tuple(dims), entries)


@torch.no_grad()
@_on_tensor_device
def closest_points(grid: DistanceGrid, points, max_dist: float = float("inf")):
    """The nearest primitive of grid's target to each of points [N, 3] (fp32, CUDA) -> (dist [N] fp32, index [N] int64,
    closest [N, 3] fp32): the exact minimum over all primitives (ties to the smallest id), the same bytes for every
    grid; inf / -1 / NaN where no primitive lies within max_dist (>= 0, inf allowed).  No host synchronisation, so it
    can be captured in a CUDA graph.  Bad arguments raise ValueError before any library call."""
    what = "closest_points"
    if not isinstance(grid, DistanceGrid):
        raise ValueError("%s: grid must be a DistanceGrid of distance_grid" % what)
    if not torch.is_tensor(points) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError("%s: points must be a float32 tensor [N, 3]" % what)
    if points.shape[0] > MAX_MESH_ELEMENTS:
        raise ValueError("%s: %d points (at most 2^31 - 1)" % (what, points.shape[0]))
    if points.device != grid.vertices.device:
        raise ValueError("%s: points must be on the grid's CUDA device" % what)
    if not isinstance(max_dist, numbers.Real) or not max_dist >= 0:
        raise ValueError("%s: max_dist must be a number >= 0 or inf (got %r)" % (what, max_dist))
    L = _lib.lib()
    p = points.contiguous()
    N, dev = p.shape[0], p.device
    dist = torch.empty(N, dtype=torch.float32, device=dev)
    index = torch.empty(N, dtype=torch.int64, device=dev)
    closest = torch.empty(N, 3, dtype=torch.float32, device=dev)
    check(L.sparf_distance_query(*grid._target(), _ptr(grid.params), _ptr(grid.cell_start), _ptr(grid.prims), _ptr(p),
                                 N, float(max_dist), _ptr(dist), _ptr(index), _ptr(closest), _stream()),
          "distance_query")
    return dist, index, closest


@torch.no_grad()
@_on_tensor_device
def raycast(grid: DistanceGrid, origins, dirs, t_min: float = 0.0, t_max: float = float("inf")):
    """The first triangle of grid's mesh that each ray o + t d meets, origins and dirs [N, 3] (fp32, CUDA) ->
    (t [N] fp32, face [N] int64, bary [N, 3] fp32): the exact minimum over all triangles of (t, id) with t in [t_min,
    t_max] (ties to the smallest id) by a watertight, two-sided hit test, the same bytes for every grid, and the hit's
    barycentrics of the face's vertices; inf / -1 / NaN for a miss (include/sparf_b200.h, mesh ray cast).  t is in
    units of d: a pixel ray of raygen (camera-space z = 1) gives the camera z-depth.  No host synchronisation, so it
    can be captured in a CUDA graph.  Bad arguments raise ValueError before any library call."""
    what = "raycast"
    if not isinstance(grid, DistanceGrid) or grid.faces is None:
        raise ValueError("%s: grid must be a DistanceGrid of a triangle mesh (distance_grid with faces)" % what)
    for name, x in (("origins", origins), ("dirs", dirs)):
        if not torch.is_tensor(x) or x.dtype != torch.float32 or x.dim() != 2 or x.shape[1] != 3:
            raise ValueError("%s: %s must be a float32 tensor [N, 3]" % (what, name))
        if x.device != grid.vertices.device:
            raise ValueError("%s: %s must be on the grid's CUDA device" % (what, name))
    if origins.shape != dirs.shape:
        raise ValueError("%s: origins %s and dirs %s differ" % (what, list(origins.shape), list(dirs.shape)))
    if origins.shape[0] > MAX_MESH_ELEMENTS:
        raise ValueError("%s: %d rays (at most 2^31 - 1)" % (what, origins.shape[0]))
    real = lambda x: isinstance(x, numbers.Real) and not isinstance(x, bool)
    if not real(t_min) or not real(t_max) or not 0 <= t_min <= t_max:
        raise ValueError("%s: need 0 <= t_min <= t_max (inf allowed), got %r, %r" % (what, t_min, t_max))
    L = _lib.lib()
    o, d = origins.contiguous(), dirs.contiguous()
    N, dev = o.shape[0], o.device
    t = torch.empty(N, dtype=torch.float32, device=dev)
    face = torch.empty(N, dtype=torch.int64, device=dev)
    bary = torch.empty(N, 3, dtype=torch.float32, device=dev)
    check(L.sparf_raycast(*grid._target(), _ptr(grid.params), _ptr(grid.cell_start), _ptr(grid.prims), _ptr(o), _ptr(d),
                          N, float(t_min), float(t_max), _ptr(t), _ptr(face), _ptr(bary), _stream()), "raycast")
    return t, face, bary


# ------------------------------------------------------------------------------------------------
# occupancy grid (no gradient)
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
@_on_tensor_device
def occupancy_build(sigma, thres: float):
    """Density lattice sigma [res+1]^3 -> occupancy bits [ceil(res^3 / 32)] (int32 storage of the uint32 words): cell
    (i,j,k) is occupied iff a lattice point with indices in [c-1, c+2] per axis has sigma >= thres or NaN (semantics in
    include/sparf_b200.h)."""
    L = _lib.lib()
    s = _f32c(sigma)
    assert s.dim() == 3 and s.shape[0] == s.shape[1] == s.shape[2] >= 2, "occupancy_build takes a [res+1]^3 lattice"
    res = s.shape[0] - 1
    bits = torch.empty((res ** 3 + 31) // 32, dtype=torch.int32, device=s.device)
    check(L.sparf_occupancy_build(_ptr(s), res, float(thres), _ptr(bits), _stream()), "occupancy_build")
    return bits


@torch.no_grad()
@_on_tensor_device
def occupancy_compact(bits, res: int, range, origins, dirs, t):
    """The samples x = o + t d (origins, dirs [R,3], t [R,S]) an occupancy grid keeps -> (sample_idx [K] int64 = r * S + k,
    origins_k [K,3], dirs_k [K,3], t_k [K,1]) in increasing sample order: the inputs of mlp_forward for exactly the kept
    samples.  One device-to-host copy (K).  Not differentiable."""
    L = _lib.lib()
    o, d, tt = _f32c(origins), _f32c(dirs), _f32c(t)
    R, S = tt.shape
    assert o.shape == (R, 3) and d.shape == (R, 3)
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.numel() == (res ** 3 + 31) // 32
    r0, r1 = float(range[0]), float(range[1])
    dev = tt.device
    ws = _workspace(L.sparf_occupancy_workspace_bytes(R, S), dev)
    K = torch.empty((), dtype=torch.int64, device=dev)
    args = (R, S, _ptr(o), _ptr(d), _ptr(tt), _ptr(bits), int(res), r0, r1)
    check(L.sparf_occupancy_count(*args, _ptr(K), _ptr(ws), ws.numel(), _stream()), "occupancy_count")
    k = int(K.item())
    sample_idx = torch.empty(k, dtype=torch.int64, device=dev)
    o_k, d_k = torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev)
    t_k = torch.empty(k, 1, device=dev)
    check(L.sparf_occupancy_emit(*args, _ptr(sample_idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(), _stream()),
          "occupancy_emit")
    return sample_idx, o_k, d_k, t_k


@torch.no_grad()
@_on_tensor_device
def occupancy_sample(bits, res: int, range, contraction, n_uniform: int, n_occupied: int, u_cell, u_jit):
    """The cells an occupancy-grid update re-samples and a jittered point in each -> (cells [N] int64 linear indices,
    points [N,3] fp32), N = n_uniform + n_occupied: the first n_uniform drawn uniformly from the interior cells, the rest
    from the occupied interior cells of `bits` (uniformly when none is), by u_cell [N] and u_jit [N,3] in [0, 1)
    (semantics in include/sparf_b200.h).  contraction None: a box grid over range^3; (center, radius): a contracted
    grid.  The occupied count stays on the device: nothing synchronises."""
    L = _lib.lib()
    n = int(n_uniform) + int(n_occupied)
    uc, uj = _f32c(u_cell), _f32c(u_jit)
    assert uc.shape == (n,) and uj.shape == (n, 3), "occupancy_sample: u_cell [N], u_jit [N,3]"
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.numel() == (res ** 3 + 31) // 32
    dev = uc.device
    cells = torch.empty(n, dtype=torch.int64, device=dev)
    points = torch.empty(n, 3, device=dev)
    if contraction is None:
        r0, r1, c, radius = float(range[0]), float(range[1]), None, 0.0
    else:
        r0, r1, c, radius = 0.0, 0.0, (ctypes.c_float * 3)(*[float(v) for v in contraction[0]]), float(contraction[1])
    ws = _workspace(L.sparf_occupancy_sample_workspace_bytes(int(res)), dev)
    check(L.sparf_occupancy_sample(int(res), _ptr(bits), r0, r1, c, radius, int(n_uniform), int(n_occupied), _ptr(uc),
                                   _ptr(uj), _ptr(cells), _ptr(points), _ptr(ws), ws.numel(), _stream()), "occupancy_sample")
    return cells, points


@torch.no_grad()
@_on_tensor_device
def occupancy_ema_(density, bits, res: int, contracted: bool, cells, sigma, decay: float, thres: float):
    """In place on density (fp32 [res^3]) and bits: every interior cell's density becomes max(decay * density, the
    largest sigma sampled in it), then bits = !(density < thres), a contracted grid's outer two-cell shell untouched and
    occupied (semantics in include/sparf_b200.h).  cells [N] int64 and sigma [N] as occupancy_sample and the density
    query give them.  Deterministic; nothing synchronises."""
    L = _lib.lib()
    s = _f32c(sigma).reshape(-1)
    n = s.numel()
    assert cells.dtype == torch.int64 and cells.is_contiguous() and cells.shape == (n,)
    assert density.dtype == torch.float32 and density.is_contiguous() and density.numel() == res ** 3
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.numel() == (res ** 3 + 31) // 32
    ws = _workspace(L.sparf_occupancy_sample_workspace_bytes(int(res)), density.device)
    check(L.sparf_occupancy_ema(int(res), int(bool(contracted)), n, _ptr(cells), _ptr(s), float(decay), float(thres),
                                _ptr(density), _ptr(bits), _ptr(ws), ws.numel(), _stream()), "occupancy_ema")
    return density, bits


# ------------------------------------------------------------------------------------------------
# early ray termination (no gradient)
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
@_on_tensor_device
def termination_compact(origins, dirs, t, k0: int, k1: int, alive=None, bits=None, res: int = 0, range=None):
    """The samples k in [k0, k1) of the rays with alive[r] != 0 (uint8 [R]; None = every ray) of origins, dirs [R,3],
    t [R,S], and with occupancy bits (res, range as in occupancy_compact) only those the grid keeps -> (sample_idx [K]
    int64 = r * S + k, origins_k [K,3], dirs_k [K,3], t_k [K,1]) in increasing sample order.  One device-to-host copy
    (K).  Not differentiable."""
    L = _lib.lib()
    o, d, tt = _f32c(origins), _f32c(dirs), _f32c(t)
    R, S = tt.shape
    assert o.shape == (R, 3) and d.shape == (R, 3)
    assert alive is None or (alive.dtype == torch.uint8 and alive.is_contiguous() and alive.shape == (R,))
    r0, r1 = (0.0, 1.0) if bits is None else (float(range[0]), float(range[1]))
    if bits is not None:
        assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.numel() == (res ** 3 + 31) // 32
    dev = tt.device
    ws = _workspace(L.sparf_termination_workspace_bytes(R, k1 - k0), dev)
    K = torch.empty((), dtype=torch.int64, device=dev)
    args = (R, S, int(k0), int(k1), _ptr(o), _ptr(d), _ptr(tt), _ptr(alive), _ptr(bits), int(res), r0, r1)
    check(L.sparf_termination_count(*args, _ptr(K), _ptr(ws), ws.numel(), _stream()), "termination_count")
    k = int(K.item())
    sample_idx = torch.empty(k, dtype=torch.int64, device=dev)
    o_k, d_k = torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev)
    t_k = torch.empty(k, 1, device=dev)
    check(L.sparf_termination_emit(*args, _ptr(sample_idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(),
                                   _stream()), "termination_emit")
    return sample_idx, o_k, d_k, t_k


@torch.no_grad()
@_on_tensor_device
def contracted_compact(origins, dirs, t, k0: int, k1: int, alive, bits, res: int, center, radius: float):
    """termination_compact with a contracted occupancy grid in place of the box grid: the samples k in [k0, k1) of the
    rays with alive[r] != 0 (None = every ray) that the contracted grid (bits over [-2, 2]^3 in res^3 cells; center
    (3 floats), radius: the contraction, include/sparf_b200.h) keeps -> (sample_idx [K] int64 = r * S + k, origins_k
    [K,3], dirs_k [K,3], t_k [K,1]) in increasing sample order.  k0 = 0, k1 = S, alive = None: the plain grid
    compaction.  One device-to-host copy (K).  Not differentiable."""
    L = _lib.lib()
    o, d, tt = _f32c(origins), _f32c(dirs), _f32c(t)
    R, S = tt.shape
    assert o.shape == (R, 3) and d.shape == (R, 3)
    assert alive is None or (alive.dtype == torch.uint8 and alive.is_contiguous() and alive.shape == (R,))
    assert bits.dtype == torch.int32 and bits.is_contiguous() and bits.numel() == (res ** 3 + 31) // 32
    c = (ctypes.c_float * 3)(*[float(v) for v in center])
    dev = tt.device
    ws = _workspace(L.sparf_termination_workspace_bytes(R, k1 - k0), dev)
    K = torch.empty((), dtype=torch.int64, device=dev)
    args = (R, S, int(k0), int(k1), _ptr(o), _ptr(d), _ptr(tt), _ptr(alive), _ptr(bits), int(res), c, float(radius))
    check(L.sparf_contracted_count(*args, _ptr(K), _ptr(ws), ws.numel(), _stream()), "contracted_count")
    k = int(K.item())
    sample_idx = torch.empty(k, dtype=torch.int64, device=dev)
    o_k, d_k = torch.empty(k, 3, device=dev), torch.empty(k, 3, device=dev)
    t_k = torch.empty(k, 1, device=dev)
    check(L.sparf_contracted_emit(*args, _ptr(sample_idx), _ptr(o_k), _ptr(d_k), _ptr(t_k), _ptr(ws), ws.numel(),
                                  _stream()), "contracted_emit")
    return sample_idx, o_k, d_k, t_k


@torch.no_grad()
@_on_tensor_device
def termination_update(sigma, t, dirs, k0: int, k1: int, tau_max: float, tau, alive):
    """In place, for every ray with alive[r] != 0: tau[r] += the optical depth of its samples k in [k0, k1) (sigma, t
    [R,S], dirs [R,3]; op order in include/sparf_b200.h), then alive[r] = 0 when tau[r] > tau_max.  tau: float32 [R],
    alive: uint8 [R], both contiguous."""
    L = _lib.lib()
    s, tt, d = _f32c(sigma), _f32c(t), _f32c(dirs)
    R, S = tt.shape
    assert s.shape == (R, S) and d.shape == (R, 3)
    assert tau.dtype == torch.float32 and tau.is_contiguous() and tau.shape == (R,)
    assert alive.dtype == torch.uint8 and alive.is_contiguous() and alive.shape == (R,)
    check(L.sparf_termination_update(R, S, int(k0), int(k1), _ptr(s), _ptr(tt), _ptr(d), float(tau_max), _ptr(tau),
                                     _ptr(alive), _stream()), "termination_update")


# ------------------------------------------------------------------------------------------------
# compositing
# ------------------------------------------------------------------------------------------------
class CompositeFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, sigma, rgb, t, dirs, white_bg: bool):
        L = _lib.lib()
        sigma, rgb, t, dirs = _f32c(sigma), _f32c(rgb), _f32c(t), _f32c(dirs)
        R, S = t.shape
        dev = t.device
        rgb_map = torch.empty(R, 3, device=dev)
        depth, opacity = torch.empty(R, device=dev), torch.empty(R, device=dev)
        depth_var, rgb_var = torch.empty(R, device=dev), torch.empty(R, device=dev)
        weights, all_cum = torch.empty(R, S, device=dev), torch.empty(R, device=dev)
        check(L.sparf_composite_forward(R, S, _ptr(sigma), _ptr(rgb), _ptr(t), _ptr(dirs), int(white_bg), _ptr(rgb_map),
                                        _ptr(depth), _ptr(opacity), _ptr(depth_var), _ptr(rgb_var), _ptr(weights),
                                        _ptr(all_cum), _stream()), "composite_forward")
        ctx.white_bg = bool(white_bg)
        ctx.save_for_backward(sigma, rgb, t, dirs)
        ctx.mark_non_differentiable(depth_var, rgb_var, all_cum)
        # outputs nobody differentiated arrive as None in backward (the C ABI takes NULL) instead of as freshly
        # zero-filled tensors: six fill kernels and a [R,S] write + read less per render call
        ctx.set_materialize_grads(False)
        return rgb_map, depth, opacity, weights, depth_var, rgb_var, all_cum

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g_rgb, g_depth, g_opacity, g_weights, *_unused):
        L = _lib.lib()
        sigma, rgb, t, dirs = ctx.saved_tensors
        R, S = t.shape
        opt = lambda g: _f32c(g) if g is not None else None
        g_rgb, g_depth, g_opacity, g_weights = opt(g_rgb), opt(g_depth), opt(g_opacity), opt(g_weights)
        d_sigma = torch.empty_like(sigma)
        d_rgb = torch.empty_like(rgb)
        d_dirs = torch.zeros_like(dirs) if ctx.needs_input_grad[3] else None
        check(L.sparf_composite_backward(R, S, _ptr(sigma), _ptr(rgb), _ptr(t), _ptr(dirs), int(ctx.white_bg),
                                         _ptr(g_rgb), _ptr(g_depth), _ptr(g_opacity), _ptr(g_weights), _ptr(d_sigma),
                                         _ptr(d_rgb), _ptr(d_dirs), _stream()), "composite_backward")
        return d_sigma, d_rgb, None, d_dirs, None


def composite(sigma, rgb, t, dirs, white_bg=False):
    """-> rgb_map [R,3], depth [R], opacity [R], weights [R,S], depth_var [R], rgb_var [R], all_cumulated [R]."""
    return CompositeFunction.apply(sigma, rgb, t, dirs, bool(white_bg))


# ------------------------------------------------------------------------------------------------
# rays
# ------------------------------------------------------------------------------------------------
class RayGenFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, pose_w2c, intr_inv, W: int, ray_idx, pixels):
        L = _lib.lib()
        pose_w2c, intr_inv = _f32c(pose_w2c), _f32c(intr_inv)
        B = pose_w2c.shape[0]
        if pixels is not None:
            pixels = _f32c(pixels)
            per_image = int(pixels.dim() == 3)
            n = pixels.shape[-2]
            idx = None
        else:
            idx = ray_idx.to(torch.int64).contiguous()
            per_image = int(idx.dim() == 2 and idx.shape[0] == B)
            n = idx.shape[-1]
        origins = torch.empty(B, n, 3, device=pose_w2c.device)
        dirs = torch.empty(B, n, 3, device=pose_w2c.device)
        check(L.sparf_raygen_forward(B, n, int(W), _ptr(pose_w2c), _ptr(intr_inv), _ptr(idx), _ptr(pixels), per_image,
                                     _ptr(origins), _ptr(dirs), _stream()), "raygen_forward")
        ctx.args = (B, n, int(W), per_image)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(pose_w2c, intr_inv, idx if idx is not None else torch.empty(0), pixels if pixels is not None else torch.empty(0))
        ctx.has_idx = idx is not None
        return origins, dirs

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g_o, g_d):
        L = _lib.lib()
        pose_w2c, intr_inv, idx, pixels = ctx.saved_tensors
        B, n, W, per_image = ctx.args
        if g_o is None and g_d is None:
            return None, None, None, None, None
        d_pose = torch.zeros_like(pose_w2c)
        g_o = _f32c(g_o) if g_o is not None else None
        g_d = _f32c(g_d) if g_d is not None else None
        # pixel locations are differentiable in the reference (camera.py:400-416); the depth-consistency loss renders at
        # pixels projected from a rendered depth and back-propagates through them (depth_cons_loss.py:247-283)
        d_px = torch.zeros_like(pixels) if (not ctx.has_idx and ctx.needs_input_grad[4]) else None
        check(L.sparf_raygen_backward(B, n, W, _ptr(pose_w2c), _ptr(intr_inv), _ptr(idx if ctx.has_idx else None),
                                      _ptr(None if ctx.has_idx else pixels), per_image, _ptr(g_o), _ptr(g_d),
                                      _ptr(d_pose), _ptr(d_px), _stream()), "raygen_backward")
        return d_pose, None, None, None, d_px


_HOST_CACHE = {}


def cached(tag: str, tensor: torch.Tensor, fn):
    """Memoise a small derived quantity of a (device) tensor that rarely changes (intrinsics, depth range), keyed
    by storage address + in-place version, so that the hot loop neither recomputes it nor synchronises."""
    key = (tag, tensor.data_ptr(), tensor._version, tuple(tensor.shape), tensor.device)
    hit = _HOST_CACHE.get(key)
    if hit is None and tensor.is_cuda and torch.cuda.is_current_stream_capturing():
        return fn(tensor)          # graph-pool temporaries must not be memoised (their addresses are recycled)
    if hit is None:
        if len(_HOST_CACHE) > 256:
            _HOST_CACHE.clear()
        # the entry keeps `tensor` alive, so its address cannot be handed to another tensor while cached
        hit = (fn(tensor), tensor)
        _HOST_CACHE[key] = hit
    return hit[0]


def raygen(pose_w2c, intr, W: int, *, ray_idx=None, pixels=None):
    """pose_w2c [B,3,4], intr [B,3,3] (or [1,3,3] / [3,3], shared by the B poses) -> (center, ray) [B,n,3] at
    ray_idx (int [n] / [1,n] shared, or [B,n] per image) or at float pixels ([n,2] / [1,n,2] shared, or [B,n,2]).
    Any other shape raises ValueError before anything is launched."""
    if (ray_idx is None) == (pixels is None):
        raise ValueError("raygen: give exactly one of ray_idx / pixels")
    if pose_w2c.dim() != 3 or tuple(pose_w2c.shape[1:]) != (3, 4):
        raise ValueError("raygen: pose_w2c must be [B,3,4], got %s" % (tuple(pose_w2c.shape),))
    B = pose_w2c.shape[0]
    if not (tuple(intr.shape) == (3, 3) or (intr.dim() == 3 and intr.shape[0] in (1, B) and tuple(intr.shape[1:]) == (3, 3))):
        raise ValueError("raygen: intr must be [B,3,3], [1,3,3] or [3,3] for B=%d poses, got %s" % (B, tuple(intr.shape)))
    if pixels is not None:
        if not (pixels.shape[-1:] == (2,) and (pixels.dim() == 2 or (pixels.dim() == 3 and pixels.shape[0] in (1, B)))):
            raise ValueError("raygen: pixels must be [n,2], [1,n,2] or [B,n,2] for B=%d poses, got %s"
                             % (B, tuple(pixels.shape)))
        if pixels.dim() == 3 and pixels.shape[0] != B:
            pixels = pixels[0]               # [1,n,2]: one list shared by the B images
    else:
        if not (ray_idx.dim() == 1 or (ray_idx.dim() == 2 and ray_idx.shape[0] in (1, B))):
            raise ValueError("raygen: ray_idx must be [n], [1,n] or [B,n] for B=%d poses, got %s"
                             % (B, tuple(ray_idx.shape)))
    # camera.py:318-319; intrinsics carry no gradient and are constant over training: invert once
    # (inv_ex: no host-side singularity check, i.e. no synchronisation)
    intr_inv = cached("Kinv", intr, lambda k: torch.linalg.inv_ex(k.detach().float()).inverse)
    if intr_inv.dim() == 2 or intr_inv.shape[0] != B:
        intr_inv = intr_inv.reshape(1, 3, 3).expand(B, 3, 3)   # the kernel reads one K^-1 per image
    return RayGenFunction.apply(pose_w2c, intr_inv, W, ray_idx, pixels)


# ------------------------------------------------------------------------------------------------
# sampling (no gradient)
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
@_on_tensor_device
def sample_depth(R: int, S: int, near: float, rng: float, *, inverse=False, rand=None, far_per_ray=None, device=None):
    L = _lib.lib()
    device = device or (rand.device if rand is not None else far_per_ray.device)
    t = torch.empty(R, S, device=device, dtype=torch.float32)
    rand_c = _f32c(rand).reshape(R, S) if rand is not None else None
    far_c = _f32c(far_per_ray).reshape(R) if far_per_ray is not None else None
    check(L.sparf_sample_depth(R, S, float(near), float(rng), int(inverse), _ptr(rand_c), _ptr(far_c), _ptr(t), _stream()),
          "sample_depth")
    return t


@torch.no_grad()
@_on_tensor_device
def sample_pdf_merge(weights, t_coarse, u_mid, near: float, far: float):
    """weights, t_coarse [R,S]; u_mid [S_fine] -> (t_fine [R,S_fine], t_all [R,S+S_fine] ascending)."""
    L = _lib.lib()
    weights, t_coarse, u_mid = _f32c(weights), _f32c(t_coarse), _f32c(u_mid)
    R, S = weights.shape
    Sf = u_mid.numel()
    t_fine = torch.empty(R, Sf, device=weights.device)
    t_all = torch.empty(R, S + Sf, device=weights.device)
    check(L.sparf_sample_pdf_merge(R, S, Sf, float(near), float(far), _ptr(weights), _ptr(t_coarse), _ptr(u_mid),
                                   _ptr(t_fine), _ptr(t_all), _stream()), "sample_pdf_merge")
    return t_fine, t_all


# ------------------------------------------------------------------------------------------------
# photometric Huber loss
# ------------------------------------------------------------------------------------------------
class Huber2Function(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, pred, target):
        L = _lib.lib()
        pred_c, target_c = _f32c(pred), _f32c(target)
        loss = torch.zeros((), device=pred.device)
        d_pred = torch.empty_like(pred_c)
        check(L.sparf_huber2_fwd_bwd(pred_c.numel(), _ptr(pred_c), _ptr(target_c), 1.0, _ptr(loss), _ptr(d_pred), _stream()),
              "huber2")
        ctx.save_for_backward(d_pred)
        ctx.shape = pred.shape
        return loss

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g):
        (d_pred,) = ctx.saved_tensors
        return (d_pred * g).view(ctx.shape), None


def huber2(pred, target):
    """2 * mean Huber(delta=0.5)(pred - target)   (base_losses.py:155-156)."""
    return Huber2Function.apply(pred, target.expand_as(pred))


# ------------------------------------------------------------------------------------------------
# stand-alone positional encoding (the MLP kernels fuse it; this is the tensor-level op)
# ------------------------------------------------------------------------------------------------
class PosEncFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, x, L: int, barf_c2f, progress):
        lib = _lib.lib()
        x_c = _f32c(x)
        C = x_c.shape[-1]
        n = x_c.numel() // C
        out = torch.empty(*x_c.shape[:-1], 2 * C * L, device=x_c.device, dtype=torch.float32)
        use = barf_c2f is not None
        start, rng = (float(barf_c2f[0]), float(barf_c2f[1] - barf_c2f[0])) if use else (0.0, 1.0)
        prog = _f32c(progress.detach()).reshape(1) if use else None
        check(lib.sparf_posenc_forward(n, C, int(L), _ptr(x_c), int(use), start, rng, _ptr(prog), _ptr(out), _stream()), "posenc_forward")
        ctx.args = (n, C, int(L), use, start, rng)
        ctx.save_for_backward(x_c, prog if use else torch.empty(0))
        return out

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g):
        lib = _lib.lib()
        x_c, prog = ctx.saved_tensors
        n, C, L, use, start, rng = ctx.args
        d_x = torch.empty_like(x_c)
        check(lib.sparf_posenc_backward(n, C, L, _ptr(x_c), int(use), start, rng, _ptr(prog if use else None), _ptr(_f32c(g)),
                                        _ptr(d_x), _stream()), "posenc_backward")
        return d_x, None, None, None


def posenc(x, L: int, barf_c2f=None, progress=None):
    """[..., C] -> [..., 2*C*L]: per channel L sines then L cosines of x * 2^j * pi, times the BARF coarse-to-fine weight of
    band j when barf_c2f = (start, end) is given (frequency_nerf.py:47-69, 248-257).  Differentiable w.r.t. x."""
    return PosEncFunction.apply(x, L, tuple(barf_c2f) if barf_c2f is not None else None, progress)


# ------------------------------------------------------------------------------------------------
# distortion regulariser (default off in the reference's configs)
# ------------------------------------------------------------------------------------------------
class DistortionFunction(torch.autograd.Function):
    @staticmethod
    @_on_tensor_device
    def forward(ctx, t, w):
        L = _lib.lib()
        t_c, w_c = _f32c(t), _f32c(w)
        S = t_c.shape[-2] if t_c.shape[-1] == 1 else t_c.shape[-1]
        R = t_c.numel() // S
        loss = torch.zeros((), device=t.device)
        d_w = torch.empty_like(w_c)
        need_t = ctx.needs_input_grad[0]
        d_t = torch.empty_like(t_c) if need_t else None
        check(L.sparf_distortion_fwd_bwd(R, S, _ptr(t_c), _ptr(w_c), 1.0, _ptr(loss), _ptr(d_w), _ptr(d_t), _stream()),
              "distortion")
        ctx.save_for_backward(d_w, d_t if need_t else d_w)
        ctx.need_t = need_t
        ctx.shapes = (t.shape, w.shape)
        return loss

    @staticmethod
    @_on_tensor_device
    def backward(ctx, g):
        d_w, d_t = ctx.saved_tensors
        return ((d_t * g).view(ctx.shapes[0]) if ctx.need_t else None), (d_w * g).view(ctx.shapes[1])


def distortion_loss(t, w):
    """mip-NeRF-360 distortion loss of the renderer's `t`, `weights` [B,R,S,1] (regularization_losses.py:20-48), O(S)."""
    return DistortionFunction.apply(t, w)
