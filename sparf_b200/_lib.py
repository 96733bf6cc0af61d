"""ctypes binding of include/sparf_b200.h.  The product path: if the library is missing this raises
(there is NO Python/torch fallback for the kernels)."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int32, c_int64, c_size_t, c_void_p

from . import build as _build

MAX_TRUNK = 12
MCUBES_MAX_TRIS = 5     # SPARF_MCUBES_MAX_TRIS: a row of the marching-cubes case table holds 3 * 5 edge ids
MCUBES_BLOCK = 8        # SPARF_MCUBES_BLOCK: cells per block edge of sparse marching cubes

ENGINE_AUTO, ENGINE_SIMT_FP32, ENGINE_TC_3X, ENGINE_TC_1X, ENGINE_TC_3X_W1 = 0, 1, 2, 3, 4
ENGINES = {"auto": 0, "simt_fp32": 1, "tc_3x": 2, "tc_1x": 3, "tc_3x_w1": 4}


class SparfMLP(ctypes.Structure):
    _fields_ = [
        ("n_trunk", c_int32), ("width", c_int32), ("head_width", c_int32), ("skip_layer", c_int32),
        ("L_xyz", c_int32), ("L_view", c_int32), ("use_c2f", c_int32),
        ("c2f_start", c_float), ("c2f_range", c_float),
        ("progress", c_void_p),
        ("trunk_w", c_void_p * MAX_TRUNK), ("trunk_b", c_void_p * MAX_TRUNK),
        ("head_w", c_void_p * 2), ("head_b", c_void_p * 2),
    ]


class SparfMLPGrad(ctypes.Structure):
    _fields_ = [
        ("trunk_w", c_void_p * MAX_TRUNK), ("trunk_b", c_void_p * MAX_TRUNK),
        ("head_w", c_void_p * 2), ("head_b", c_void_p * 2),
    ]


_P = c_void_p
_SIGNATURES = {
    "sparf_version": (c_int32, []),
    "sparf_last_error": (c_char_p, []),
    "sparf_launch_count": (ctypes.c_uint64, []),
    "sparf_engine_available": (c_int32, [c_int32]),
    "sparf_raygen_forward": (c_int32, [c_int32, c_int32, c_int32, _P, _P, _P, _P, c_int32, _P, _P, _P]),
    "sparf_raygen_backward": (c_int32, [c_int32, c_int32, c_int32, _P, _P, _P, _P, c_int32, _P, _P, _P, _P, _P]),
    "sparf_sample_depth": (c_int32, [c_int32, c_int32, c_float, c_float, c_int32, _P, _P, _P, _P]),
    "sparf_sample_pdf_merge": (c_int32, [c_int32, c_int32, c_int32, c_float, c_float, _P, _P, _P, _P, _P, _P]),
    "sparf_mlp_workspace_bytes": (c_size_t, [POINTER(SparfMLP), c_int32, c_int32, c_int32, c_int32]),
    "sparf_mlp_forward": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_mlp_backward": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P,
                                     POINTER(SparfMLPGrad), _P, _P, _P, c_size_t, _P]),
    "sparf_mlp_tape_bytes": (c_size_t, [POINTER(SparfMLP), c_int32, c_int32, c_int32]),
    "sparf_mlp_forward_tape": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, c_size_t,
                                         _P, c_size_t, _P]),
    "sparf_mlp_backward_tape": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P,
                                          POINTER(SparfMLPGrad), _P, _P, _P, c_size_t, _P, c_size_t, _P]),
    "sparf_mlp_forward_tape_rows": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                              c_size_t, _P, c_size_t, _P]),
    "sparf_mlp_backward_tape_rows": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                               POINTER(SparfMLPGrad), _P, _P, _P, c_size_t, _P, c_size_t, _P]),
    "sparf_compact_scatter": (c_int32, [c_int64, _P, _P, c_int32, _P, _P, _P]),
    "sparf_compact_gather": (c_int32, [c_int64, _P, _P, c_int32, _P, _P, _P]),
    "sparf_compact_ray_sum": (c_int32, [c_int64, c_int32, c_int64, _P, _P, c_int32, _P, _P, _P]),
    "sparf_mlp_forward_tape_span": (c_int32, [POINTER(SparfMLP), c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                              _P, c_size_t, _P, c_size_t, _P]),
    "sparf_compact_scatter_span": (c_int32, [c_int64, _P, c_int32, _P, c_int32, _P, _P, _P]),
    "sparf_compact_gather_span": (c_int32, [c_int64, _P, c_int32, _P, c_int32, _P, _P, _P]),
    "sparf_compact_ray_sum_segments": (c_int32, [c_int64, c_int32, c_int32, _P, _P, c_int32, _P, _P, _P]),
    "sparf_density_workspace_bytes": (c_size_t, [POINTER(SparfMLP), c_int64, c_int32, c_int32]),
    "sparf_density_forward": (c_int32, [POINTER(SparfMLP), c_int32, c_int64, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_density_backward": (c_int32, [POINTER(SparfMLP), c_int32, c_int64, _P, _P, _P, POINTER(SparfMLPGrad), _P, _P,
                                         c_size_t, _P]),
    "sparf_density_gradient": (c_int32, [POINTER(SparfMLP), c_int32, c_int64, _P, _P, _P, c_size_t, _P]),
    "sparf_mcubes_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64]),
    "sparf_mcubes_count": (c_int32, [_P, c_int64, c_int64, c_int64, c_float, _P, _P, c_size_t, _P]),
    "sparf_mcubes_emit": (c_int32, [_P, c_int64, c_int64, c_int64, c_float, _P, _P, _P, c_size_t, _P]),
    "sparf_mcubes_count_masked": (c_int32, [_P, c_int64, c_int64, c_int64, c_float, _P, _P, c_size_t, _P]),
    "sparf_mcubes_emit_masked": (c_int32, [_P, c_int64, c_int64, c_int64, c_float, _P, _P, _P, c_size_t, _P]),
    "sparf_mcubes_table": (c_int32, [_P]),
    "sparf_mcubes_sparse_workspace_bytes": (c_size_t, [c_int32, c_int64, c_int64]),
    "sparf_mcubes_sparse_classify": (c_int32, [_P, c_int32, c_float, _P, _P, _P, c_size_t, _P]),
    "sparf_mcubes_sparse_blocks": (c_int32, [_P, c_int32, _P, _P]),
    "sparf_mcubes_sparse_points": (c_int32, [_P, c_int32, _P, c_int64, c_int64, _P, _P]),
    "sparf_mcubes_sparse_count": (c_int32, [_P, c_int32, _P, _P, c_int64, c_float, _P, _P, c_size_t, _P]),
    "sparf_mcubes_sparse_emit": (c_int32, [_P, c_int32, _P, _P, c_int64, c_float, c_int64, c_int64, _P, _P, _P, c_size_t,
                                           _P]),
    "sparf_tsdf_integrate": (c_int32, [_P, c_int32, c_float, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                       _P]),
    "sparf_mesh_components_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "sparf_mesh_components": (c_int32, [_P, c_int64, c_int64, _P, _P, _P, c_size_t, _P]),
    "sparf_mesh_component_faces": (c_int32, [_P, c_int64, c_int64, _P, c_int64, _P, _P]),
    "sparf_mesh_select_count": (c_int32, [_P, c_int64, c_int64, _P, _P, c_int64, _P, _P, c_size_t, _P]),
    "sparf_mesh_select_emit": (c_int32, [_P, c_int64, c_int64, _P, _P, c_int64, _P, _P, _P, c_size_t, _P]),
    "sparf_mesh_simplify_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int32]),
    "sparf_mesh_simplify_init": (c_int32, [_P, _P, _P, c_int64, c_int64, c_int32, _P, _P, c_size_t, _P]),
    "sparf_mesh_simplify_round": (c_int32, [c_int64, c_int64, c_int32, c_int64, c_int64, _P, _P, c_size_t, _P]),
    "sparf_mesh_simplify_emit": (c_int32, [c_int64, c_int64, c_int32, c_int64, _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_distance_grid_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "sparf_distance_grid_count": (c_int32, [_P, c_int64, _P, c_int64, c_int32, c_int32, c_int32, _P, _P, _P, c_size_t,
                                            _P]),
    "sparf_distance_grid_fill": (c_int32, [_P, c_int64, _P, c_int64, _P, c_int64, c_int64, _P, _P, _P, c_size_t, _P]),
    "sparf_distance_query": (c_int32, [_P, c_int64, _P, c_int64, _P, _P, _P, _P, c_int64, c_float, _P, _P, _P, _P]),
    "sparf_raycast": (c_int32, [_P, c_int64, _P, c_int64, _P, _P, _P, _P, _P, c_int64, c_float, c_float, _P, _P, _P,
                                _P]),
    "sparf_occupancy_build": (c_int32, [_P, c_int32, c_float, _P, _P]),
    "sparf_occupancy_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "sparf_occupancy_count": (c_int32, [c_int64, c_int32, _P, _P, _P, _P, c_int32, c_float, c_float, _P, _P, c_size_t, _P]),
    "sparf_occupancy_emit": (c_int32, [c_int64, c_int32, _P, _P, _P, _P, c_int32, c_float, c_float, _P, _P, _P, _P, _P,
                                       c_size_t, _P]),
    "sparf_termination_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "sparf_termination_count": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, c_float, c_float,
                                          _P, _P, c_size_t, _P]),
    "sparf_termination_emit": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, c_float, c_float,
                                         _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_termination_update": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, c_float, _P, _P, _P]),
    "sparf_termination_append": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, c_float, c_float,
                                           _P, c_int32, _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_contracted_append": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, POINTER(c_float),
                                          c_float, _P, c_int32, _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_contracted_count": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, POINTER(c_float),
                                         c_float, _P, _P, c_size_t, _P]),
    "sparf_contracted_emit": (c_int32, [c_int64, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_int32, POINTER(c_float),
                                        c_float, _P, _P, _P, _P, _P, c_size_t, _P]),
    "sparf_occupancy_sample_workspace_bytes": (c_size_t, [c_int32]),
    "sparf_occupancy_sample": (c_int32, [c_int32, _P, c_float, c_float, POINTER(c_float), c_float, c_int64, c_int64, _P, _P,
                                         _P, _P, _P, c_size_t, _P]),
    "sparf_occupancy_ema": (c_int32, [c_int32, c_int32, c_int64, _P, _P, c_float, c_float, _P, _P, _P, c_size_t, _P]),
    "sparf_composite_forward":(c_int32, [c_int32, c_int32, _P, _P, _P, _P, c_int32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "sparf_composite_backward": (c_int32, [c_int32, c_int32, _P, _P, _P, _P, c_int32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "sparf_huber2_fwd_bwd": (c_int32, [c_int64, _P, _P, c_float, _P, _P, _P]),
    "sparf_posenc_forward": (c_int32, [c_int64, c_int32, c_int32, _P, c_int32, c_float, c_float, _P, _P, _P]),
    "sparf_posenc_backward": (c_int32, [c_int64, c_int32, c_int32, _P, c_int32, c_float, c_float, _P, _P, _P, _P]),
    "sparf_distortion_fwd_bwd": (c_int32, [c_int32, c_int32, _P, _P, c_float, _P, _P, _P, _P]),
    "sparf_adam_step": (c_int32, [c_int64, _P, _P, _P, _P, _P, _P] + [ctypes.c_double] * 7 + [_P]),
    "sparf_tc_selftest": (c_int32, [_P, _P, c_int32, _P, _P, _P]),
    "sparf_tc_selftest_tn": (c_int32, [_P, _P, c_int32, _P, _P]),
    "sparf_tc_selftest_images": (c_int32, [_P, _P, _P, _P, c_int32, _P, _P, _P, _P]),
    "sparf_tc_selftest_persistent": (c_int32, [_P, _P, _P, _P, c_int32, _P, _P, _P, c_int32, _P]),
    "sparf_tc_selftest_head": (c_int32, [_P, _P, _P, _P, _P, _P, c_int32, c_int32, c_int32, c_int32, _P, _P, _P]),
    "sparf_tc_selftest_featgrad": (c_int32, [_P, _P, _P, c_int32, c_int32, c_int32, c_int32, _P, _P, _P]),
    "sparf_tc_selftest_wgrad": (c_int32, [_P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                          _P, _P, _P]),
    "sparf_tc_selftest_wgrad_rows": (c_int32, [_P, _P, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                               c_int32, _P, _P, _P, _P]),
    "sparf_tc_selftest_mask_bits": (c_int32, [_P, _P, _P, c_int32, c_int32, c_int32, c_int32, _P, _P]),
    "sparf_tc_selftest_chain": (c_int32, [_P, c_int32, c_int32, c_int32, c_int32, _P, _P, c_int32, c_int32, c_int32, c_int32,
                                          ctypes.c_uint32, _P, _P, _P, _P]),
    "sparf_tc_selftest_chain_bits": (c_int32, [_P, c_int32, c_int32, c_int32, c_int32, _P, _P, c_int32, c_int32, c_int32,
                                               _P, _P, _P, _P]),
    "sparf_tc_selftest_dgrad_chain": (c_int32, [_P, c_int32, c_int32, c_int32, c_int32, _P, _P, c_int32, c_int32, c_int32,
                                                c_int32, _P, _P, _P, _P, _P]),
}

_lib = None


def exported_symbols():
    """Names every entry point include/sparf_b200.h declares (used by the CPU-side ABI test)."""
    return list(_SIGNATURES)


def lib():
    """Load (building first if the sources are newer) the shared library; fail loudly otherwise."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    override = os.environ.get("SPARF_B200_LIB")     # experiment builds (python -m sparf_b200.build --variant), tools only
    if override:
        if not os.path.exists(override):
            raise RuntimeError("SPARF_B200_LIB=%s does not exist" % override)
        path = override
    elif not os.path.exists(path) or _build._stale():
        try:
            path = _build.build()
        except Exception as e:  # no nvcc on this box and no prebuilt library: nothing to run
            if not os.path.exists(path):
                raise RuntimeError(
                    "sparf_b200: native library %s is missing and could not be built (%s). "
                    "There is no fallback path." % (path, e))
    L = ctypes.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().sparf_last_error()
        raise RuntimeError("sparf_b200 %s failed (code %d): %s" % (what, rc, msg.decode() if msg else "?"))
