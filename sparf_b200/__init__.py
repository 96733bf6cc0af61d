"""sparf_b200: volumetric renderer for SPARF's ray-marching hot path on the H100 (sm_90a).

Host side (this package) mirrors the reference's Python API (`Graph`, `NeRF`, loss modules); all
arithmetic runs in hand-written sm_90a CUDA behind the C ABI in include/sparf_b200.h.
"""
from . import ops  # noqa: F401
from .ops import set_engine, get_engine  # noqa: F401

__version__ = "0.1.0"


def install_as_reference_renderer() -> None:
    """Make `import source.models.renderer` / `source.models.frequency_nerf` resolve to this package's mirrors, so that
    the reference's trainers (`source/training/nerf_trainer.py:112-114`, `joint_pose_nerf_trainer.py:474-477`) and loss
    modules run on the CUDA path without touching the checkout.  Call it once (top of `run_trainval.py`, or a
    `sitecustomize.py`) after the reference checkout is on `sys.path` and BEFORE any `source.training.*` import."""
    import importlib
    import sys

    from . import frequency_nerf, renderer
    sys.modules["source.models.renderer"] = renderer
    sys.modules["source.models.frequency_nerf"] = frequency_nerf
    try:      # also as attributes of the package, for `from source.models import renderer`
        pkg = importlib.import_module("source.models")
        pkg.renderer, pkg.frequency_nerf = renderer, frequency_nerf
    except ImportError:
        pass
