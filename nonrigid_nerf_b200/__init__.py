"""nonrigid_nerf_b200 -- H100-native (sm_90a) implementation of NR-NeRF's per-ray volumetric
rendering hot path behind the reference's Python entry points.  See DESIGN.md / INTEGRATION.md."""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
__version__ = "0.1.0"
