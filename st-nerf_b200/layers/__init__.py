"""Reference import name `layers` (layers/__init__.py:1-3): per-stage operators on the native kernels.

Submodules that exist here (`RaySamplePoint`, `render_layer`, `loss`) replace the reference's; any other `layers.<name>`
(e.g. `layers.camera_transform`) falls through to the reference tree when one is on sys.path (stnerf_b200/_fallthrough.py)."""
from stnerf_b200 import _fallthrough

_fallthrough.extend("layers", __path__)

from .RaySamplePoint import RaySamplePoint, RaySamplePoint_Near_Far  # noqa: E402
from .render_layer import VolumeRenderer  # noqa: E402
from .loss import make_loss  # noqa: E402

__all__ = ["RaySamplePoint", "RaySamplePoint_Near_Far", "VolumeRenderer", "make_loss"]
