"""stnerf_b200 -- H100-native (sm_90a) implementation of the st-nerf layered ray-march hot path.

Python here is plumbing (device memory, streams, torch.distributed); the arithmetic lives in
libstnerf_b200.so (st-nerf_b200/csrc, C ABI in include/stnerf.h).  The sibling packages `modeling`, `utils`,
`layers` and `engine` re-export it under the reference's own import names so reference-side callers
(`render/layered_neural_renderer.py`, `demo/*.py`) run unchanged with `st-nerf_b200/` on sys.path.
"""
from . import _lib
from ._lib import StnerfError
from .model import LayeredRFRender, build_layered_model, fresh_state_dict
from .native import NativeRenderer, launch_count, split_planes
from . import ops
from .pose_renderer import PoseRenderer
from .camera_path import CameraPath
from . import checkpoint_io
from . import nets
from . import volume
from .extract import Mesh, extract_mesh, layer_density, write_ply

__all__ = ["LayeredRFRender", "build_layered_model", "fresh_state_dict", "NativeRenderer", "StnerfError", "ops",
           "launch_count", "split_planes", "PoseRenderer", "CameraPath", "checkpoint_io", "nets", "volume",
           "Mesh", "extract_mesh", "layer_density", "write_ply"]
