"""Harness that drives the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE ONLY (see ``oracle/stnerf_oracle.py``).  Used by
``tests/golden/make_golden*.py`` to produce the committed golden vectors, by the
``not gpu`` pinning tests, and -- always in a SEPARATE PROCESS, through
``oracle/run_reference.py`` -- by the ``gpu`` parity-at-scale test and the CPU legs of
``bench.py``.  The reference root is ``/root/reference`` in the build container and the
archive packed by ``oracle/stash_reference.py`` (unpacked outside the repository) on the
GPU box, which has no ``/root/reference``.

Three shims, all harness-side (SURVEY 8c):
  1. ``sys.path`` insert + import of ``modeling`` / ``layers`` / ``utils`` only;
  2. ``torch.Tensor.cuda`` made a no-op while a reference call runs (the
     reference hard-codes ``.cuda()``, modeling/layered_rfrender.py:191,195,207);
  3. ``torch.rand`` replaced by a popper of pre-generated uniforms, in the order
     the reference draws them: jitter for layers 0..L
     (layers/RaySamplePoint.py:98) then u for layers 0..L (utils/sample_pdf.py:31).
"""
from __future__ import annotations

import contextlib
import os
import sys
import types

import torch

try:
    from . import stash_reference as _stash
except ImportError:                                  # imported as a top-level module
    import stash_reference as _stash

REFERENCE_ROOT = _stash.reference_root() or "/root/reference"


def available() -> bool:
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "modeling", "layered_rfrender.py"))


_mods = None


def modules():
    """Import the reference's own packages (torch+numpy only)."""
    global _mods
    if _mods is None:
        if not available():
            raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
        # The facade packages in st-nerf_b200/ reuse the reference's top-level names;
        # the two must never be mixed in one interpreter.
        for name in ("modeling", "layers", "utils", "engine"):
            if name in sys.modules and REFERENCE_ROOT not in (getattr(sys.modules[name], "__file__", "") or ""):
                raise RuntimeError("module %r already imported from the native facade; "
                                   "run reference-driving code in a separate process" % name)
        sys.path.insert(0, REFERENCE_ROOT)
        import io
        with contextlib.redirect_stdout(io.StringIO()):
            import modeling, layers, utils  # noqa: E401
            from layers.RaySamplePoint import intersection  # noqa: F401
            from layers.render_layer import VolumeRenderer, gen_weight  # noqa: F401
            from utils.render_helpers import generate_rays  # noqa: F401
        _mods = types.SimpleNamespace(modeling=modeling, layers=layers, utils=utils)
    return _mods


def make_cfg(layer_num: int, n1: int, n2: int, use_space_time: bool):
    """The 15 fields LayeredRFRender.__init__ reads (modeling/layered_rfrender.py:23-37)."""
    M = types.SimpleNamespace(
        BOARDER_WEIGHT=1e10, SAMPLE_METHOD="BBOX", SAME_SPACENET=False, TKERNEL_INC_RAW=True,
        POSE_REFINEMENT=False, USE_DIR=True, USE_DEFORM_VIEW=False, USE_DEFORM_TIME=True,
        USE_SPACE_TIME=use_space_time, BKGD_USE_DEFORM_TIME=False, BKGD_USE_SPACE_TIME=False,
        DEEP_RGB=False, COARSE_RAY_SAMPLING=n1, FINE_RAY_SAMPLING=n2)
    return types.SimpleNamespace(MODEL=M, DATASETS=types.SimpleNamespace(LAYER_NUM=layer_num))


@contextlib.contextmanager
def cpu_cuda_shim():
    had = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = had


@contextlib.contextmanager
def injected_uniforms(draws):
    """Replace torch.rand by a popper over ``draws`` (list of tensors)."""
    real = torch.rand
    queue = list(draws)

    def fake(*size, **kw):
        t = queue.pop(0)
        shape = tuple(size[0]) if len(size) == 1 and not isinstance(size[0], int) else tuple(size)
        assert tuple(t.shape) == tuple(shape), (t.shape, shape)
        return t.clone()

    torch.rand = fake
    try:
        yield
    finally:
        torch.rand = real


def build_model(state_dict, layer_num, n1, n2, use_space_time, bkgd_bbox, bboxes, scale=None, shift=None):
    import io
    m = modules()
    with contextlib.redirect_stdout(io.StringIO()):
        model = m.modeling.build_layered_model(make_cfg(layer_num, n1, n2, use_space_time), 0, scale, shift)
    model.load_state_dict(state_dict)
    model.set_bkgd_bbox(bkgd_bbox)
    model.set_bboxes(bboxes)
    model.eval()
    return model


def forward(model, rays, jitter, u, only_coarse=False, density_threshold=1e-4, bkgd_density_threshold=0.0):
    """Run LayeredRFRender.forward with injected uniforms; returns the reference 5-tuple."""
    draws = [jitter[i] for i in range(jitter.shape[0])]
    if not only_coarse:
        draws += [u[i] for i in range(u.shape[0])]
    labels = torch.zeros(rays.shape[0])
    with torch.no_grad(), cpu_cuda_shim(), injected_uniforms(draws):
        return model(rays, labels, None, only_coarse=only_coarse, density_threshold=density_threshold,
                     bkgd_density_threshold=bkgd_density_threshold)


def load_checkpoint(scene: str):
    path = os.path.join(REFERENCE_ROOT, "outputs", scene, "layered_rfnr_checkpoint_1.pt")
    if not os.path.isfile(path):
        path = os.path.join(_stash.CKPT, scene + ".pt")
    return torch.load(path, map_location="cpu")["model"]
