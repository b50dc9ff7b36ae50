"""The drop-in boundary as INTEGRATION.md documents it: `st-nerf_b200/` ahead of the reference root on sys.path.

Executes the EXACT import block of the reference's demos (demo/taekwondo_demo.py:16-23, demo/walking_demo.py:16-24) in a
fresh interpreter with that path order (cwd = reference root, `sys.path.append('.')` as the demos do, PYTHONPATH =
st-nerf_b200) and third-party packages this image lacks (yacs, imageio, matplotlib, kornia) stubbed.  Hot-path names must
come from the native facade, everything else (`engine.layered_trainer`, `config`, `solver`, `utils.metrics`) from the reference
through the facade packages' fall-through (`stnerf_b200/_fallthrough.py`).  A second test builds a miniature fake reference
tree so the mechanism is covered where no reference checkout exists."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "st-nerf_b200")
sys.path.insert(0, ROOT)
from oracle import stash_reference  # noqa: E402

STUBS = textwrap.dedent('''
    import sys, types
    for _m in ("yacs", "yacs.config", "imageio", "matplotlib", "matplotlib.pyplot", "kornia", "kornia.losses", "robopy"):
        sys.modules.setdefault(_m, types.ModuleType(_m))
    class _CN(dict):
        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__
        def merge_from_file(self, f): pass
        def freeze(self): pass
    sys.modules["yacs.config"].CfgNode = _CN
    sys.modules["kornia.losses"].ssim = lambda *a, **k: None
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
''')

CHECK = textwrap.dedent('''
    import os, sys
    import engine, layers, utils, modeling, render, config, solver
    pkg = os.environ["STNERF_TEST_PKG"]; ref = os.path.realpath(os.getcwd())
    here = lambda m: os.path.realpath(sys.modules[m.__module__ if not hasattr(m, "__file__") else m.__name__].__file__)
    # hot-path names: the native facade
    for obj in (make_loss, RaySamplePoint, batchify_ray, vis_density, LayeredNeuralRenderer, setup_logger):
        assert here(obj).startswith(pkg), (obj, here(obj))
    for mod in (engine, layers, utils, modeling, render):
        assert os.path.realpath(mod.__file__).startswith(pkg), mod
    # everything the facade does not replace: the reference's own files
    for obj in (do_train, make_optimizer, WarmupMultiStepLR, build_scheduler):
        assert here(obj).startswith(ref), (obj, here(obj))
    assert os.path.realpath(config.__file__).startswith(ref) and os.path.realpath(solver.__file__).startswith(ref)
    import utils.metrics, layers.camera_transform
    assert os.path.realpath(utils.metrics.__file__).startswith(ref)
    assert os.path.realpath(layers.camera_transform.__file__).startswith(ref)
    print("IMPORT-BLOCK-OK")
''')


def _import_block(path, first, last):
    """Lines first..last (1-based, inclusive) of a demo script, minus its third-party imports handled by the stubs."""
    lines = open(path).read().split("\n")[first - 1:last]
    assert any("from render import LayeredNeuralRenderer" in x for x in lines) and any("from config import cfg" in x for x in lines)
    return "\n".join(lines)


def _run(code, cwd):
    """Run `code` as a SCRIPT (sys.path[0] = the script's directory, like `python demo/taekwondo_demo.py`; `python -c` would
    put the cwd -- the reference root -- first and defeat the documented order)."""
    import tempfile
    env = dict(os.environ, PYTHONPATH=PKG, STNERF_TEST_PKG=os.path.realpath(PKG))
    env.pop("STNERF_REFERENCE_ROOT", None)
    with tempfile.TemporaryDirectory(prefix="stnerf_demo_") as d:
        script = os.path.join(d, "demo_block.py")
        with open(script, "w") as f:
            f.write(code)
        r = subprocess.run([sys.executable, script], cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "IMPORT-BLOCK-OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("demo,first,last,extra", [("taekwondo_demo.py", 16, 23, ""),
                                                   ("walking_demo.py", 16, 24, "assert build_model is modeling.build_layered_model\n")])
def test_reference_demo_import_block(demo, first, last, extra):
    ref = stash_reference.reference_root()
    if ref is None:
        pytest.skip("no reference checkout or archive")
    block = _import_block(os.path.join(ref, "demo", demo), first, last)
    # the demos run from the reference root and extend sys.path themselves (demo/taekwondo_demo.py:15 `sys.path.append('.')`)
    _run(STUBS + "sys.path.append('.')\n" + block + "\n" + CHECK + extra, cwd=ref)


def test_fall_through_on_a_miniature_reference_tree(tmp_path):
    ref = tmp_path / "ref"
    files = {
        "modeling/layered_rfrender.py": "raise RuntimeError('the facade must win')\n",
        "modeling/__init__.py": "raise RuntimeError('the facade must win')\n",
        "utils/__init__.py": "raise RuntimeError('the facade must win')\n",
        "utils/metrics.py": "def psnr(a, b):\n    return 42\n",
        "utils/logger.py": "raise RuntimeError('the facade ships utils.logger')\n",
        "layers/__init__.py": "raise RuntimeError('the facade must win')\n",
        "layers/camera_transform.py": "class CameraTransformer: pass\n",
        "engine/__init__.py": "raise RuntimeError('the facade must win')\n",
        "engine/layered_trainer.py": "from utils import layered_batchify_ray, vis_density, metrics\nfrom utils.metrics import *\ndef do_train(*a): return psnr(0, 0)\n",
        "config/__init__.py": "cfg = {'from': 'reference'}\n",
        "solver/__init__.py": "def make_optimizer(): pass\nclass WarmupMultiStepLR: pass\ndef build_scheduler(): pass\n",
    }
    for rel, body in files.items():
        p = ref / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(body)
    block = textwrap.dedent('''
        from config import cfg
        from engine.layered_trainer import do_train
        from solver import make_optimizer, WarmupMultiStepLR, build_scheduler
        from layers import make_loss
        from utils.logger import setup_logger
        from layers.RaySamplePoint import RaySamplePoint
        from utils import batchify_ray, vis_density
        from render import LayeredNeuralRenderer
        assert do_train() == 42 and cfg == {'from': 'reference'}
    ''')
    _run("import sys\nsys.path.append('.')\n" + block + CHECK, cwd=str(ref))


def test_facade_stands_alone_without_a_reference(tmp_path):
    code = textwrap.dedent('''
        from layers import make_loss, RaySamplePoint, VolumeRenderer
        from layers.RaySamplePoint import RaySamplePoint as R2, intersection
        from utils.logger import setup_logger
        from utils import batchify_ray, vis_density, add_two_dim_dict, Trigonometric_kernel, sample_pdf
        from engine import render as engine_render
        from render import LayeredNeuralRenderer
        from modeling import build_layered_model, build_model
        import utils
        assert len(utils.__path__) == 1 and R2 is RaySamplePoint
        d = {}; add_two_dim_dict(d, 1, 2, 3); assert d == {1: {2: 3}}
        try:
            import engine.layered_trainer
        except ImportError:
            print("IMPORT-BLOCK-OK")
    ''')
    _run(code, cwd=str(tmp_path))
