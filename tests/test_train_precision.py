"""The training-precision knob on the host: header enum == Python map, and the knob reaches every network submodule."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_train_precision_enum_matches_python_map():
    from stnerf_b200 import _lib as L
    with open(os.path.join(ROOT, "include", "stnerf.h")) as f:
        hdr = f.read()
    enum = {m.group(1): int(m.group(2)) for m in re.finditer(r"STNERF_TRAIN_(\w+)\s*=\s*(\d+)", hdr)}
    assert enum == {"FP32": 0, "TC_3XTF32": 1}
    assert L.TRAIN_PRECISIONS == {"fp32": enum["FP32"], "tf32x3": enum["TC_3XTF32"]}
    for name in ("stnerf_train_scratch_bytes_prec", "stnerf_spacenet_train_forward_prec", "stnerf_spacenet_backward_prec",
                 "stnerf_motionnet_train_forward_prec", "stnerf_motionnet_backward_prec"):
        assert name in L.EXPORTS and re.search(r"\b%s\s*\(" % name, hdr)


def _networks(model):
    from stnerf_b200 import nets
    return [m for m in model.modules() if isinstance(m, (nets.SpaceNet, nets.MotionNet))]


def _trainable(**kw):
    import modeling
    from tests_support import make_cfg
    cfg = make_cfg(2, 8, 8, True, "fp32")         # 2 performers: 2 + 2 SpaceNets, 2 background SpaceNets, 2 MotionNets
    cfg.MODEL.B200_TRAINABLE = True
    for k, v in kw.items():
        setattr(cfg.MODEL, k, v)
    return cfg, modeling.build_layered_model(cfg, 0)


def test_default_is_fp32():
    from stnerf_b200 import nets
    assert nets.SpaceNet().train_precision == "fp32" and nets.MotionNet(4, input_time=True).train_precision == "fp32"
    _, model = _trainable()
    assert model.train_precision == "fp32"
    assert len(_networks(model)) == 8 and all(m.train_precision == "fp32" for m in _networks(model))


def test_cfg_knob_and_constructor_reach_every_network():
    from stnerf_b200 import nets
    from stnerf_b200.train import TrainableLayeredRFRender
    cfg, model = _trainable(B200_TRAIN_PRECISION="tf32x3")
    assert model.train_precision == "tf32x3"
    assert len(_networks(model)) == 8 and all(m.train_precision == "tf32x3" for m in _networks(model))
    model = TrainableLayeredRFRender(cfg, train_precision="fp32")        # the argument wins over the knob
    assert all(m.train_precision == "fp32" for m in _networks(model))
    d = nets.from_layered(model, train_precision="tf32x3")
    assert len(_networks(d)) == 8 and all(m.train_precision == "tf32x3" for m in _networks(d))
    assert all(m.train_precision == "fp32" for m in _networks(nets.from_layered(model)))


def test_unknown_names_raise():
    from stnerf_b200 import _lib as L
    from stnerf_b200 import nets
    with pytest.raises(ValueError):
        L.train_precision_code("tf32")
    with pytest.raises(ValueError):
        nets.SpaceNet(train_precision="exact")
    with pytest.raises(ValueError):
        nets.MotionNet(4, input_time=True, train_precision="fp16")
    with pytest.raises(ValueError):
        _trainable(B200_TRAIN_PRECISION="bf16")
