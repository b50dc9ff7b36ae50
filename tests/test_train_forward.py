"""Host logic of the trainable LayeredRFRender (stnerf_b200.train), no GPU needed: the facade flag, the parameter and
state_dict layout of the reference module, loading, and the argument checks that run before any kernel."""
import os

import pytest
import torch

import cases as C
from stnerf_b200 import _lib as L
from stnerf_b200.model import LayeredRFRender, fresh_state_dict
from tests_support import make_cfg


def _cfg(L_=2, space_time=True, trainable=None):
    cfg = make_cfg(L_, 64, 128, space_time, "fp32")
    if trainable is not None:
        cfg.MODEL.B200_TRAINABLE = trainable
    return cfg


def test_facade_flag_selects_the_trainable_model():
    import modeling
    from stnerf_b200.train import TrainableLayeredRFRender
    assert type(modeling.build_layered_model(_cfg())) is LayeredRFRender                  # flag absent: default False
    assert type(modeling.build_layered_model(_cfg(trainable=False))) is LayeredRFRender
    m = modeling.build_layered_model(_cfg(trainable=True), 0, [1, 0.8, 1.2], [[0, 0, 0], None, [0, 1, 0]])
    assert isinstance(m, TrainableLayeredRFRender) and isinstance(m, LayeredRFRender)
    assert m.scale == [1, 0.8, 1.2] and m.shift[1] is None


@pytest.mark.parametrize("L_,space_time", [(1, True), (2, True), (2, False), (4, False)])
def test_parameters_and_state_dict_have_the_reference_layout(L_, space_time):
    from stnerf_b200.train import TrainableLayeredRFRender
    m = TrainableLayeredRFRender(_cfg(L_, space_time))
    want = fresh_state_dict(L_, space_time)
    sd = m.state_dict()
    assert list(sd) == list(want)
    assert [tuple(v.shape) for v in sd.values()] == [tuple(v.shape) for v in want.values()]
    assert [k for k, _ in m.named_parameters()] == list(want)
    assert all(p.requires_grad for p in m.parameters())
    # the initial weights are the reference's initialisation, with its clones (spacenets_fine = deepcopy of spacenets)
    assert torch.equal(sd["spacenets_fine.0.stage1.0.weight"], sd["spacenets.0.stage1.0.weight"])
    assert torch.equal(sd["bkgd_spacenet_fine.rgb_net.3.bias"], sd["bkgd_spacenet.rgb_net.3.bias"])


def test_load_state_dict_loads_into_the_submodules():
    from stnerf_b200.train import TrainableLayeredRFRender
    case = C.CASES["syn_L2_64_128"]
    sd = C.state_dict_for(case)
    m = TrainableLayeredRFRender(_cfg())
    m.load_state_dict(sd)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert torch.equal(m.time_deform_nets[1].motion_net[10].bias.detach(), sd["time_deform_nets.1.motion_net.10.bias"])
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if not k.startswith("bkgd_spacenet_fine")})
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad["spacenets.0.stage1.0.weight"] = torch.zeros(3, 3)
        m.load_state_dict(bad)
    m.double().float()                                     # nn.Module.to-style moves act on the parameters
    assert next(m.parameters()).dtype == torch.float32


def test_plain_model_keeps_no_parameters():
    m = LayeredRFRender(_cfg())
    assert list(m.parameters()) == []
    assert list(m.state_dict()) == list(fresh_state_dict(2, True))


def test_cpu_rays_and_bad_width_are_rejected_before_any_kernel():
    from stnerf_b200.train import TrainableLayeredRFRender
    case = C.CASES["syn_L2_64_128"]
    m = TrainableLayeredRFRender(_cfg())
    bkgd, frames = C.boxes_for(case)
    m.set_bkgd_bbox(bkgd)
    m.set_bboxes(frames)
    rays = C.rays_for(case)
    with pytest.raises(L.StnerfError):
        m(rays, None, None)
    with pytest.raises(ValueError):
        m(rays[:, :8], None, None)
    with torch.no_grad(), pytest.raises(L.StnerfError):
        m(rays, None, None)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement of a training step, pinned to the unmodified reference's gradients (tests/golden/train_grads.npz)
# ---------------------------------------------------------------------------------------------------------------------
import make_golden_train_grads as TG  # noqa: E402
import numpy as np  # noqa: E402
import train_restatement as TR  # noqa: E402

TRAIN_GOLDEN = np.load(os.path.join(os.path.dirname(TG.__file__), "train_grads.npz"))
PIN_TOL = 1e-9      # relative to the largest of the case: the same float64 arithmetic in another order


def restated_step(name, dtype=torch.float64, device="cpu"):
    case = TG.CASES[name]
    rays, jit, u, labels, target, sd = TG.case_inputs(name)
    p = {k: v.to(device, dtype).clone().requires_grad_(True) for k, v in sd.items()}
    only_coarse = bool(case.get("only_coarse", False))
    out = TR.forward(p, TR.scene(case, dtype), rays, case["n1"], case["n2"], jit, u, only_coarse, case["thr"][0], case["thr"][1],
                     bool(case.get("seven")), dtype, device)
    loss = TG.trainer_loss(out, labels.to(device), target.to(device, dtype), only_coarse, rays.shape[0])
    loss.backward()
    return loss, {k: v.grad for k, v in p.items()}, list(sd)


@pytest.mark.parametrize("name", list(TG.CASES))
def test_float64_restatement_matches_the_reference_gradients(name):
    loss, grads, keys = restated_step(name)
    assert list(TRAIN_GOLDEN[name + ".keys"]) == keys
    proj, norm = TG.summarize(grads, keys)
    want_p, want_n = TRAIN_GOLDEN[name + ".proj"], TRAIN_GOLDEN[name + ".norm"]
    want_loss = float(TRAIN_GOLDEN[name + ".loss"][0])
    err_l = abs(float(loss) - want_loss) / abs(want_loss)
    assert np.array_equal(norm > 0, want_n > 0), [k for k, a, b in zip(keys, norm, want_n) if (a > 0) != (b > 0)]
    err_p = float(np.abs(proj - want_p).max() / np.abs(want_p).max())
    err_n = float(np.abs(norm - want_n).max() / np.abs(want_n).max())
    print("%s: restatement vs reference: loss %.2e, gradient projections %.2e, norms %.2e (relative)" % (name, err_l, err_p, err_n))
    assert err_l <= PIN_TOL and err_p <= PIN_TOL and err_n <= PIN_TOL, (err_l, err_p, err_n)
