"""Trainable SpaceNet / MotionNet (stnerf_b200.nets), the parts that need no device: the modules' parameter names and shapes
against the reference's state_dict keys, the configurations that raise, the absence of a CPU path, and the test-side float64
autograd truth pinned to the unmodified reference's own gradients (tests/golden/nets_grad.npz, make_golden_grads.py)."""
import os

import numpy as np
import pytest
import torch

import cases as C
import make_golden_grads as G
from oracle import stnerf_oracle as O
from stnerf_b200 import StnerfError, fresh_state_dict, nets
from stnerf_b200.config import make_cfg

GOLDEN = np.load(os.path.join(os.path.dirname(G.__file__), "nets_grad.npz"))


def _shapes(sd, prefix):
    return {k[len(prefix):]: tuple(v.shape) for k, v in sd.items() if k.startswith(prefix)}


@pytest.mark.parametrize("use_time", [False, True])
def test_module_keys_and_shapes_match_the_reference(use_time):
    sd = fresh_state_dict(1, use_time)
    got = {k: tuple(v.shape) for k, v in nets.SpaceNet(use_time=use_time).state_dict().items()}
    assert list(got) == list(_shapes(sd, "spacenets.0.")) and got == _shapes(sd, "spacenets.0.")
    got = {k: tuple(v.shape) for k, v in nets.MotionNet(c_input=4, input_time=True).state_dict().items()}
    assert list(got) == list(_shapes(sd, "time_deform_nets.0.")) and got == _shapes(sd, "time_deform_nets.0.")


@pytest.mark.parametrize("scene", ["taekwondo", "walking"])
def test_module_keys_match_the_shipped_checkpoint(scene):
    p = C.find_checkpoint(scene)
    if p is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    sd = torch.load(p, map_location="cpu")
    sd = sd["model"] if "model" in sd else sd
    use_time = sd["spacenets.0.rgb_net.1.weight"].shape[1] == 304
    net = nets.SpaceNet(use_time=use_time)
    net.load_state_dict({k[len("spacenets.0."):]: v for k, v in sd.items() if k.startswith("spacenets.0.")})
    mn = nets.MotionNet(c_input=4, input_time=True)
    mn.load_state_dict({k[len("time_deform_nets.0."):]: v for k, v in sd.items() if k.startswith("time_deform_nets.0.")})


def test_unsupported_configurations_raise():
    for kw in ({"deep_rgb": True}, {"use_dir": False}, {"include_input": False}, {"c_pos": 4}):
        with pytest.raises(NotImplementedError):
            nets.SpaceNet(**kw)
    for kw in ({}, {"c_input": 4}, {"input_time": True}, {"c_input": 4, "input_time": True, "include_input": False}):
        with pytest.raises(NotImplementedError):
            nets.MotionNet(**kw)


def test_cpu_tensors_raise():
    sn, mn = nets.SpaceNet(use_time=True), nets.MotionNet(c_input=4, input_time=True)
    pos, rays, t = torch.zeros(4, 3), torch.zeros(4, 6), torch.zeros(4, 1)
    with pytest.raises(StnerfError):
        sn(pos, rays, t)
    with pytest.raises(StnerfError):
        mn(torch.zeros(4, 4))


def test_from_layered_keys_round_trip():
    import modeling
    model = modeling.build_layered_model(make_cfg(2, 64, 128, True))
    d = nets.from_layered(model)
    sd = d.state_dict()
    assert list(sd) == list(model.state_dict())
    for k, v in model.state_dict().items():
        assert torch.equal(sd[k], v), k
    model.load_state_dict(sd)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 autograd truth of the GPU tests against the reference's own gradients
# ---------------------------------------------------------------------------------------------------------------------
def truth_grads(case, device="cpu"):
    """float64 autograd of the oracle's restatement, same weights / points / loss as make_golden_grads.py."""
    w = {k: v.to(device, torch.float64).requires_grad_(True) for k, v in G.weights(case).items()}
    pos, dirs, times = (x.to(device, torch.float64) for x in G.inputs(case))
    proj_out, proj_par = G.projections(case, {k: tuple(v.shape) for k, v in w.items()})
    if G.CASES[case][3] == "space":
        pos.requires_grad_(True)
        outs = O.spacenet_forward(w, pos, dirs, times if G.CASES[case][1] else None)
    else:
        outs = [O.motionnet_forward(w, torch.cat([pos, times], 1))]
    loss = sum((o * r.to(device)).sum() for o, r in zip(outs, proj_out))
    loss.backward()
    return (pos.grad if pos.requires_grad else None), {k: v.grad for k, v in w.items()}, proj_par


@pytest.mark.parametrize("case", list(G.CASES))
def test_f64_autograd_matches_the_reference_gradients(case):
    d_pos, grads, proj = truth_grads(case)
    if d_pos is not None:
        want = torch.from_numpy(GOLDEN[case + ".d_pos"]).double()
        err = (d_pos - want).abs().max() / want.abs().max()
        assert err < 2e-5, (case, float(err))
    for k, g in grads.items():
        n = float(GOLDEN["%s.norm.%s" % (case, k)])
        assert abs(float(g.norm()) - n) <= 1e-5 * n + 1e-12, (case, k, float(g.norm()), n)
        p = float(GOLDEN["%s.proj.%s" % (case, k)])
        scale = n * np.sqrt(g.numel())                          # |proj| <= |g| |r|, |r| ~ sqrt(numel)
        assert abs(float((g * proj[k]).sum()) - p) <= 1e-5 * scale + 1e-12, (case, k)
