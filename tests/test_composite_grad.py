"""Differentiable compositing (stnerf_b200.volume), the parts that need no device: the test-side restatement of
layers/render_layer.py:8-58 and its float64 autograd, pinned to the unmodified reference's own gradients
(tests/golden/composite_grad.npz, make_golden_composite_grads.py), and the absence of a CPU path.
tests/test_gpu_composite_grad.py holds the native backward to this restatement."""
import os

import numpy as np
import pytest
import torch

import make_golden_composite_grads as G
from stnerf_b200 import StnerfError, volume

GOLDEN = np.load(os.path.join(os.path.dirname(G.__file__), "composite_grad.npz"))


def composite_ref(t, rgb, sigma, boarder=1e10):
    """gen_weight + VolumeRenderer.forward (render_layer.py:8-58) in the dtype / on the device of its inputs, for any S >= 1.
    t (N,S), rgb (N,S,3) raw, sigma (N,S) raw -> color (N,3), depth (N,1), acc (N,1), w (N,S)."""
    n = t.shape[0]
    delta = torch.cat([t[:, 1:] - t[:, :-1], torch.full((n, 1), boarder, dtype=t.dtype, device=t.device)], -1)
    alpha = 1.0 - torch.exp(-torch.nn.functional.relu(sigma) * delta)
    trans = torch.cumprod(torch.cat([torch.ones((n, 1), dtype=t.dtype, device=t.device), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    color = torch.sum(torch.sigmoid(rgb) * w[..., None], dim=1)
    depth = torch.sum(w * t, dim=1, keepdim=True)
    acc = torch.sum(w, dim=1, keepdim=True)
    return color, depth, acc, w


def merged_ref(ts, rgbs, sigmas, boarder=1e10, near=None):
    """layered_rfrender.py:425-448 / :587-606 on composite_ref: stable sort of the concatenated depths, gather, near cut."""
    tm, order = torch.sort(torch.cat(ts, 1), dim=1, stable=True)
    rm = torch.cat(rgbs, 1).gather(1, order[..., None].expand(-1, -1, 3))
    sm = torch.cat(sigmas, 1).gather(1, order)
    if near is not None:
        sm = torch.where(tm < near, torch.zeros_like(sm), sm)
    return composite_ref(tm, rm, sm, boarder)[:3]


def projected_loss(outs, proj):
    color, depth, acc, w = outs
    return ((color * proj["color"]).sum() + (depth * proj["depth"]).sum() + (acc * proj["acc"]).sum()
            + (w * proj["w"]).sum())


def golden_case(S):
    """fp32 inputs and float64 projection of one golden sample count."""
    k = "S%d." % S
    t, rgb, sigma = (torch.from_numpy(GOLDEN[k + n]) for n in ("t", "rgb", "sigma"))
    proj = {n: torch.from_numpy(GOLDEN[k + "proj." + n]) for n in ("color", "depth", "acc", "w")}
    return t, rgb, sigma, proj


def ref_grads(t, rgb, sigma, proj, dtype=torch.float64, device="cpu"):
    r = rgb.to(device, dtype).requires_grad_(True)
    s = sigma.to(device, dtype).requires_grad_(True)
    loss = projected_loss(composite_ref(t.to(device, dtype), r, s), {k: v.to(device, dtype) for k, v in proj.items()})
    loss.backward()
    return r.grad, s.grad


@pytest.mark.parametrize("S", G.SAMPLE_COUNTS)
def test_f64_restatement_matches_the_reference_gradients(S):
    t, rgb, sigma, proj = golden_case(S)
    d_rgb, d_sigma = ref_grads(t, rgb, sigma, proj)
    assert torch.isfinite(d_rgb).all() and torch.isfinite(d_sigma).all()
    if S >= 2:
        for got, name in ((d_rgb, "d_rgb"), (d_sigma, "d_sigma")):
            want = torch.from_numpy(GOLDEN["S%d.%s" % (S, name)])
            assert torch.allclose(got, want, rtol=1e-9, atol=1e-12 * float(want.abs().max())), (S, name)
    s = sigma.double().requires_grad_(True)
    (composite_ref(t.double(), torch.zeros(rgb.shape, dtype=torch.float64), s)[3] * proj["w"]).sum().backward()
    want = torch.from_numpy(GOLDEN["S%d.gw_d_sigma" % S])
    assert torch.allclose(s.grad, want, rtol=1e-9, atol=1e-12 * float(want.abs().max())), S


def test_golden_inputs_hold_the_hazards():
    """The fixture exercises what the backward must survive: negative sigma, sigma = 0, an early opaque sample behind which
    the fp32 transmittance underflows to 0, and a tiny positive sigma on the border sample."""
    for S in G.SAMPLE_COUNTS:
        t, rgb, sigma, _ = golden_case(S)
        assert float(sigma[3, -1]) == pytest.approx(1e-9)
        if S > 1:
            assert bool((sigma < 0).any()) and bool((sigma == 0).any())
        if S > 22:
            w = composite_ref(t, rgb, sigma)[3]
            assert float(w[2, 5]) > 0.0 and float(w[2, 22:].abs().max()) == 0.0


def test_cpu_tensors_raise():
    t, rgb, sigma = torch.zeros(2, 4), torch.zeros(2, 4, 3, requires_grad=True), torch.zeros(2, 4)
    with pytest.raises(StnerfError):
        volume.composite(t, rgb, sigma)
    with pytest.raises(StnerfError):
        volume.composite_merged([t, t], [rgb, rgb], [sigma, sigma])
    import layers
    with pytest.raises(StnerfError):
        layers.VolumeRenderer()(t[..., None], rgb, sigma[..., None])
