#!/usr/bin/env python
"""Generate tests/golden/nets_grad.npz: gradients of the UNMODIFIED reference's SpaceNet / MotionNet under torch.autograd (CPU).

Run where the reference tree exists:

    python tests/golden/make_golden_grads.py

For seeded synthetic weights with and without a time input, the reference modules (modeling/spacenet.py, modeling/motion_net.py)
run forward on GRAD_POINTS seeded points, the loss is a seeded random projection of their outputs, and the fixture stores
  <case>.d_pos            the gradient of the loss with respect to the SpaceNet's positions, in full;
  <case>.norm.<param>     the gradient norm of every parameter tensor;
  <case>.proj.<param>     the gradient's projection onto a seeded random tensor of the parameter's shape.
MotionNet runs once with integer and once with fractional times (the lerped encoding, motion_net.py:53-63).
tests/test_nets_grad_golden.py checks the test-side float64 autograd of the oracle's restatement against these numbers.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases as C  # noqa: E402

GRAD_POINTS = 256
# case -> (state_dict seed, use_time, network prefix, network kind)
CASES = {
    "space_t": (31, True, "spacenets.0.", "space"),
    "space": (32, False, "bkgd_spacenet.", "space"),
    "motion_int": (31, True, "time_deform_nets.0.", "motion"),
    "motion_frac": (31, True, "time_deform_nets.0.", "motion"),
}


def weights(case):
    seed, use_time, prefix, _ = CASES[case]
    sd = C.O.synthetic_state_dict(1, use_time, seed=seed)
    return {k[len(prefix):]: v.clone() for k, v in sd.items() if k.startswith(prefix)}


def inputs(case):
    """pos (P,3), dirs (P,3), times (P,1): Gaussian positions with a few far ones, unit directions, times per case."""
    g = torch.Generator().manual_seed(4321)
    pos = torch.randn((GRAD_POINTS, 3), generator=g) * 1.5
    pos[:16] *= 40.0
    dirs = torch.randn((GRAD_POINTS, 3), generator=g)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    times = torch.randint(0, 100, (GRAD_POINTS, 1), generator=g).float()
    if case == "motion_frac":
        times = times + torch.rand((GRAD_POINTS, 1), generator=g)
    return pos, dirs, times


def projections(case, shapes):
    """Seeded random tensors: one per output (rgb, sigma or flow) for the loss, one per parameter for the projection."""
    g = torch.Generator().manual_seed(777)
    outs = [torch.randn((GRAD_POINTS, 3), generator=g, dtype=torch.float64)]
    if CASES[case][3] == "space":
        outs.append(torch.randn((GRAD_POINTS, 1), generator=g, dtype=torch.float64))
    params = {k: torch.randn(s, generator=g, dtype=torch.float64) for k, s in shapes.items()}
    return outs, params


def main():
    from oracle import reference_shim as R
    R.modules()
    from modeling.spacenet import SpaceNet
    from modeling.motion_net import MotionNet

    out = {}
    for case, (_, use_time, _, kind) in CASES.items():
        w = weights(case)
        pos, dirs, times = inputs(case)
        if kind == "space":
            net = SpaceNet(include_input=True, use_dir=True, use_time=use_time)
            net.load_state_dict(w)
            pos = pos.clone().requires_grad_(True)
            rgb, sigma = net(pos, torch.cat([pos.detach(), dirs], 1), times)
            outs = [rgb, sigma]
        else:
            net = MotionNet(include_input=True, c_input=4, input_time=True)
            net.load_state_dict(w)
            outs = [net(torch.cat([pos, times], 1))]
        proj_out, proj_par = projections(case, {k: tuple(v.shape) for k, v in w.items()})
        loss = sum((o.double() * r).sum() for o, r in zip(outs, proj_out))
        loss.backward()
        if kind == "space":
            out[case + ".d_pos"] = pos.grad.numpy()
        for k, p in net.named_parameters():
            gd = p.grad.double()
            out["%s.norm.%s" % (case, k)] = np.float64(gd.norm())
            out["%s.proj.%s" % (case, k)] = np.float64((gd * proj_par[k]).sum())
    np.savez_compressed(os.path.join(HERE, "nets_grad.npz"), **out)
    print("nets_grad.npz: %d arrays" % len(out))


if __name__ == "__main__":
    main()
