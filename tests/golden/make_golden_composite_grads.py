#!/usr/bin/env python
"""Generate tests/golden/composite_grad.npz: gradients of the UNMODIFIED reference's compositing (layers/render_layer.py:8-58,
`VolumeRenderer.forward` and `gen_weight`) under torch.autograd on the CPU, in float64.

Run where the reference tree exists:

    python tests/golden/make_golden_composite_grads.py

Per sample count S in SAMPLE_COUNTS, seeded inputs (t, rgb, sigma) of RAYS rays hold the hazards of the backward: negative
sigma, sigma exactly 0, a ray made opaque early (its transmittance underflows behind), and a tiny positive sigma on the border
sample (delta = 1e10).  The fixture stores, per S:
  S<S>.t / .rgb / .sigma     the fp32 inputs (the reference runs on them upcast to float64);
  S<S>.proj.*                the seeded projection of color / depth / acc / w that makes the loss;
  S<S>.d_rgb / .d_sigma      VolumeRenderer's gradients of that loss, in full (S >= 2: the reference's delta `.squeeze()` drops
                             the border delta of a one-sample ray, so it cannot composite S = 1);
  S<S>.gw_d_sigma            gen_weight's gradient of sum(w * proj.w) with the same deltas (every S, including 1).
tests/test_composite_grad.py pins the test-side float64 restatement and its autograd to these numbers.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SAMPLE_COUNTS = (1, 33, 64, 192)
RAYS = 8
BOARDER = 1e10


def inputs(S):
    """fp32 t (RAYS,S) ascending, rgb (RAYS,S,3), sigma (RAYS,S) with the edge cases placed on fixed rays."""
    g = torch.Generator().manual_seed(1000 + S)
    t = 2.0 + torch.cumsum(torch.rand((RAYS, S), generator=g) * 0.1 + 0.005, 1)
    rgb = torch.randn((RAYS, S, 3), generator=g) * 2.0
    sigma = torch.randn((RAYS, S), generator=g) * 8.0                 # about half negative
    sigma[1, ::3] = 0.0                                                # exactly 0: relu has no gradient there
    sigma[2, 5::4] = 3.0e3                                             # opaque every 4th sample: T underflows to 0 by the 5th
    sigma[3, -1] = 1e-9                                                # border sample, tiny positive: huge finite d_sigma
    sigma[4] = sigma[4].abs() * 30.0                                   # dense ray: every sample absorbs
    return t.float(), rgb.float(), sigma.float()


def projections(S):
    g = torch.Generator().manual_seed(2000 + S)
    return {k: torch.randn(s, generator=g, dtype=torch.float64)
            for k, s in (("color", (RAYS, 3)), ("depth", (RAYS, 1)), ("acc", (RAYS, 1)), ("w", (RAYS, S)))}


def main():
    from oracle import reference_shim as R
    R.modules()
    from layers.render_layer import VolumeRenderer, gen_weight

    out = {}
    for S in SAMPLE_COUNTS:
        t, rgb, sigma = inputs(S)
        proj = projections(S)
        key = "S%d." % S
        out[key + "t"], out[key + "rgb"], out[key + "sigma"] = t.numpy(), rgb.numpy(), sigma.numpy()
        for k, v in proj.items():
            out[key + "proj." + k] = v.numpy()
        t64 = t.double()
        if S >= 2:
            r = rgb.double().requires_grad_(True)
            s = sigma.double()[..., None].requires_grad_(True)
            color, depth, acc, w = VolumeRenderer(boarder_weight=BOARDER)(t64[..., None], r, s)
            loss = ((color * proj["color"]).sum() + (depth * proj["depth"]).sum() + (acc * proj["acc"]).sum()
                    + (w[..., 0] * proj["w"]).sum())
            loss.backward()
            out[key + "d_rgb"], out[key + "d_sigma"] = r.grad.numpy(), s.grad[..., 0].numpy()
        delta = torch.cat([t64[:, 1:] - t64[:, :-1], torch.full((RAYS, 1), BOARDER, dtype=torch.float64)], 1)
        s = sigma.double()[..., None].requires_grad_(True)
        (gen_weight(s, delta) * proj["w"]).sum().backward()
        out[key + "gw_d_sigma"] = s.grad[..., 0].numpy()
    np.savez_compressed(os.path.join(HERE, "composite_grad.npz"), **out)
    print("composite_grad.npz: %d arrays" % len(out))


if __name__ == "__main__":
    main()
