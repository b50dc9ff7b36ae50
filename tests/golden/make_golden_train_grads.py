#!/usr/bin/env python
"""Generate tests/golden/train_grads.npz: one training step of the UNMODIFIED reference's LayeredRFRender, on the CPU in
float64 -- `LayeredRFRender.forward` (modeling/layered_rfrender.py:141-734) with injected uniforms, the trainer's loss
(engine/layered_trainer.py:216-281: mse of the coarse and fine images, the REMOVE_OUTLIERS mask losses under their `scalar`
rule, the COARSE_STAGE sum for `only_coarse`), then backward.

Run where the reference tree exists:

    python tests/golden/make_golden_train_grads.py

The model and every input are upcast to float64 (torch's default dtype is float64 while the reference runs, so the zeros it
allocates are float64 too).  Per case of CASES the fixture stores the loss and, per parameter (state_dict order), a seeded
random projection of its gradient, sum(grad * r) with r ~ N(0,1) seeded by the parameter's index (`projection`), plus the
gradient's norm.  tests/test_train_forward.py pins the test-side float64 restatement (tests/train_restatement.py) to them;
tests/test_gpu_train_forward.py then holds the native gradients to float64 on the same cases.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE, os.path.join(ROOT, "st-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases as C  # noqa: E402
from oracle import stnerf_oracle as O  # noqa: E402

# small synthetic cases (synthetic weights and boxes of the shipped shapes), each a layout / feature set of the trainer
CASES = {
    # the trainer's batches: 7-column rays, every ray with its own integer frame id -> boxes per ray (:193), no thresholds
    "mixed7": dict(weights="synthetic", seed=51, L=2, space_time=True, n1=16, n2=16, seven=True, mixed_frames=(3, 60),
                   frame_ids=[10, 10, 10], thr=(1e-4, 0.0), n_rays=48, ray_seed=61,
                   shift=[[0, 0, 0], [0, 0.5, 0], [0, -0.5, 0]], scale=[1, 0.9, 1.2]),
    # retiming rays with fractional frame ids (MotionNet lerp), density thresholds, a scale / shift edit whose shift has a None
    # entry (the fine pass then skips that layer's scale, :468-469), alpha on layer 2, a near plane and a hidden layer
    "retime": dict(weights="synthetic", seed=52, L=2, space_time=True, n1=16, n2=16, frame_ids=[0, 10.5, 11.25],
                   thr=(1e-4, 0.0), n_rays=48, ray_seed=62, shift=[[0, 0, 0], [0, 0.3, 0], None], scale=[1, 0.8, 1.2],
                   alpha=0.5, near=0.5, hidden=[1]),
    # COARSE_STAGE: only_coarse, retiming rays, thresholds
    "coarse": dict(weights="synthetic", seed=53, L=1, space_time=True, n1=16, n2=0, only_coarse=True, frame_ids=[0, 10],
                   thr=(1e-4, 0.0), n_rays=48, ray_seed=63),
}
MASK_SCALAR = 100000.0          # layered_trainer.py:244 `scalar_max`


def case_inputs(name):
    """fp32 rays, jitter (l,N,n1), u (l,N,n2) or None, labels (N,1) int64, target (N,3), state_dict.  name: a key of CASES,
    or a case dict of the same form."""
    case = CASES[name] if isinstance(name, str) else name
    rays = C.rays_for(case)
    jit, u = C.uniforms_for(case)
    g = torch.Generator().manual_seed(700 + case["ray_seed"])
    labels = torch.randint(0, case["L"] + 1, (rays.shape[0], 1), generator=g)
    target = torch.rand((rays.shape[0], 3), generator=g)
    return rays, jit, u, labels, target, C.state_dict_for(case)


def trainer_loss(out, labels, target, only_coarse, n_rays):
    """engine/layered_trainer.py:216-281 (REMOVE_OUTLIERS, epoch < 3) on a 5-tuple; labels (N,1)."""
    stage2, stage1, stage2_layer, stage1_layer, _ = out
    mse = torch.nn.functional.mse_loss
    loss1, loss2 = mse(stage1[0], target), mse(stage2[0], target)
    outliers_1 = torch.cat([stage1_layer[i][2][labels == 0] for i in range(1, len(stage1_layer))], 0)
    outliers_2 = torch.cat([stage2_layer[i][2][labels == 0] for i in range(1, len(stage2_layer))], 0)
    inliers_1 = torch.cat([stage1_layer[i][2][labels == i] for i in range(len(stage1_layer))], 0)
    inliers_2 = torch.cat([stage2_layer[i][2][labels == i] for i in range(len(stage2_layer))], 0)
    m0 = torch.sum(torch.abs(outliers_1)) + torch.sum(torch.abs(1 - inliers_1))
    m1 = torch.sum(torch.abs(outliers_2)) + torch.sum(torch.abs(1 - inliers_2))
    zero = torch.zeros((1,), dtype=target.dtype, device=target.device)
    m0 = m0 / MASK_SCALAR if float(m0.detach()) > n_rays * 0.0005 else zero
    m1 = m1 / MASK_SCALAR if float(m1.detach()) > n_rays * 0.0005 else zero
    return (loss1 + m0) if only_coarse else (loss1 + loss2 + m0 + m1)


def projection(index, shape):
    g = torch.Generator().manual_seed(90000 + index)
    return torch.randn(tuple(shape), generator=g, dtype=torch.float64)


def summarize(grads, keys):
    """grads: key -> gradient (or None) -> (projections, norms) in `keys` order."""
    proj, norm = [], []
    for j, k in enumerate(keys):
        g = grads.get(k)
        g = torch.zeros(1, dtype=torch.float64) if g is None else g.detach().to("cpu", torch.float64)
        proj.append(float((g * projection(j, g.shape)).sum()) if g.numel() > 1 else float(g.sum()))
        norm.append(float(g.norm()))
    return np.array(proj), np.array(norm)


def main():
    from oracle import reference_shim as R
    R.modules()
    out = {}
    for name, case in CASES.items():
        rays, jit, u, labels, target, sd = case_inputs(name)
        bkgd, frames = C.boxes_for(case)
        keys = list(sd)
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)
        try:
            model = R.build_model({k: v.double() for k, v in sd.items()}, case["L"], case["n1"], case["n2"], case["space_time"],
                                  bkgd.double(), frames.double(), case.get("scale"), case.get("shift"))
            model.near = case.get("near", 0.0)
            model.alpha = case.get("alpha", 1.0)
            for i in case.get("hidden", []):
                model.hide_layer(i)
            only_coarse = bool(case.get("only_coarse", False))
            draws = [jit[i].double() for i in range(jit.shape[0])]
            if not only_coarse:
                draws += [u[i].double() for i in range(u.shape[0])]
            with R.cpu_cuda_shim(), R.injected_uniforms(draws):
                res = model(rays.double(), labels, None, only_coarse, density_threshold=case["thr"][0],
                            bkgd_density_threshold=case["thr"][1])
            loss = trainer_loss(res, labels, target.double(), only_coarse, rays.shape[0])
            loss.backward()
            grads = {k: p.grad for k, p in model.named_parameters()}
        finally:
            torch.set_default_dtype(prev)
        proj, norm = summarize(grads, keys)
        out[name + ".loss"] = np.array([float(loss)])
        out[name + ".proj"], out[name + ".norm"] = proj, norm
        out[name + ".keys"] = np.array(keys)
        print("%s: loss %.12g, %d parameters, %d with a gradient" % (name, float(loss), len(keys), int((norm > 0).sum())))
    np.savez_compressed(os.path.join(HERE, "train_grads.npz"), **out)


if __name__ == "__main__":
    main()
