"""GPU tests of the reference-named call surface (SURVEY 8b): engine.render.render, utils.batchify_ray,
utils.layered_batchify_ray, utils.ray_sampling / generate_rays, walking_demo's `build_model` alias."""
import numpy as np
import pytest
import torch

import cases as C
from oracle import stnerf_oracle as O
from tests_support import build_case_model

pytestmark = pytest.mark.gpu


def test_engine_render_returns_reference_shapes_and_matches_forward():
    import engine
    from stnerf_b200 import ops
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "exact")
    H, W = 40, 96                                     # 3840 rays >= 3584: thresholds forwarded like render_pose
    K, T = O.synthetic_camera(5, 16, H, W)
    seed0 = model.seed
    stage2, stage1 = engine.render(model, K, T, (H, W), frame_ids=case["frame_ids"], density_threshold=0.2,
                                   bkgd_density_threshold=0.05)
    assert [tuple(t.shape) for t in stage2] == [(H, W, 3), (H, W), (H, W)]
    assert [tuple(t.shape) for t in stage1] == [(H, W, 3), (H, W), (H, W)]
    rays = ops.generate_rays(K, T, H, W, frame_ids=case["frame_ids"])
    model.seed = seed0
    with torch.no_grad():
        out = model(rays, None, None, density_threshold=0.2, bkgd_density_threshold=0.05)
    assert torch.equal(stage2[0], out[0][0].reshape(H, W, 3))
    assert torch.equal(stage1[2], out[1][2].reshape(H, W))
    # ROI: pixels outside stay zero, pixels inside equal the full render (rays are independent; Philox ids differ -> inject)
    roi = (8, 16, 20, 40)
    s2r, _ = engine.render(model, K, T, (H, W), ROI=roi, frame_ids=case["frame_ids"], only_coarse=True)
    m = torch.zeros(H, W, dtype=torch.bool)
    m[roi[0]:roi[0] + roi[2], roi[1]:roi[1] + roi[3]] = True
    assert (s2r[0][~m.cuda()] == 0).all() and s2r[0][m.cuda()].abs().sum() > 0


def test_batchify_facades():
    import utils
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "exact")
    rays = C.rays_for(case).cuda()
    labels = torch.zeros(rays.shape[0], device="cuda")
    model.seed = 7
    five = utils.layered_batchify_ray(model, rays, labels, None, density_threshold=20, bkgd_density_threshold=0.8)
    model.seed = 7
    direct = model(rays, labels, None)                # N < chunks: the facade must NOT have forwarded the thresholds
    assert torch.equal(five[0][0], direct[0][0]) and len(five[2]) == 3 and five[4][1].dtype == torch.bool
    model.seed = 7
    three = utils.batchify_ray(model, rays, None)
    assert len(three) == 3 and torch.equal(three[0][0], direct[0][0]) and torch.equal(three[2], direct[4][0])


def test_ray_sampling_facade_with_mask():
    import utils
    H, W = 24, 40
    Kt, Tt = C.function_inputs()["rays.K"], C.function_inputs()["rays.T"]
    full, _ = utils.ray_sampling(Kt[None], Tt[None], (H, W))
    want = C.load_golden("functions")["rays.rays"]
    assert np.abs(full.cpu().numpy() - want).max() < 2e-6
    mask = torch.zeros(1, H, W); mask[0, 3:9, 5:25] = 1
    sub, _ = utils.ray_sampling(Kt[None], Tt[None], (H, W), masks=mask)
    assert sub.shape == (6 * 20, 6)
    assert torch.equal(sub, full.reshape(H, W, 6)[3:9, 5:25].reshape(-1, 6))
    rays, rmask = utils.generate_rays(Kt, Tt, None, H, W)
    assert torch.equal(rays, full) and rmask.shape == (H, W, 1)


def test_walking_demo_import_alias():
    import modeling
    from tests_support import make_cfg
    m = modeling.build_model(make_cfg(2, 64, 128, False))       # demo/walking_demo.py:18 imports this name
    assert m.state_dict()["spacenets.0.rgb_net.1.weight"].shape == (128, 283)


def test_example_demo_runs(tmp_path):
    """The scripted edit sessions of demo/taekwondo_demo.py on the native path (tiny size)."""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "examples", "taekwondo_demo_b200.py"), "--size", "96x54",
                        "--steps", "3"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
    assert r.stdout.count("frames of 96x54") == 3
