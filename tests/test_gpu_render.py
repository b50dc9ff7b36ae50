"""GPU parity of the full hot path (through the facade -> C ABI) against the reference's golden outputs.

Tolerance (BASELINE.json north_star): pixel RGB within 1e-3 of the reference on identical rays / weights / uniforms.
fp32 and exact (3-term fp16 split on the tensor cores) modes must meet it on every ray; depth is checked relatively
(depths reach ~10 and are sums of w*t)."""
import numpy as np
import pytest
import torch

import cases as C
from tests_support import run_case_native, build_case_model, psnr

pytestmark = pytest.mark.gpu

RGB_TOL = 1e-3


def _check(name, precision, rgb_tol):
    gold = C.load_golden(name)
    got = run_case_native(name, precision=precision)
    if got is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    assert set(got) == set(gold)
    worst = 0.0
    for k in sorted(gold):
        if k.startswith("ray_mask"):
            assert np.array_equal(got[k], gold[k]), k                       # bit-exact: geometry is integer-like
            continue
        err = np.abs(got[k].astype(np.float64) - gold[k])
        if k.endswith("rgb") or k.endswith("acc"):
            worst = max(worst, float(err.max()))
            assert err.max() <= rgb_tol, "%s: max err %.3e (tol %.1e), %d rays over" % (
                k, err.max(), rgb_tol, int((err.max(axis=1) > rgb_tol).sum()))
        else:
            tol = 2e-2 + 2e-3 * np.abs(gold[k])
            assert (err <= tol).all(), "%s: max err %.3e" % (k, err.max())
    return worst


@pytest.mark.parametrize("name", list(C.CASES))
def test_render_fp32_matches_reference(name):
    _check(name, "fp32", RGB_TOL)


@pytest.mark.parametrize("name", list(C.CASES))
def test_render_exact_tc_matches_reference(name):
    _check(name, "exact", RGB_TOL)


@pytest.mark.parametrize("name", list(C.CASES))
def test_render_exact_cf_tc_matches_reference(name):
    """`exact_cf` (STNERF_PREC_TC_3XF16_CF): the correction products of the split go first in the coarse pass and the MotionNets."""
    _check(name, "exact_cf", RGB_TOL)


@pytest.mark.parametrize("name", list(C.CASES))
def test_render_mixed_tc_matches_reference(name):
    """`mixed`: 3-term split wherever the density depends on it, one fp16 pass on the colour-only layer rgb_net.1 -- same 1e-3
    gate on every ray, and the sampling (depths, masks) must be EXACTLY what `exact` produces (the colour branch cannot move a sample)."""
    _check(name, "mixed", RGB_TOL)
    a, b = run_case_native(name, precision="exact"), run_case_native(name, precision="mixed")
    for k in a:
        if k.endswith("depth") or k.endswith("acc") or k.startswith("ray_mask"):
            assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("name", ["syn_L2_64_128", "tkd_64_128"])
def test_render_fast_tc_psnr(name):
    """Single-pass fp16 tensor-core mode: not a parity mode (SURVEY App. C.3); gate on PSNR vs the reference."""
    gold = C.load_golden(name)
    got = run_case_native(name, precision="fast")
    if got is None:
        pytest.skip("checkpoint copy not present")
    assert psnr(got["fine_mixed.rgb"], gold["fine_mixed.rgb"]) > 30.0


def test_chunking_is_not_observable():
    """Same rays through 64-ray internal chunks == one chunk, bit for bit (size-independent property; SURVEY C.6)."""
    a = run_case_native("syn_L2_64_128", precision="exact", chunk_rays=0)
    b = run_case_native("syn_L2_64_128", precision="exact", chunk_rays=64)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_split_call_equals_single_call():
    """Rendering rows [0:n/2) and [n/2:n) in two calls with the sliced uniforms equals one call (rays are independent)."""
    name = "syn_L2_64_128"
    case = C.CASES[name]
    rays = C.rays_for(case)
    jit, u = C.uniforms_for(case)
    full = run_case_native(name, precision="exact")
    h = rays.shape[0] // 2
    lo = run_case_native(name, precision="exact", rays=rays[:h], uniforms=(jit[:, :h].contiguous(), u[:, :h].contiguous()))
    hi = run_case_native(name, precision="exact", rays=rays[h:], uniforms=(jit[:, h:].contiguous(), u[:, h:].contiguous()))
    for k in full:
        assert np.array_equal(full[k], np.concatenate([lo[k], hi[k]], 0)), k


def test_philox_mode_is_sane_and_deterministic():
    """Production RNG path (no injected uniforms): finite, acc in [0,1], identical for the same seed."""
    a = run_case_native("syn_L2_64_128", precision="exact", inject=False)
    b = run_case_native("syn_L2_64_128", precision="exact", inject=False)
    for k in a:
        assert np.isfinite(a[k]).all(), k
        assert np.array_equal(a[k], b[k]), k
    assert a["fine_mixed.acc"].min() >= 0 and a["fine_mixed.acc"].max() <= 1 + 1e-5
    gold = C.load_golden("syn_L2_64_128")
    # different uniforms -> statistically the same picture
    assert psnr(a["fine_mixed.rgb"], gold["fine_mixed.rgb"]) > 20.0


def test_only_coarse_aliases_fine():
    got = run_case_native("syn_L1_coarse", precision="fp32")
    assert np.array_equal(got["fine_mixed.rgb"], got["coarse_mixed.rgb"])


def test_bad_ray_width_is_rejected():
    model = build_case_model("syn_L2_64_128", "fp32")
    with pytest.raises(ValueError):
        model(torch.zeros(8, 8, device="cuda"), None)
    with pytest.raises(Exception):
        model(torch.zeros(8, 9), None)          # CPU tensor: no fallback


def test_large_call_properties():
    """BASELINE-sized sanity at full chunk size: 100k rays of view 0, Philox uniforms; masks agree with the stage op,
    outputs finite, per-layer images are zero exactly where the layer is missed."""
    from stnerf_b200 import ops
    from oracle import stnerf_oracle as O
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "exact")
    K, T = O.synthetic_camera(0, 16, 1080, 1920)
    rays = ops.generate_rays(K, T, 1080, 1920, frame_ids=case["frame_ids"], row0=500, row_step=1, n_rows=60)
    with torch.no_grad():
        out = model(rays, None, None, density_threshold=0.0, bkgd_density_threshold=0.0)
    torch.cuda.synchronize()
    fine_mixed, coarse_mixed, fine_layer, coarse_layer, masks = out
    assert rays.shape[0] == 60 * 1920
    for trip in [fine_mixed, coarse_mixed] + fine_layer + coarse_layer:
        for t in trip:
            assert torch.isfinite(t).all()
    sc = C.scene_for(case)
    for i in range(1, 3):
        _, _, m, _ = ops.intersect_sample(rays, sc["bmin"][i], sc["bmax"][i], 64,
                                          torch.zeros(rays.shape[0], 64, device="cuda"), want_xyz=False)
        assert torch.equal(m, masks[i])
        assert (fine_layer[i][0][~m] == 0).all() and (fine_layer[i][2][~m] == 0).all()
        assert m.any() and not m.all()


def _views_for(model, nat, K, T, frame_ids, seed, thr=(0.0, 0.0)):
    scene = model._resolve_scene(torch.tensor(frame_ids, dtype=torch.float32), thr[0], thr[1])
    return [nat.make_view(K, T, frame_ids, scene, seed)]


def test_row_sharded_render_equals_unsharded():
    """Multi-GPU layout on one device: rendering the rows of rank 0/2 and rank 1/2 separately (in-kernel Philox keyed by
    the global pixel id), each straight into its slot of the gather buffer, equals the unsharded image bit for bit
    (SURVEY section 4, item 3).  H is odd: the last rank's padding row is rendered and discarded."""
    from oracle import stnerf_oracle as O
    from stnerf_b200.dist import ShardedViewRenderer, rows_view
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "exact")
    dev = torch.device("cuda", 0)
    nat = model._ensure_native(dev)
    H, W = 55, 96
    K, T = O.synthetic_camera(2, 16, H, W)
    views = _views_for(model, nat, K, T, case["frame_ids"], seed=5)
    full = ShardedViewRenderer(nat, H, W, 64, 128, 0, 1)
    img = full.assembled(full.render(views)).clone()                    # (1, l+1, H, W, 5)
    assert tuple(img.shape) == (1, 4, H, W, 5)                          # mixed + 3 layer images
    buf = None
    for r in range(2):
        sh = ShardedViewRenderer(nat, H, W, 64, 128, r, 2)
        if buf is not None:
            sh._gather[1] = buf                                           # both "ranks" share one gather buffer: no process group here
        buf = sh.render_local(views)
    both = sh.assembled(rows_view(buf, W))
    assert torch.equal(both, img)
    assert torch.isfinite(img).all() and img[0, 0, ..., 4].max() <= 1 + 1e-5
    # the plane-layout entry point on explicit rays of the same view and seed: same pixels, other layout
    from stnerf_b200 import ops, split_planes
    nat.set_scene(model._resolve_scene(torch.tensor(case["frame_ids"], dtype=torch.float32), 0.0, 0.0))
    rays = ops.generate_rays(K, T, H, W, frame_ids=case["frame_ids"])
    out, _ = nat.render(rays, 64, 128, seed=5)
    fm, _, fl, _ = split_planes(out, 3)
    assert torch.equal(fm[0].reshape(H, W, 3), img[0, 0, ..., :3]) and torch.equal(fl[2][1].reshape(H, W), img[0, 3, ..., 3])


def test_pose_renderer_matches_forward_on_device_rays():
    """SURVEY 8(f) row 1: render_pose fast path (device ray generation + one native call) returns what
    LayeredNeuralRenderer.render_pose derives from layered_batchify_ray on the same rays."""
    import utils
    from oracle import stnerf_oracle as O
    from stnerf_b200 import PoseRenderer, ops
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "exact")
    H, W = 72, 64                                       # 4608 rays >= the 3584-ray chunk: thresholds are forwarded
    K, T = O.synthetic_camera(3, 16, H, W)
    pairs = [(0, 0), (1, 10), (2, 11)]
    pr = PoseRenderer(model, H, W, far=20.0)
    seed0 = model.seed
    color, depth, color_layer, depth_layer = pr.render_pose(T, K, pairs, density_threshold=0.3, bkgd_density_threshold=0.05)
    assert color.shape == (H, W, 3) and depth.shape == (H, W, 1) and len(color_layer) == 3 and depth_layer[2].shape == (H, W, 1)
    # reference flow on the same (device-generated) rays and the same Philox seed
    rays = ops.generate_rays(K, T, H, W, frame_ids=[0, 10, 11])
    model.seed = seed0
    with torch.no_grad():
        stage2, stage1, stage2_layer, stage1_layer, _ = utils.layered_batchify_ray(
            model, rays, torch.zeros(H * W, device="cuda"), None, density_threshold=0.3, bkgd_density_threshold=0.05)
    assert torch.equal(color, stage2[0].reshape(H, W, 3))
    d = stage2[1].reshape(H, W, 1).clone(); d[d < 0] = 0
    assert torch.equal(depth, d / 20.0)
    for i in range(3):
        assert torch.equal(color_layer[i], stage2_layer[i][0].reshape(H, W, 3))
        assert torch.equal(depth_layer[i], stage2_layer[i][1].reshape(H, W, 1) / 20.0)
    # path form: several poses per native call (batch 2 of 3 frames), device->host copies inside the call, CPU tensors
    pr.batch = 2
    seed1 = model.seed
    frames = list(pr.render_path([T, T, T], [K, K, K], [pairs, pairs, pairs], density_threshold=0.3, bkgd_density_threshold=0.05))
    assert len(frames) == 3 and not frames[0][0].is_cuda and frames[1][0].shape == (H, W, 3)
    model.seed = seed1 + 1                               # frame 1 of the path again, alone: same seed -> same pixels
    c1, d1, _, dl1 = pr.render_pose(T, K, pairs, density_threshold=0.3, bkgd_density_threshold=0.05)
    assert torch.equal(frames[1][0], c1.cpu())
    assert float((frames[1][3][2] - dl1[2].cpu()).abs().max()) <= 1e-7      # raw / far: divided on the host here, on the device there
    assert float((frames[1][1] - d1.cpu()).abs().max()) <= 1e-7


def test_render_pose_against_the_oracle():
    """`PoseRenderer.render_pose` against the CPU oracle (pinned to the reference) fed the very uniforms the kernels draw
    (host restatement of the Philox stream): colours within the 1e-3 gate, and the post-processing of
    render/layered_neural_renderer.py:380-390 -- negative mixed depths clamped to 0, everything divided by `far`, the
    per-layer zeroing that tests the ALREADY clamped mixed depth and therefore never fires."""
    from oracle import stnerf_oracle as O
    from stnerf_b200 import PoseRenderer
    from tests_support import philox_draws
    name = "tkd_64_128"
    case = C.CASES[name]
    sd = C.state_dict_for(case)
    if sd is None:
        pytest.skip("checkpoint copy absent")
    H, W, far = 40, 64, 20.0
    K, T = O.synthetic_camera(5, 16, H, W)
    pairs = [(0, 0), (1, 10.5), (2, 11.25)]                 # fractional frame ids: bbox lerp + MotionNet lerp
    ids = [0.0, 10.5, 11.25]
    thr = (0.5, 0.05)
    # tolerances: every pixel but a handful (inverse-CDF resampling is ill-conditioned where the coarse pdf is tiny, so a
    # 1e-6-level difference of a coarse weight can move a fine sample by a visible fraction of its bin; test_gpu_parity_scale.py
    # attributes such pixels one by one) -- at most 0.2 % of the pixels may exceed `tol`, none may exceed 10 x tol
    def close(a, b, tol, what):
        d = (a - b).abs().reshape(-1)
        assert float((d > tol).float().mean()) <= 2e-3 and float(d.max()) < 10 * tol, (what, float(d.max()), float((d > tol).float().mean()))

    for prec, tol in (("fp32", 1e-3), ("exact", 1e-3)):
        model = build_case_model(name, prec)
        model.near = -1.0                                   # no near cut ...
        pr = PoseRenderer(model, H, W, far=far)
        seed = model.seed + 1
        color, depth, color_layer, depth_layer = pr.render_pose(T, K, pairs, density_threshold=thr[0], bkgd_density_threshold=thr[1])
        # the oracle on the same pixels and draws
        rays = torch.cat([O.generate_rays(K, T, H, W), torch.tensor(ids)[None].expand(H * W, -1)], 1)
        jit, u = philox_draws(seed, 3, H * W, case["n1"], case["n2"])
        bkgd, frames = C.boxes_for(case)
        sc = O.resolve_scene(frames, bkgd, ids, None, None)
        sc.update(scale=None, shift=None, shown=[True] * 3, near=-1.0, alpha=1.0, boarder=1e10)
        with torch.no_grad():
            want = O.render(O.split_state_dict(sd, 2), sc, rays, case["n1"], case["n2"], jit, u, density_threshold=thr[0],
                            bkgd_density_threshold=thr[1])
        w_color = want["fine_mixed"][0].reshape(H, W, 3)
        w_depth = want["fine_mixed"][1].reshape(H, W, 1).clone()
        w_depth[w_depth < 0] = 0                                                     # :382
        w_depth = w_depth / far                                                      # :383
        close(color.cpu(), w_color, tol, prec)
        close(depth.cpu(), w_depth, (2e-2 + 2e-3 * 20) / far, prec + " depth")
        assert float(depth.min()) >= 0.0
        for i in range(3):
            wl = want["fine_layer"][i]
            close(color_layer[i].cpu(), wl[0].reshape(H, W, 3), tol, (prec, i))
            d1 = wl[1].reshape(H, W, 1).clone()
            d1[w_depth < 0] = 0                                                      # :387 -- never true after :382
            close(depth_layer[i].cpu(), d1 / far, (2e-2 + 2e-3 * 20) / far, (prec, i, "depth"))
            # rays that miss layer i: exactly zero colour and depth in its image (SURVEY C.6)
            miss = ~want["ray_mask"][i].reshape(H, W)
            assert (color_layer[i].cpu()[miss] == 0).all() and (depth_layer[i].cpu()[miss] == 0).all()
        del model
