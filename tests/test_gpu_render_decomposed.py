"""stnerf_render as the composition of its unit entry points, bit for bit, and its images against float64 on its own depths.

(a) One stnerf_render call (chunk_rays >= n, so stnerf_debug_read_depths sees the whole call) is restated from the pieces:
    the coarse and fine depths (and, where flow reuse ran, z_new / src_map) are read back; every layer's marched points are
    restated in fp32 op by op (t*d + o, the pass' shift, the scale about the pivot -- skipped in the fine pass under a None
    shift entry -- on the stnerf_rotate_rays copy of a rotated layer's rays); a performer's points go through stnerf_motionnet
    on (p, the frame id of its column) with the lerp decided over the call's hit rays (motion_net.py:53), and one fp32 add;
    stnerf_spacenet_pass(layer, fine) runs on the explicit points and directions (stnerf_spacenet in the render's schedule for
    the pass: in exact_cf the fine pass interleaves the correction products, stnerf_spacenet adds them first in both passes);
    stnerf_composite_pass composites the coarse pass
    (injected uniforms, or the Philox stream of the render's seed) and the fine pass on the read-back depths.  The resampled
    depths, the origin map and every image of both passes (merged and per layer: colour, depth, opacity) must equal the
    render's bit for bit, in all five precisions.  Each unit entry point has its own float64 test (test_gpu_networks_f64,
    test_gpu_composite_pass_f64), so this pins the render's wiring: which point and which ray / time column each network row
    gets, the inverse edit of each pass, hit lists, flow reuse, the fused coarse pass, rotation and hidden layers.
    A chunked call whose later chunk alone holds fractional frame ids must equal the same rays in one chunk.

(b) On the render's own coarse and fine depths, the networks in float64 on float64 points and the float64 compositing of
    tests/composite_pass_restatement.py give the images the render would produce without rounding (placement held fixed,
    DESIGN §4).  `fp32` is held to 2x the error of the same pipeline in torch fp32 on the CPU (plus 1e-6); the tensor-core
    modes to IMAGE_BUDGETS (2x the errors measured on an H100).  With the split emulated on the CPU, losing one Ahi*Wlo stage
    of one layer of the fine background net breaks the `exact` budget.

Measured against float64 on one NVIDIA H100 80GB HBM3 at a 700 W power limit, over the merged and every per-layer image,
absolute, rms / max (MEASURED below has both passes, rounded up; the budgets are twice these).  Fine pass (coarse for
syn_L1_coarse):
  case                 mode     rgb                depth              acc
  syn_L1_coarse        exact    1.3e-07/9.5e-07  6.6e-06/2.6e-05  8.0e-08/4.2e-07
  syn_L1_coarse        exact_cf 1.0e-07/8.4e-07  4.9e-06/2.1e-05  7.3e-08/3.6e-07
  syn_L1_coarse        mixed    1.7e-06/9.7e-06  6.6e-06/2.6e-05  8.0e-08/4.2e-07
  syn_L1_coarse        fast     6.5e-06/5.5e-05  4.3e-04/1.5e-03  2.9e-06/4.4e-05
  syn_L2_64_128        exact    2.3e-07/2.1e-06  5.4e-06/2.6e-05  3.8e-07/3.2e-06
  syn_L2_64_128        exact_cf 2.3e-07/2.1e-06  4.6e-06/2.3e-05  3.7e-07/3.3e-06
  syn_L2_64_128        mixed    2.8e-06/1.1e-05  5.4e-06/2.6e-05  3.8e-07/3.2e-06
  syn_L2_64_128        fast     8.8e-06/6.7e-05  5.6e-04/1.7e-03  1.2e-05/1.1e-04
  tkd_64_128           exact    1.3e-06/3.4e-05  3.2e-06/6.8e-05  4.7e-07/9.6e-06
  tkd_64_128           exact_cf 6.9e-07/9.9e-06  2.2e-06/4.3e-05  3.5e-07/6.1e-06
  tkd_64_128           mixed    2.4e-05/3.2e-04  3.2e-06/6.8e-05  4.7e-07/9.6e-06
  tkd_64_128           fast     4.9e-04/1.1e-02  3.7e-04/7.3e-03  7.5e-05/1.4e-03
  tkd_edit_frac        exact    6.8e-07/1.1e-05  2.2e-06/2.4e-05  3.4e-07/3.9e-06
  tkd_edit_frac        exact_cf 5.5e-07/7.4e-06  1.7e-06/1.4e-05  2.5e-07/2.3e-06
  tkd_edit_frac        mixed    2.5e-05/7.4e-04  2.2e-06/2.4e-05  3.4e-07/3.9e-06
  tkd_edit_frac        fast     1.3e-04/1.6e-03  3.6e-04/4.0e-03  6.3e-05/8.4e-04
  walk_90_30_hide      exact    5.7e-07/3.4e-06  7.3e-06/7.1e-05  1.4e-06/2.3e-05
  walk_90_30_hide      exact_cf 5.7e-07/3.6e-06  6.2e-06/5.2e-05  6.4e-07/1.2e-05
  walk_90_30_hide      mixed    8.8e-06/6.6e-05  7.3e-06/7.1e-05  1.4e-06/2.3e-05
  walk_90_30_hide      fast     2.3e-04/3.7e-03  1.0e-02/1.7e-01  8.5e-04/2.0e-02
  tkd_eval_7col        exact    4.3e-06/1.2e-04  2.3e-06/3.4e-05  3.3e-07/4.7e-06
  tkd_eval_7col        exact_cf 2.8e-06/7.6e-05  1.7e-06/1.8e-05  2.6e-07/2.4e-06
  tkd_eval_7col        mixed    4.3e-05/7.3e-04  2.3e-06/3.4e-05  3.3e-07/4.7e-06
  tkd_eval_7col        fast     7.3e-04/2.0e-02  4.2e-04/6.4e-03  6.5e-05/8.9e-04
  tkd_train_7col_mixed exact    1.5e-06/2.2e-05  3.9e-06/6.7e-05  6.9e-07/1.0e-05
  tkd_train_7col_mixed exact_cf 8.1e-07/9.0e-06  1.9e-06/1.8e-05  3.6e-07/3.1e-06
  tkd_train_7col_mixed mixed    2.5e-05/2.3e-04  3.9e-06/6.7e-05  6.9e-07/1.0e-05
  tkd_train_7col_mixed fast     3.5e-04/6.8e-03  4.0e-04/4.3e-03  1.0e-04/1.2e-03
  walk_L4_64_128       exact    9.2e-07/1.2e-05  1.8e-05/2.8e-04  2.8e-06/5.1e-05
  walk_L4_64_128       exact_cf 6.1e-07/6.3e-06  9.5e-06/1.1e-04  1.3e-06/2.1e-05
  walk_L4_64_128       mixed    8.8e-06/1.4e-04  1.8e-05/2.8e-04  2.8e-06/5.1e-05
  walk_L4_64_128       fast     3.2e-04/6.0e-03  3.6e-03/4.2e-02  4.9e-04/7.6e-03
"""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import cases as C
import composite_pass_restatement as RS
import test_gpu_networks_f64 as NF
from oracle import stnerf_oracle as O
from stnerf_b200 import native as N
from stnerf_b200 import ops
from tests_support import make_cfg

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODES = ("fp32", "exact", "exact_cf", "mixed", "fast")
R_GEN = Rotation.from_rotvec([0.31, -0.52, 0.77]).as_matrix().astype(np.float32)
C_GEN = np.float32([0.13, -0.21, 0.4])

_SYN = dict(weights="synthetic", seed=12, L=2, space_time=True, frame_ids=[0, 10, 11], thr=(0.0, 0.0), ray_seed=2)
# synthetic scenes at the edges of the render path
SYNTH = {
    # n1 = 64: the fused coarse pass; edits with a None shift entry (the fine pass skips that layer's scale), fractional frame
    # ids, near plane, thresholds, alpha on layer 2
    "syn64_edits": dict(_SYN, n1=64, n2=128, n_rays=384, frame_ids=[0, 10.5, 11.25], thr=(0.5, 0.2), near=1.5, alpha=0.4,
                        scale=[1.1, 0.9, 1.2], shift=[[0.5, 0, 0], None, [0, -0.5, 0.25]]),
    # n1 = 32 with 7-column rays of mixed integer frames: the per-ray box table
    "syn32_table": dict(_SYN, n1=32, n2=64, n_rays=320, seven=True, mixed_frames=(3, 60), ray_seed=9,
                        shift=[[0, 0, 0], [0, 0.5, 0], [0, -0.5, 0]], scale=[1, 0.9, 1.2]),
    # n1 = 90 + 30, three performers, one hidden
    "syn90_hidden": dict(_SYN, L=3, n1=90, n2=30, n_rays=320, frame_ids=[0, 30, 31, 32], thr=(2.0, 0.8), near=4.0,
                         hidden=[2], ray_seed=5),
    # n1 + n2 = 256: flow reuse at its last size;  320: reuse off, the generic resampling path
    "syn128_128": dict(_SYN, n1=128, n2=128, n_rays=256, frame_ids=[0, 10.25, 11]),
    "syn128_192": dict(_SYN, n1=128, n2=192, n_rays=256, frame_ids=[0, 10.25, 11]),
    # rotated performers: about the default (box) centre and about an explicit centre, on 9-column rays
    "syn64_rot": dict(_SYN, n1=64, n2=128, n_rays=320, rotation=[None, R_GEN, (R_GEN, C_GEN)]),
    # a performer whose box no ray hits (its box is moved away after the rays were aimed)
    "syn64_miss": dict(_SYN, n1=64, n2=64, n_rays=256, miss=2),
    # one ray, and a few thousand
    "syn64_one": dict(_SYN, n1=64, n2=128, n_rays=160, keep=1),
    "syn90_many": dict(_SYN, n1=90, n2=166, n_rays=3000, frame_ids=[0, 10.5, 11], ray_seed=7),
}
GOLDEN = tuple(C.CASES)


def case_of(name):
    return C.CASES[name] if name in C.CASES else SYNTH[name]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


CHUNK = 4096                     # rays per chunk: more than any case here has, so one call is one chunk (and a small workspace)


def build(name, precision, chunk_rays=CHUNK):
    import modeling
    case = case_of(name)
    sd = C.state_dict_for(case)
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    shift = case.get("shift")
    if case.get("miss"):
        shift = [[0, 0, 0]] * (case["L"] + 1)
        shift[case["miss"]] = [0, 40.0, 0]
    model = modeling.build_layered_model(make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], precision, chunk_rays),
                                         0, case.get("scale"), shift, rotation=case.get("rotation"))
    model.load_state_dict(sd)
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model.near = case.get("near", 0.0)
    model.alpha = case.get("alpha", 1.0)
    for i in case.get("hidden", []):
        model.hide_layer(i)
    return model.cuda(), sd


def inputs(name):
    case = case_of(name)
    rays = C.rays_for(case)
    jit, u = C.uniforms_for(case)
    if u is None:
        u = torch.zeros((case["L"] + 1, rays.shape[0], 0))
    return rays, jit, u


def render(model, name, rays, uni, seed):
    """One stnerf_render call on the model's context (the facade's prologue sets the scene, the box table and the rotation);
    the last `keep` rays only when the case says so.  -> dict of what the render produced and what it read back."""
    case = case_of(name)
    n1, n2 = case["n1"], case["n2"]
    nat, r32 = model._prologue(rays.to(DEV), case["thr"][0], case["thr"][1])
    n = case.get("keep", r32.shape[0])                 # `keep`: the last rays only (aimed at a performer)
    r32 = r32[r32.shape[0] - n:].contiguous()
    jit = u = None
    if uni is not None:
        jit, u = (x[:, x.shape[1] - n:].to(DEV).contiguous() for x in uni)
    out, mask = nat.render(r32, n1, n2, only_coarse=bool(case.get("only_coarse")), jitter=jit, u=u, seed=seed)
    torch.cuda.synchronize()
    l = nat.l
    res = dict(nat=nat, rays=r32, n=n, out=out, mask=mask, jit=jit, u=u, seed=seed, n1=n1, n2=n2, l=l)
    res["t_c"] = torch.stack([nat.read_depths(False, i, n, n1) for i in range(l)])
    if n2 > 0:
        res["t_f"] = torch.stack([nat.read_depths(True, i, n, n1 + n2) for i in range(l)])
    res["reuse"] = model.precision != "fp32" and n2 > 0 and n1 + n2 <= 256
    if res["reuse"]:
        zs = [nat.read_origin(i, n, n1, n2) for i in range(l)]
        res["z_new"], res["src_map"] = torch.stack([z for z, _ in zs]), torch.stack([s for _, s in zs])
    res["rot"] = layer_rotations(model, nat)
    torch.cuda.synchronize()
    return res


def layer_rotations(model, nat):
    """Layer -> (R (3,3) float32, centre (3,) float32) of every rotated layer the render samples rotated (hidden ones are not)."""
    sc = nat._scene
    rot = {}
    for i, e in enumerate(model._rotation_entries()):
        if e is None or (i > 0 and not sc.shown[i]):
            continue
        R, c = e
        if c is None:
            c = (np.float32(list(sc.bmin[i])) + np.float32(list(sc.bmax[i]))) * np.float32(0.5)
        rot[i] = (np.asarray(R, np.float32), np.asarray(c, np.float32))
    return rot


def hit_rows(res, i):
    return torch.arange(res["n"], device=DEV) if i == 0 else torch.nonzero(res["mask"][i]).reshape(-1)


def time_column(scene, i):
    return 6 + (0 if scene.shared_frame_id else i)


def call_lerp(res, i):
    """motion_net.py:53 for the call: any hit ray's frame id of layer i fractional."""
    f = res["rays"][hit_rows(res, i), time_column(res["nat"]._scene, i)]
    return int(bool((torch.floor(f) != f).any()))


def layer_rays(res, i):
    if i in res["rot"]:
        R, c = res["rot"][i]
        return N.rotate_rays(res["rays"], R, c)
    return res["rays"]


# ------------------------------------------------------------------------------------------------------- (a) composition
def compose_nets(res, fine, t):
    """raw (l,n,S,4) of one pass from the unit entry points on depths t (l,n,S)."""
    nat, sc = res["nat"], res["nat"]._scene
    l, n, S = t.shape
    raw = torch.zeros((l, n, S, 4), dtype=torch.float32, device=DEV)
    for i in range(l):
        if i > 0 and not sc.shown[i]:
            continue
        rows = hit_rows(res, i)
        if rows.numel() == 0:
            continue
        r = layer_rays(res, i)[rows]
        p = t[i][rows][..., None] * r[:, None, 3:6] + r[:, None, :3]
        if sc.shift_on[i]:
            p = p - torch.tensor(list(sc.shift[i]), dtype=torch.float32, device=DEV)
        if (sc.scale_fine_on if fine else sc.scale_coarse_on)[i]:
            piv = torch.tensor(list(sc.pivot), dtype=torch.float32, device=DEV)
            p = (p - piv) / torch.tensor(sc.scale[i], dtype=torch.float32, device=DEV) + piv
        p = p.reshape(-1, 3)
        tm = r[:, time_column(sc, i)][:, None].expand(-1, S).reshape(-1, 1).contiguous()
        if i > 0:
            p = p + nat.motionnet(i, torch.cat([p, tm], 1), call_lerp(res, i))
        dirs = r[:, None, 3:6].expand(-1, S, -1).reshape(-1, 3)
        rgb, sig = nat.spacenet(i, fine, p, dirs, tm.reshape(-1), render_schedule=True)
        raw[i, rows] = torch.cat([rgb, sig], 1).reshape(-1, S, 4)
    return raw


def check_composition(res):
    sc, l, n, n1, n2 = res["nat"]._scene, res["l"], res["n"], res["n1"], res["n2"]
    mask = res["mask"]
    raw_c = compose_nets(res, False, res["t_c"])
    cp = ops.composite_pass(sc, res["t_c"], raw_c, mask, fine=False, n2=n2, u=res["u"], seed=res["seed"],
                            want_origin=res["reuse"])
    torch.cuda.synchronize()
    assert _same(cp["images"], res["out"][0]), "coarse images"
    if n2 == 0:
        return
    for i in range(l):
        rows = hit_rows(res, i)
        assert _same(cp["t_fine"][i][rows], res["t_f"][i][rows]), ("t_fine", i)
        if res["reuse"]:
            assert _same(cp["z_new"][i][rows], res["z_new"][i][rows]), ("z_new", i)
            assert torch.equal(cp["src_map"][i][rows], res["src_map"][i][rows]), ("src_map", i)
    t_f = res["t_f"].clone()
    for i in range(1, l):
        t_f[i][mask[i] == 0] = 0.0                   # rows of missed layers are stale in the workspace; no kernel reads them
    raw_f = compose_nets(res, True, t_f)
    fp = ops.composite_pass(sc, t_f, raw_f, mask, fine=True)
    torch.cuda.synchronize()
    assert _same(fp["images"], res["out"][1]), "fine images"


@pytest.mark.parametrize("name", GOLDEN + tuple(SYNTH))
@pytest.mark.parametrize("mode", MODES)
def test_render_is_the_composition(mode, name):
    """Injected uniforms, then the in-kernel Philox draws of a seed: both renders equal their composition bit for bit."""
    model, _ = build(name, mode)
    rays, jit, u = inputs(name)
    for uni, seed in (((jit, u), 5), (None, 77)):
        check_composition(render(model, name, rays, uni, seed))


@pytest.mark.parametrize("mode", ["fp32", "exact"])
def test_lerp_is_decided_per_call_across_chunks(mode):
    """Mixed-frame 7-column rays, chunks of 128: only the last chunk holds fractional frame ids.  The MotionNet lerps for the
    whole call (motion_net.py:53 sees every hit ray of the forward), so the chunked render equals the one-chunk render, and the
    first chunk's images equal a composition that lerps."""
    name = "syn32_table"
    rays, jit, u = inputs(name)
    rays = rays.clone()
    rays[-40:, 6] += 0.5                              # fractional ids in the last chunk only (the box table truncates them)
    one, _ = build(name, mode)
    chunked, _ = build(name, mode, chunk_rays=128)
    a = render(one, name, rays, (jit, u), 3)
    b_nat, r32 = chunked._prologue(rays.to(DEV), 0.0, 0.0)
    b_out, b_mask = b_nat.render(r32, a["n1"], a["n2"], jitter=a["jit"], u=a["u"], seed=3)
    torch.cuda.synchronize()
    assert call_lerp(a, 1) or call_lerp(a, 2)
    assert torch.equal(b_mask, a["mask"])
    assert _same(b_out, a["out"])
    check_composition(a)


def test_spacenet_pass_is_the_render_schedule():
    """stnerf_spacenet_pass is stnerf_spacenet except for exact_cf's fine weights, which run exact's interleaved schedule
    there (the render's fine pass) and the corrections-first schedule in stnerf_spacenet."""
    model, _ = build("syn_L2_64_128", "exact")
    rays, _, _ = inputs("syn_L2_64_128")
    res = render(model, "syn_L2_64_128", rays, None, 9)
    nat = res["nat"]
    g = torch.Generator().manual_seed(3)
    pos = (torch.randn((3001, 3), generator=g) * 1.5).to(DEV)
    dirs = torch.nn.functional.normalize(torch.randn((3001, 3), generator=g), dim=1).to(DEV)
    tm = torch.full((3001,), 10.5, device=DEV)
    outs = {}
    for mode in MODES:
        nat.set_precision(mode)
        for layer in (0, 1):
            for fine in (False, True):
                for sched in (False, True):
                    outs[(mode, layer, fine, sched)] = torch.cat(nat.spacenet(layer, fine, pos, dirs, tm, render_schedule=sched), 1)
    torch.cuda.synchronize()
    for (mode, layer, fine, sched), v in outs.items():
        if not sched:
            continue
        plain = outs[(mode, layer, fine, False)]
        if mode == "exact_cf" and fine:
            assert _same(v, outs[("exact", layer, fine, False)]) and not _same(v, plain), (layer,)
        else:
            assert _same(v, plain), (mode, layer, fine)


# --------------------------------------------------------------------------------------------- (b) images against float64
def scene_dict(sc, l):
    return dict(near=sc.near_plane, alpha2=sc.alpha_layer2, thr_layer=sc.density_threshold, thr_bkgd=sc.bkgd_density_threshold,
                boarder=sc.boarder_weight, apply_thr=bool(sc.apply_thresholds), shown=[bool(sc.shown[i]) for i in range(l)])


def nets_of(sd, L, dtype, device):
    nets = O.split_state_dict(sd, L)
    cast = lambda w: {k: v.to(device, dtype) for k, v in w.items()}  # noqa: E731
    return {"space": [[cast(nets["bkgd"])] + [cast(w) for w in nets["space"]],
                      [cast(nets["bkgd_fine"])] + [cast(w) for w in nets["space_fine"]]],
            "motion": [None] + [cast(w) for w in nets["motion"]]}


def restated_pass(res, nets, fine, dtype, device):
    """One pass in `dtype` on `device` on the render's depths: points (rotation, edit), MotionNet, SpaceNet, compositing.
    -> images (l+1, n, 5)."""
    sc, l = res["nat"]._scene, res["l"]
    mask = res["mask"].to(device).bool()
    t = (res["t_f"] if fine else res["t_c"]).to(device, dtype).clone()
    for i in range(1, l):
        t[i][~mask[i]] = 0.0
    raw = torch.zeros(t.shape + (4,), dtype=dtype, device=device)
    rays = res["rays"].to(device, dtype)
    for i in range(l):
        if i > 0 and not sc.shown[i]:
            continue
        rows = hit_rows(res, i).to(device)
        if rows.numel() == 0:
            continue
        r = rays[rows]
        o, d = r[:, :3], r[:, 3:6]
        if i in res["rot"]:
            R, c = (torch.from_numpy(x).to(device, dtype) for x in res["rot"][i])
            o, d = (o - c) @ R + c, d @ R                  # c + R^T (o - c), R^T d
        S = t.shape[2]
        p = t[i][rows][..., None] * d[:, None] + o[:, None]
        if sc.shift_on[i]:
            p = p - torch.tensor(list(sc.shift[i]), dtype=torch.float32).to(device, dtype)
        if (sc.scale_fine_on if fine else sc.scale_coarse_on)[i]:
            piv = torch.tensor(list(sc.pivot), dtype=torch.float32).to(device, dtype)
            p = (p - piv) / float(np.float32(sc.scale[i])) + piv
        p = p.reshape(-1, 3)
        tm = r[:, time_column(sc, i)][:, None].expand(-1, S).reshape(-1, 1)
        if i > 0:
            p = p + NF.motion_forward(nets["motion"][i], torch.cat([p, tm], 1), bool(call_lerp(res, i)))
        w = nets["space"][int(fine)][i]
        rgb, sig = O.spacenet_forward(w, p, d[:, None].expand(-1, S, -1).reshape(-1, 3), tm if NF.uses_time(w) else None)
        raw[i, rows] = torch.cat([rgb, sig.reshape(-1, 1)], 1).reshape(-1, S, 4)
    return RS.run_pass(scene_dict(sc, l), fine, t.cpu(), raw.cpu(), mask.cpu())["images"]       # the restatement runs on the CPU


def planes(images, n):
    return torch.cat([images[:, :3 * n].reshape(-1, n, 3), images[:, 3 * n:4 * n, None], images[:, 4 * n:, None]], -1)


CHANNELS = (("rgb", slice(0, 3)), ("depth", slice(3, 4)), ("acc", slice(4, 5)))


def image_errors(got):
    """{pass.channel: (rms, max)} over the merged and every per-layer image."""
    e = {}
    for p, (g, tr) in got.items():
        for ch, s in CHANNELS:
            d = g[..., s].to(torch.float64).cpu() - tr[..., s].to(torch.float64).cpu()
            e["%s.%s" % (p, ch)] = (float(d.pow(2).mean().sqrt()), float(d.abs().max()))
    return e


def f64_errors(name, mode):
    """Errors of the render (and, for fp32, of the CPU torch fp32 pipeline) against float64 on the render's own depths, with
    the render's read-back (`res`), the weights and the float64 images.  Nothing is cached: a context holds device workspace."""
    model, sd = build(name, mode)
    rays, jit, u = inputs(name)
    res = render(model, name, rays, (jit, u), 5)
    L, n = res["l"] - 1, res["n"]
    n64 = nets_of(sd, L, torch.float64, DEV)
    passes = ("coarse", "fine") if res["n2"] > 0 else ("coarse",)
    truth = {p: restated_pass(res, n64, p == "fine", torch.float64, DEV) for p in passes}
    got = {p: (planes(res["out"][k], n), truth[p]) for k, p in enumerate(passes)}
    out = {"render": image_errors(got)}
    if mode == "fp32":
        n32 = nets_of(sd, L, torch.float32, "cpu")
        with torch.no_grad():
            yard = {p: (restated_pass(res, n32, p == "fine", torch.float32, "cpu"), truth[p]) for p in passes}
        out["yard"] = image_errors(yard)
    out["res"], out["sd"], out["truth"] = res, sd, truth
    return out


def measured_table():
    """(case, mode) -> {pass.channel: (rms, max)}: the rows IMAGE_BUDGETS is refreshed from (twice these)."""
    return {(name, mode): f64_errors(name, mode)["render"] for name in GOLDEN for mode in MODES[1:]}


# (case, mode) -> {pass.channel: (rms, max)} budget: twice the error measured on an H100 (MEASURED), rounded up.
MEASURED = {
    ("syn_L1_coarse", "exact"): {"coarse.rgb": (1.4e-07, 9.6e-07), "coarse.depth": (6.6e-06, 2.7e-05), "coarse.acc": (8.1e-08, 4.3e-07)},
    ("syn_L1_coarse", "exact_cf"): {"coarse.rgb": (1.1e-07, 8.4e-07), "coarse.depth": (4.9e-06, 2.2e-05), "coarse.acc": (7.4e-08, 3.7e-07)},
    ("syn_L1_coarse", "mixed"): {"coarse.rgb": (1.8e-06, 9.8e-06), "coarse.depth": (6.6e-06, 2.7e-05), "coarse.acc": (8.1e-08, 4.3e-07)},
    ("syn_L1_coarse", "fast"): {"coarse.rgb": (6.5e-06, 5.6e-05), "coarse.depth": (0.00043, 0.0016), "coarse.acc": (2.9e-06, 4.5e-05)},
    ("syn_L2_64_128", "exact"): {"coarse.rgb": (8.6e-08, 6.8e-07), "coarse.depth": (2.7e-06, 1.2e-05), "coarse.acc": (9.2e-08, 9e-07), "fine.rgb": (2.4e-07, 2.1e-06), "fine.depth": (5.4e-06, 2.7e-05), "fine.acc": (3.8e-07, 3.3e-06)},
    ("syn_L2_64_128", "exact_cf"): {"coarse.rgb": (8e-08, 7.3e-07), "coarse.depth": (2.3e-06, 1e-05), "coarse.acc": (8.2e-08, 8.6e-07), "fine.rgb": (2.4e-07, 2.2e-06), "fine.depth": (4.6e-06, 2.4e-05), "fine.acc": (3.8e-07, 3.4e-06)},
    ("syn_L2_64_128", "mixed"): {"coarse.rgb": (2.6e-06, 9.8e-06), "coarse.depth": (2.7e-06, 1.2e-05), "coarse.acc": (9.2e-08, 9e-07), "fine.rgb": (2.8e-06, 1.1e-05), "fine.depth": (5.4e-06, 2.7e-05), "fine.acc": (3.8e-07, 3.3e-06)},
    ("syn_L2_64_128", "fast"): {"coarse.rgb": (6.6e-06, 5.2e-05), "coarse.depth": (0.00013, 0.00054), "coarse.acc": (5.8e-06, 6.9e-05), "fine.rgb": (8.8e-06, 6.8e-05), "fine.depth": (0.00056, 0.0018), "fine.acc": (1.3e-05, 0.00012)},
    ("tkd_64_128", "exact"): {"coarse.rgb": (1.3e-06, 2.8e-05), "coarse.depth": (2.1e-06, 3.5e-05), "coarse.acc": (3.5e-07, 5.1e-06), "fine.rgb": (1.3e-06, 3.5e-05), "fine.depth": (3.2e-06, 6.9e-05), "fine.acc": (4.8e-07, 9.6e-06)},
    ("tkd_64_128", "exact_cf"): {"coarse.rgb": (8e-07, 1.5e-05), "coarse.depth": (1.2e-06, 1.7e-05), "coarse.acc": (2.2e-07, 3.3e-06), "fine.rgb": (6.9e-07, 1e-05), "fine.depth": (2.3e-06, 4.4e-05), "fine.acc": (3.5e-07, 6.1e-06)},
    ("tkd_64_128", "mixed"): {"coarse.rgb": (4.1e-05, 0.00045), "coarse.depth": (2.1e-06, 3.5e-05), "coarse.acc": (3.5e-07, 5.1e-06), "fine.rgb": (2.4e-05, 0.00032), "fine.depth": (3.2e-06, 6.9e-05), "fine.acc": (4.8e-07, 9.6e-06)},
    ("tkd_64_128", "fast"): {"coarse.rgb": (0.00032, 0.009), "coarse.depth": (0.00041, 0.0054), "coarse.acc": (9.6e-05, 0.0017), "fine.rgb": (0.0005, 0.011), "fine.depth": (0.00037, 0.0073), "fine.acc": (7.5e-05, 0.0015)},
    ("tkd_edit_frac", "exact"): {"coarse.rgb": (1.1e-06, 2.5e-05), "coarse.depth": (2.3e-06, 3.4e-05), "coarse.acc": (3.6e-07, 5.5e-06), "fine.rgb": (6.8e-07, 1.1e-05), "fine.depth": (2.3e-06, 2.5e-05), "fine.acc": (3.5e-07, 3.9e-06)},
    ("tkd_edit_frac", "exact_cf"): {"coarse.rgb": (5.6e-07, 1.2e-05), "coarse.depth": (1.6e-06, 3e-05), "coarse.acc": (2.6e-07, 4.9e-06), "fine.rgb": (5.5e-07, 7.4e-06), "fine.depth": (1.7e-06, 1.4e-05), "fine.acc": (2.5e-07, 2.4e-06)},
    ("tkd_edit_frac", "mixed"): {"coarse.rgb": (3e-05, 0.00038), "coarse.depth": (2.3e-06, 3.4e-05), "coarse.acc": (3.6e-07, 5.5e-06), "fine.rgb": (2.6e-05, 0.00074), "fine.depth": (2.3e-06, 2.5e-05), "fine.acc": (3.5e-07, 3.9e-06)},
    ("tkd_edit_frac", "fast"): {"coarse.rgb": (0.00017, 0.0025), "coarse.depth": (0.0007, 0.015), "coarse.acc": (0.00016, 0.0034), "fine.rgb": (0.00014, 0.0016), "fine.depth": (0.00037, 0.0041), "fine.acc": (6.4e-05, 0.00084)},
    ("walk_90_30_hide", "exact"): {"coarse.rgb": (6.7e-07, 1.1e-05), "coarse.depth": (4.1e-06, 3.9e-05), "coarse.acc": (6.3e-07, 1.1e-05), "fine.rgb": (5.7e-07, 3.4e-06), "fine.depth": (7.3e-06, 7.1e-05), "fine.acc": (1.4e-06, 2.4e-05)},
    ("walk_90_30_hide", "exact_cf"): {"coarse.rgb": (4.1e-07, 6.1e-06), "coarse.depth": (2.1e-06, 2.3e-05), "coarse.acc": (3.6e-07, 6.2e-06), "fine.rgb": (5.8e-07, 3.6e-06), "fine.depth": (6.2e-06, 5.3e-05), "fine.acc": (6.5e-07, 1.3e-05)},
    ("walk_90_30_hide", "mixed"): {"coarse.rgb": (7.3e-06, 3.6e-05), "coarse.depth": (4.1e-06, 3.9e-05), "coarse.acc": (6.3e-07, 1.1e-05), "fine.rgb": (8.8e-06, 6.7e-05), "fine.depth": (7.3e-06, 7.1e-05), "fine.acc": (1.4e-06, 2.4e-05)},
    ("walk_90_30_hide", "fast"): {"coarse.rgb": (0.00017, 0.0029), "coarse.depth": (0.0012, 0.02), "coarse.acc": (0.00014, 0.0026), "fine.rgb": (0.00024, 0.0038), "fine.depth": (0.01, 0.18), "fine.acc": (0.00086, 0.021)},
    ("tkd_eval_7col", "exact"): {"coarse.rgb": (1.1e-06, 2e-05), "coarse.depth": (1.5e-05, 0.00033), "coarse.acc": (2.2e-06, 4.7e-05), "fine.rgb": (4.3e-06, 0.00012), "fine.depth": (2.3e-06, 3.4e-05), "fine.acc": (3.4e-07, 4.7e-06)},
    ("tkd_eval_7col", "exact_cf"): {"coarse.rgb": (9e-07, 2.1e-05), "coarse.depth": (1.6e-05, 0.00034), "coarse.acc": (2.2e-06, 5e-05), "fine.rgb": (2.9e-06, 7.7e-05), "fine.depth": (1.7e-06, 1.8e-05), "fine.acc": (2.6e-07, 2.5e-06)},
    ("tkd_eval_7col", "mixed"): {"coarse.rgb": (4.7e-05, 0.00088), "coarse.depth": (1.5e-05, 0.00033), "coarse.acc": (2.2e-06, 4.7e-05), "fine.rgb": (4.4e-05, 0.00073), "fine.depth": (2.3e-06, 3.4e-05), "fine.acc": (3.4e-07, 4.7e-06)},
    ("tkd_eval_7col", "fast"): {"coarse.rgb": (0.00036, 0.0075), "coarse.depth": (0.00098, 0.017), "coarse.acc": (0.00019, 0.0025), "fine.rgb": (0.00074, 0.02), "fine.depth": (0.00043, 0.0064), "fine.acc": (6.5e-05, 0.00089)},
    ("tkd_train_7col_mixed", "exact"): {"coarse.rgb": (1.9e-06, 3.1e-05), "coarse.depth": (3e-06, 5.4e-05), "coarse.acc": (4.7e-07, 8e-06), "fine.rgb": (1.6e-06, 2.2e-05), "fine.depth": (3.9e-06, 6.7e-05), "fine.acc": (7e-07, 1.1e-05)},
    ("tkd_train_7col_mixed", "exact_cf"): {"coarse.rgb": (7.9e-07, 1.1e-05), "coarse.depth": (1.4e-06, 2.1e-05), "coarse.acc": (2.3e-07, 3.1e-06), "fine.rgb": (8.1e-07, 9.1e-06), "fine.depth": (2e-06, 1.9e-05), "fine.acc": (3.7e-07, 3.1e-06)},
    ("tkd_train_7col_mixed", "mixed"): {"coarse.rgb": (3.4e-05, 0.00035), "coarse.depth": (3e-06, 5.4e-05), "coarse.acc": (4.7e-07, 8e-06), "fine.rgb": (2.5e-05, 0.00023), "fine.depth": (3.9e-06, 6.7e-05), "fine.acc": (7e-07, 1.1e-05)},
    ("tkd_train_7col_mixed", "fast"): {"coarse.rgb": (0.00041, 0.0074), "coarse.depth": (0.00055, 0.007), "coarse.acc": (0.00012, 0.0015), "fine.rgb": (0.00036, 0.0069), "fine.depth": (0.0004, 0.0043), "fine.acc": (0.00011, 0.0013)},
    ("walk_L4_64_128", "exact"): {"coarse.rgb": (8.9e-07, 1.5e-05), "coarse.depth": (1.1e-05, 0.00026), "coarse.acc": (1.8e-06, 4.5e-05), "fine.rgb": (9.3e-07, 1.3e-05), "fine.depth": (1.9e-05, 0.00029), "fine.acc": (2.9e-06, 5.2e-05)},
    ("walk_L4_64_128", "exact_cf"): {"coarse.rgb": (4.3e-07, 6.4e-06), "coarse.depth": (4.9e-06, 0.00012), "coarse.acc": (7.7e-07, 2e-05), "fine.rgb": (6.1e-07, 6.3e-06), "fine.depth": (9.6e-06, 0.00012), "fine.acc": (1.4e-06, 2.1e-05)},
    ("walk_L4_64_128", "mixed"): {"coarse.rgb": (8e-06, 4.2e-05), "coarse.depth": (1.1e-05, 0.00026), "coarse.acc": (1.8e-06, 4.5e-05), "fine.rgb": (8.9e-06, 0.00015), "fine.depth": (1.9e-05, 0.00029), "fine.acc": (2.9e-06, 5.2e-05)},
    ("walk_L4_64_128", "fast"): {"coarse.rgb": (0.002, 0.052), "coarse.depth": (0.021, 0.51), "coarse.acc": (0.0037, 0.11), "fine.rgb": (0.00033, 0.0061), "fine.depth": (0.0036, 0.042), "fine.acc": (0.0005, 0.0077)},
}
IMAGE_BUDGETS = {k: {c: (2 * r, 2 * m) for c, (r, m) in v.items()} for k, v in MEASURED.items()}


@pytest.mark.parametrize("name", GOLDEN)
def test_fp32_images_within_twice_the_torch_fp32_error(name):
    e = f64_errors(name, "fp32")
    bad = ["%s: %.3e / %.3e vs torch fp32 %.3e / %.3e" % (c, r, m, e["yard"][c][0], e["yard"][c][1])
           for c, (r, m) in e["render"].items() if r > 2 * e["yard"][c][0] + 1e-6 or m > 4 * e["yard"][c][1] + 1e-6]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", GOLDEN)
@pytest.mark.parametrize("mode", MODES[1:])
def test_tensor_core_images_within_budget(mode, name):
    e = f64_errors(name, mode)["render"]
    b = IMAGE_BUDGETS[(name, mode)]
    bad = ["%s: %.3e / %.3e > %.3e / %.3e" % (c, r, m, b[c][0], b[c][1]) for c, (r, m) in e.items()
           if r > b[c][0] or m > b[c][1]]
    assert not bad, "\n".join(bad)


def _split_linear(drop=None):
    """F.linear with the `exact` split emulated (round-to-nearest fp32 accumulation; 1- and 3-wide heads in fp32); `drop` =
    (weight tensor, k0, k1): that layer's Ahi*Wlo product loses weight columns k0..k1-1 (one 32-k lo stage)."""
    real = torch.nn.functional.linear

    def linear(x, wt, b=None):
        if wt.shape[0] <= 3:
            return real(x, wt, b)
        xh, xl = NF._split(x.clamp(-65504.0, 65504.0))
        wh, wl = NF._split(wt)
        if drop is not None and wt is drop[0]:
            wl = wl.clone()
            wl[:, drop[1]:drop[2]] = 0.0
        acc = real(xh, wh) + real(xl, wh) + real(xh, wl)
        return acc if b is None else acc + b
    return real, linear


def test_exact_budget_separates_a_dropped_lo_stage():
    """On the render's depths of syn_L2_64_128 in `exact`: the fine images of an emulated correct split are within the `exact`
    image budget; with the Ahi*Wlo product of one 32-k stage of stage1.4 of the fine background net dropped, they are not."""
    name = "syn_L2_64_128"
    e = f64_errors(name, "exact")
    res, truth, n = e["res"], e["truth"], e["res"]["n"]
    b = IMAGE_BUDGETS[(name, "exact")]
    over = {}
    for tag in ("ok", "drop"):
        nets = nets_of(e["sd"], res["l"] - 1, torch.float32, "cpu")
        w = nets["space"][1][0]["stage1.4.weight"]
        real, linear = _split_linear(None if tag == "ok" else (w, 0, 32))
        O.F.linear = linear
        try:
            with torch.no_grad():
                img = restated_pass(res, nets, True, torch.float32, "cpu")
        finally:
            O.F.linear = real
        err = image_errors({"fine": (img, truth["fine"])})
        over[tag] = [c for c, (r, m) in err.items() if r > b[c][0] or m > b[c][1]]
    assert not over["ok"], over
    assert over["drop"], over
