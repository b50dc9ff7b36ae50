"""Geometry extraction on the device: stnerf_layer_field / stnerf_layer_grid are the render's field, and marching cubes.

The field: bit for bit a torch composition of the edit + stnerf_motionnet + an fp32 add + stnerf_spacenet (every precision,
coarse and fine nets, background and performer, integer and fractional frames, edits on / off / with a None shift entry);
layer_grid bit for bit layer_field on the grid's points (odd shapes, chunk boundaries); against TrainableLayeredRFRender's
own fp32 sigma of the samples it drew (through its `trace` hook); against float64 within test_gpu_networks_f64's budgets.
Marching cubes: analytic and random fields against the float64 restatement of tests/mc_restatement.py, closedness, Euler
characteristic, volume, vertex placement, empty / full grids, repeatability.  End to end: the taekwondo performer's mesh
(when its checkpoint copy is present) and extract_mesh after an Adam step."""
import math

import numpy as np
import pytest
import torch

import cases as C
import mc_restatement as M
import test_gpu_networks_f64 as NF
from oracle import stnerf_oracle as O
from stnerf_b200 import extract as X
from stnerf_b200 import native as N
from tests_support import make_cfg

pytestmark = pytest.mark.gpu

DEV = "cuda"
SYN = C.CASES["syn_L2_64_128"]
EDITS = {
    "none": {},
    "scale_shift": dict(scale=[1, 0.75, 1.5], shift=[[0, 0, 0], [0, 0.3, 0], [0, -0.3, 0]]),
    "none_shift": dict(scale=[1.1, 0.9, 1.2], shift=[[0.5, 0, 0], None, [0, -0.5, 0.25]]),
}
MODES = ("fp32", "exact", "exact_cf", "mixed")


def _model(case, precision, trainable=False, sd=None):
    import modeling
    cfg = make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], precision)
    cfg.MODEL.B200_TRAINABLE = trainable
    model = modeling.build_layered_model(cfg, 0, case.get("scale"), case.get("shift"))
    model.load_state_dict(C.state_dict_for(case) if sd is None else sd)
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    return model.cuda()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _points(scene, layer, n, seed):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(scene.bmin[layer]), torch.tensor(scene.bmax[layer])
    xyz = lo + (hi - lo) * (torch.rand((n, 3), generator=g) * 1.2 - 0.1)
    d = torch.randn((n, 3), generator=g)
    return xyz.to(DEV), (d / d.norm(dim=1, keepdim=True)).to(DEV)


def _composition(nat, scene, layer, fine, frame, xyz, dirs):
    """The field restated on the per-point entry points: edit in torch fp32, stnerf_motionnet, fp32 add, stnerf_spacenet."""
    p = xyz.clone()
    if scene.shift_on[layer]:
        p = p - torch.tensor(list(scene.shift[layer]), dtype=torch.float32, device=DEV)
    if (scene.scale_fine_on if fine else scene.scale_coarse_on)[layer]:
        piv = torch.tensor(list(scene.pivot), dtype=torch.float32, device=DEV)
        p = (p - piv) / torch.tensor(scene.scale[layer], dtype=torch.float32, device=DEV) + piv
    t = torch.full((p.shape[0], 1), frame, dtype=torch.float32, device=DEV)
    if layer > 0:
        flow = nat.motionnet(layer, torch.cat([p, t], 1), 1 if math.floor(frame) != frame else 0)
        p = p + flow
    rgb, sig = nat.spacenet(layer, fine, p, dirs, t)
    return rgb, sig.reshape(-1)


@pytest.mark.parametrize("edit", sorted(EDITS))
@pytest.mark.parametrize("mode", MODES)
def test_field_is_the_composition(mode, edit):
    case = dict(SYN, **EDITS[edit])
    model = _model(case, mode)
    for frame in (10.0, 10.5):
        nat, scene = X._scene_at(model, frame)
        for layer in range(case["L"] + 1):
            for fine in (False, True):
                xyz, dirs = _points(scene, layer, 3001, seed=layer * 7 + fine)
                rgb, sig = nat.layer_field(layer, fine, frame, xyz, dirs)
                want_rgb, want_sig = _composition(nat, scene, layer, fine, frame, xyz, dirs)
                assert _same(sig, want_sig) and _same(rgb, want_rgb), (frame, layer, fine)
                _, sig_only = nat.layer_field(layer, fine, frame, xyz, None, want_rgb=False)
                assert _same(sig_only, sig)


@pytest.mark.parametrize("dims", [(2, 2, 2), (2, 9, 17), (33, 2, 5), (7, 129, 65), (130, 90, 91)])
@pytest.mark.parametrize("mode", ["fp32", "exact"])
def test_grid_is_the_field_on_its_points(mode, dims):
    """(130, 90, 91) = 1 064 700 points: more than one 2^20-point chunk."""
    case = dict(SYN, **EDITS["none_shift"])
    model = _model(case, mode)
    frame = 10.5
    nat, scene = X._scene_at(model, frame)
    lo, hi = X.layer_box(model, 1, frame)
    origin, step, _ = X._grid(lo, hi, dims)
    for layer in (0, 1):
        grid = nat.layer_grid(layer, True, frame, origin, step, dims)
        ax = [torch.tensor(origin[a], dtype=torch.float32) + torch.arange(dims[a], dtype=torch.float32) *
              torch.tensor(step[a], dtype=torch.float32) for a in range(3)]
        pts = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3).to(DEV)
        _, sig = nat.layer_field(layer, True, frame, pts, None, want_rgb=False)
        assert _same(grid.reshape(-1), sig), (layer, dims)


def test_field_validation():
    import ctypes
    from stnerf_b200 import _lib as L
    model = _model(SYN, "fp32")
    nat, _ = X._scene_at(model, 10.0)
    lib, s = L.lib(), L.stream_ptr()
    x = torch.zeros((4, 3), device=DEV)
    out = torch.zeros(4, device=DEV)
    assert lib.stnerf_layer_field(nat._h, 3, 1, 10.0, L.ptr(x), None, 4, None, L.ptr(out), s) == -1
    assert lib.stnerf_layer_field(nat._h, -1, 1, 10.0, L.ptr(x), None, 4, None, L.ptr(out), s) == -1
    assert lib.stnerf_layer_field(nat._h, 1, 1, float("nan"), L.ptr(x), None, 4, None, L.ptr(out), s) == -1
    assert lib.stnerf_layer_field(nat._h, 1, 1, 10.0, None, None, 0, None, None, s) == 0
    g = N.make_grid((0, 0, 0), (0.1, 0.1, 0.1), (1, 4, 4))
    assert lib.stnerf_layer_grid(nat._h, 1, 1, 10.0, ctypes.byref(g), L.ptr(out), s) == -1
    g = N.make_grid((0, 0, 0), (0.1, float("inf"), 0.1), (2, 2, 2))
    assert lib.stnerf_layer_grid(nat._h, 1, 1, 10.0, ctypes.byref(g), L.ptr(out), s) == -1
    empty = N.NativeRenderer(3, [True, True, True], "fp32")
    empty.set_scene(X._scene(model, 10.0))
    assert lib.stnerf_layer_field(empty._h, 1, 1, 10.0, L.ptr(x), None, 4, None, L.ptr(out), s) == -4
    g = N.make_grid((0, 0, 0), (0.1, 0.1, 0.1), (2, 2, 2))
    assert lib.stnerf_layer_grid(empty._h, 0, 0, 10.0, ctypes.byref(g), L.ptr(out), s) == -4
    torch.cuda.synchronize()


@pytest.mark.parametrize("frame", [10.0, 10.5])
@pytest.mark.parametrize("edit", ["none", "none_shift"])
def test_field_matches_the_trainable_render(edit, frame):
    """fp32, under grad, 7-column rays with a shared frame id: the sigma the training forward computed for every sample equals
    stnerf_layer_field at the sample's world point o + t*d (coarse and fine pass)."""
    case = dict(SYN, **EDITS[edit], seven=True, frame_ids=[frame] * 3, n_rays=96)
    model = _model(case, "fp32", trainable=True)
    seen = {}
    model.trace = lambda name, x: seen.__setitem__(name, x.detach().clone())
    rays = C.rays_for(case).to(DEV)
    rays[:, 6] = frame
    with torch.enable_grad():
        model(rays, torch.zeros(rays.shape[0], device=DEV), None, density_threshold=0.0, bkgd_density_threshold=0.0)
    model.trace = None
    nat, _ = X._scene_at(model, frame)
    o, d = rays[:, :3], rays[:, 3:6]
    checked = 0
    for layer in range(case["L"] + 1):
        idx = torch.arange(rays.shape[0], device=DEV) if layer == 0 else torch.nonzero(seen["mask"][layer]).reshape(-1)
        for p, t in (("c", seen["t_coarse"][layer]), ("f", seen["t_fine.%d" % layer])):
            t = t[idx]
            xyz = (t[:, :, None] * d[idx][:, None, :] + o[idx][:, None, :]).reshape(-1, 3)
            dirs = d[idx][:, None, :].expand(-1, t.shape[1], -1).reshape(-1, 3)
            rgb, sig = nat.layer_field(layer, p == "f", frame, xyz, dirs)
            assert _same(sig, seen["sigma.%s%d" % (p, layer)].reshape(-1)), (layer, p)
            assert _same(rgb, seen["rgb.%s%d" % (p, layer)]), (layer, p)
            checked += sig.numel()
    assert checked > 10000


@pytest.mark.parametrize("tag", ["syn_t", "syn", "tkd", "walk"])
def test_field_against_float64(tag):
    """Grid points of the performer's box at an integer and a fractional frame: the MotionNet flow and the sigma at the
    deformed point within the budgets of test_gpu_networks_f64 (fp32 and mixed are held to `exact`'s)."""
    sd = NF.state_dict(tag)
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    nets = O.split_state_dict(sd, 1)
    case = dict(weights="synthetic", L=1, space_time=NF.uses_time(nets["space"][0]), n1=64, n2=128)
    for mode in MODES:
        model = _model(case, mode, sd=sd)
        for frame in (10.0, 37.25):
            nat, _ = X._scene_at(model, frame)
            lo, hi = X.layer_box(model, 1, frame)
            origin, step, dims = X._grid(lo, hi, 24)
            ax = [torch.tensor(origin[a]) + torch.arange(dims[a], dtype=torch.float32) * torch.tensor(step[a]) for a in range(3)]
            pts = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3).to(DEV)
            sig = nat.layer_grid(1, True, frame, origin, step, dims).reshape(-1)
            t = torch.full((pts.shape[0], 1), frame, device=DEV)
            lerp = math.floor(frame) != frame
            flow = nat.motionnet(1, torch.cat([pts, t], 1), int(lerp))
            flow64 = NF.motion_forward(NF.to64(nets["motion"][0], DEV), torch.cat([pts, t], 1).double(), lerp)
            deformed = pts + flow
            rgb64, sig64 = NF.space_truth(NF.to64(nets["space_fine"][0], DEV), deformed, torch.zeros_like(deformed), t)
            e = NF.space_errors(torch.zeros_like(rgb64), sig, (rgb64, sig64))
            ef = NF.flow_errors(flow, flow64)
            bm = "exact" if mode in ("fp32", "mixed") else mode
            bs, bf = NF.BUDGETS[(bm, tag, "space", "scene")], NF.BUDGETS[(bm, tag, "motion", "scene")]
            assert e["sig_rms"] <= bs["sig_rms"] and e["sig_max"] <= bs["sig_max"], (mode, frame, e, bs)
            assert ef["flow_rms"] <= bf["flow_rms"] and ef["flow_max"] <= bf["flow_max"], (mode, frame, ef, bf)


# ---- marching cubes ------------------------------------------------------------------------------------------------------
def _mc(g, origin, step, level):
    v, f = N.marching_cubes(torch.from_numpy(g).to(DEV), origin, step, level)
    return v.cpu(), f.cpu()


def _check_against_restatement(g, origin, step, level):
    v, f = _mc(g, origin, step, level)
    v64, f64, owner = M.marching_cubes(g, origin, step, level)
    assert v.shape == v64.shape and f.shape == f64.shape
    assert np.array_equal(f.numpy().astype(np.int64), f64)
    ext = max(abs(origin[a]) + g.shape[a] * step[a] for a in range(3))
    assert np.abs(v.numpy().astype(np.float64) - v64).max() <= 4 * ext * 2.0 ** -24
    # every vertex on its grid edge, interpolating to the level within fp32 rounding
    s = g.reshape(-1).astype(np.float64)
    stride = np.array([g.shape[1] * g.shape[2], g.shape[2], 1])
    p, a = owner[:, 0], owner[:, 1]
    ijk = np.stack([p // stride[0], (p // stride[1]) % g.shape[1], p % g.shape[2]], 1)
    x0 = np.asarray(origin, np.float32)[None] + ijk.astype(np.float32) * np.asarray(step, np.float32)[None]
    vv = v.numpy()
    for ax in range(3):
        off = a != ax
        assert np.array_equal(vv[off, ax], x0[off, ax].astype(np.float32))
    tt = (vv[np.arange(len(a)), a] - x0[np.arange(len(a)), a]) / np.asarray(step, np.float64)[a]
    v0, v1 = s[p], s[p + stride[a]]
    tol = 4 * ext * 2.0 ** -24 / np.asarray(step, np.float64)[a]      # a coordinate's rounding, in units of the step
    assert (tt >= -tol).all() and (tt <= 1 + tol).all()
    interp = v0 + tt * (v1 - v0)
    assert (np.abs(interp - level) <= tol * np.abs(v1 - v0) + 1e-6 * (abs(level) + 1)).all()
    return v, f


FIELDS = {
    "sphere": (M.sphere((0.1, -0.05, 0.02), 0.7), (33, 33, 33), (0.05, 0.05, 0.05), 0.0, 2, 4 / 3 * math.pi * 0.7 ** 3),
    "aniso": (M.sphere((0.1, -0.05, 0.02), 0.7), (25, 41, 33), (0.07, 0.045, 0.055), 0.0, 2, 4 / 3 * math.pi * 0.7 ** 3),
    "torus": (M.torus(0.6, 0.25), (40, 40, 20), (0.05, 0.05, 0.05), 0.0, 0, 2 * math.pi ** 2 * 0.6 * 0.25 ** 2),
    "touching": (lambda x, y, z: np.maximum(M.sphere((-0.4, 0, 0), 0.4)(x, y, z), M.sphere((0.4, 0, 0), 0.4)(x, y, z)),
                 (41, 41, 41), (0.05, 0.05, 0.05), 0.0, None, 2 * 4 / 3 * math.pi * 0.4 ** 3),
}


@pytest.mark.parametrize("name", sorted(FIELDS))
def test_mc_analytic_fields(name):
    fn, dims, h, level, chi, vol = FIELDS[name]
    origin = tuple(-(d - 1) * s / 2 for d, s in zip(dims, h))
    g = M.grid_values(fn, origin, h, dims)
    v, f = _check_against_restatement(g, origin, h, level)
    f = f.numpy()
    assert M.is_closed(f) and M.oriented_consistently(f)
    if chi is not None:
        assert M.euler_characteristic(v.numpy(), f) == chi
    vv = v.numpy().astype(np.float64)
    assert M.signed_volume(vv, f) > 0
    assert abs(M.signed_volume(vv, f) - vol) <= max(h) ** 2 * M.area(vv, f)


@pytest.mark.parametrize("seed", range(3))
def test_mc_random_gaussians(seed):
    rs = np.random.RandomState(100 + seed)
    cs, ws, amp = rs.uniform(-0.5, 0.5, (8, 3)), rs.uniform(0.08, 0.3, 8), rs.uniform(0.5, 2.0, 8)

    def fn(x, y, z):
        return sum(a * np.exp(-((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) / (2 * w * w)) for c, w, a in zip(cs, ws, amp))

    origin, h = (-1.2, -1.1, -1.0), (2.4 / 37, 2.2 / 45, 2.0 / 29)
    g = M.grid_values(fn, origin, h, (38, 46, 30))
    level = 0.35
    assert max(g[0].max(), g[-1].max(), g[:, 0].max(), g[:, -1].max(), g[:, :, 0].max(), g[:, :, -1].max()) < level
    v, f = _check_against_restatement(g, origin, h, level)
    assert M.is_closed(f.numpy()) and M.oriented_consistently(f.numpy())
    assert M.signed_volume(v.numpy().astype(np.float64), f.numpy()) > 0


def test_mc_planes_through_grid_values():
    """Planes that cross exactly at grid values (v == level is outside): vertices land on grid points."""
    h = (0.25, 0.5, 0.125)
    origin = (-1.0, -2.0, -0.5)
    g = M.grid_values(lambda x, y, z: np.minimum(x - 0.25, 1.0 - y), origin, h, (9, 9, 9))
    _check_against_restatement(g, origin, h, 0.0)
    _check_against_restatement(g, origin, h, 0.5)


def test_mc_empty_full_and_high_level():
    h = (0.1, 0.1, 0.1)
    for g, level in ((np.zeros((5, 6, 7), np.float32), 0.5), (np.ones((5, 6, 7), np.float32), 0.5),
                     (np.random.RandomState(0).rand(9, 9, 9).astype(np.float32), 2.0),
                     (np.full((4, 4, 4), np.nan, np.float32), 0.0)):
        v, f = _mc(g, (0, 0, 0), h, level)
        assert v.shape == (0, 3) and f.shape == (0, 3)


def test_mc_repeatable_and_validated():
    from stnerf_b200 import _lib as L
    g = M.grid_values(M.torus(0.6, 0.25), (-1, -1, -0.5), (0.03, 0.03, 0.03), (67, 67, 34))
    a, b = _mc(g, (-1, -1, -0.5), (0.03, 0.03, 0.03), 0.0), _mc(g, (-1, -1, -0.5), (0.03, 0.03, 0.03), 0.0)
    assert _same(a[0], b[0]) and torch.equal(a[1], b[1])
    import ctypes
    for bad in (((0, 0, 0), (0.1, 0.1, 0.1), (1, 4, 4)), ((0, 0, 0), (0.1, -0.1, 0.1), (4, 4, 4)),
                ((0, float("nan"), 0), (0.1, 0.1, 0.1), (4, 4, 4))):
        assert L.lib().stnerf_mc_scratch_bytes(ctypes.byref(N.make_grid(*bad))) == 0
        with pytest.raises(L.StnerfError):
            N.marching_cubes(torch.zeros(tuple(max(d, 1) for d in bad[2]), device=DEV), bad[0], bad[1], 0.0)


# ---- end to end --------------------------------------------------------------------------------------------------------
def _boundary_ok(mesh, lo, hi, h):
    """Edges used by one face only lie on the faces of the box (the grid border)."""
    keys, counts = M.edge_face_counts(mesh.faces.cpu().numpy())
    assert (counts <= 2).all()
    v = mesh.verts.cpu().numpy().astype(np.float64)
    ends = v[keys[counts == 1].reshape(-1)]
    tol = 1e-5 * (np.abs(np.asarray(hi)).max() + 1)
    on_face = (np.abs(ends - np.asarray(lo)) <= tol) | (np.abs(ends - np.asarray(hi)) <= tol)
    assert on_face.any(1).all()


@pytest.mark.parametrize("frame", [1.0, 1.5])
def test_taekwondo_performer_mesh(frame):
    sd = NF.state_dict("tkd")
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    case = dict(weights="taekwondo", L=1, space_time=True, n1=64, n2=128)
    model = _model(case, "exact", sd=sd)
    # where is the performer?  a coarse look over the background box, then a box around its dense part
    blo, bhi = X.layer_box(model, 0, frame)
    d = X.layer_density(model, 1, frame, resolution=48, bbox=[blo, bhi])
    s = d.sigma.cpu().numpy()
    level = 0.25 * float(s.max())
    assert level > 0
    ijk = np.argwhere(s > level)
    lo = [d.origin[a] + (ijk[:, a].min() - 2) * d.step[a] for a in range(3)]
    hi = [d.origin[a] + (ijk[:, a].max() + 2) * d.step[a] for a in range(3)]
    mesh = X.extract_mesh(model, 1, frame, level, resolution=96, bbox=[lo, hi])
    assert mesh.faces.shape[0] > 100 and mesh.faces.dtype == torch.int64
    v = mesh.verts.cpu().numpy()
    assert (v >= np.asarray(lo, np.float32) - 1e-5).all() and (v <= np.asarray(hi, np.float32) + 1e-5).all()
    _boundary_ok(mesh, lo, hi, None)
    col = mesh.colors.cpu()
    assert col.shape == mesh.verts.shape and bool(((col >= 0) & (col <= 1)).all())
    # the field at a vertex is within the interpolation bound of the level: the field varies along the vertex's grid edge by
    # no more than the range of 17 samples of it there (plus what lies between them: half that range again)
    dens = X.layer_density(model, 1, frame, 96, [lo, hi])
    _, _, owner = M.marching_cubes(dens.sigma.cpu().numpy(), dens.origin, dens.step, level)
    stride = np.array([96 * 96, 96, 1])
    p, a = owner[:, 0], owner[:, 1]
    ijk = np.stack([p // stride[0], (p // stride[1]) % 96, p % 96], 1).astype(np.float64)
    x0 = np.asarray(dens.origin)[None] + ijk * np.asarray(dens.step)[None]
    s = np.linspace(0.0, 1.0, 17)
    pts = np.repeat(x0[:, None, :], 17, 1)
    pts[np.arange(len(a)), :, a] += s[None, :] * np.asarray(dens.step)[a][:, None]
    nat, _ = X._scene_at(model, frame)
    _, along = nat.layer_field(1, True, frame, torch.from_numpy(pts.reshape(-1, 3).astype(np.float32)).to(DEV), None,
                               want_rgb=False)
    along = along.cpu().numpy().astype(np.float64).reshape(-1, 17)
    _, at = nat.layer_field(1, True, frame, mesh.verts, None, want_rgb=False)
    bound = 1.5 * (along.max(1) - along.min(1)) + 1e-3 * abs(level)
    assert (np.abs(at.cpu().numpy().astype(np.float64) - level) <= bound).all()


def test_extract_after_an_adam_step():
    case = dict(SYN)
    model = _model(case, "exact", trainable=True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    rays = C.rays_for(case).to(DEV)
    with torch.enable_grad():
        out = model(rays, torch.zeros(rays.shape[0], device=DEV), None, density_threshold=0.0, bkgd_density_threshold=0.0)
        out[0][0].square().mean().backward()
    opt.step()
    fresh = _model(case, "exact", sd={k: v.detach().cpu() for k, v in model.state_dict().items()})
    d0 = X.layer_density(fresh, 1, 10.0, 40)
    level = float(d0.sigma.float().quantile(0.9))
    a = X.extract_mesh(model, 1, 10.0, level, resolution=40)
    b = X.extract_mesh(fresh, 1, 10.0, level, resolution=40)
    assert a.faces.shape[0] > 0
    assert _same(a.verts, b.verts) and torch.equal(a.faces, b.faces) and _same(a.colors, b.colors)
    before = _model(case, "exact")
    c = X.extract_mesh(before, 1, 10.0, level, resolution=40)
    assert not (c.verts.shape == a.verts.shape and _same(c.verts, a.verts))
