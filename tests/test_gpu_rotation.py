"""The rotation edit on the device.

A layer rotated by R about c samples, marches and looks along its own rays o' = c + R^T (o - c), d' = R^T d.  So rendering a
model whose every layer carries the same (R, c) along rays r must equal, bit for bit, rendering the unrotated model along the
fp32 restatement r' -- through stnerf_render (9- and 7-column rays, fp32 and exact) and through stnerf_render_views
(PoseRenderer).  Also: the rotate kernel against its fp32 restatement and float64, oriented-box clipping against a float64 slab
test, the R versus R^T convention of the field, selectivity and hidden layers, and the differentiable forward."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import cases as C
from oracle import stnerf_oracle as O
from stnerf_b200 import extract as X
from stnerf_b200 import native as N
from stnerf_b200 import ops, split_planes
from stnerf_b200 import rotation as ROT
from tests_support import make_cfg

pytestmark = pytest.mark.gpu

DEV = "cuda"
SYN = C.CASES["syn_L2_64_128"]
R_GEN = Rotation.from_rotvec([0.31, -0.52, 0.77]).as_matrix().astype(np.float32)     # not axis-aligned
C_GEN = np.float32([0.13, -0.21, 0.4])


def rotate_rays_f32(rays, R, c):
    """The kernel's op order in numpy float32: q = o - c; o'_a = ((Rt[a,0] q0 + Rt[a,1] q1) + Rt[a,2] q2) + c_a; d' likewise."""
    r = np.array(rays, dtype=np.float32, copy=True)
    Rt = np.asarray(R, np.float32).T
    c = np.asarray(c, np.float32)
    q = [r[:, a] - c[a] for a in range(3)]
    d = [r[:, 3 + a].copy() for a in range(3)]
    for a in range(3):
        r[:, a] = ((Rt[a, 0] * q[0] + Rt[a, 1] * q[1]) + Rt[a, 2] * q[2]) + c[a]
        r[:, 3 + a] = (Rt[a, 0] * d[0] + Rt[a, 1] * d[1]) + Rt[a, 2] * d[2]
    return r


def _model(case, precision, rotation=None, trainable=False):
    import modeling
    cfg = make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], precision)
    cfg.MODEL.B200_TRAINABLE = trainable
    model = modeling.build_layered_model(cfg, 0, case.get("scale"), case.get("shift"), rotation=rotation)
    model.load_state_dict(C.state_dict_for(case))
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    return model.cuda()


def _forward(model, rays, uni, thr=(0.0, 0.0)):
    jit, u = uni
    model.inject_uniforms(jit.to(DEV).contiguous(), u.to(DEV).contiguous())
    with torch.no_grad():
        out = model(rays.to(DEV), None, None, density_threshold=thr[0], bkgd_density_threshold=thr[1])
    torch.cuda.synchronize()
    return C.flatten_outputs(*out)


def _equal(a, b, keys=None):
    for k in (keys or a):
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


def _rays(columns):
    rays = C.rays_for(SYN)
    if columns == 7:
        rays = rays[:, :7].clone()
        rays[:, 6] = 10.0
    return rays.contiguous()


# ---------------------------------------------------------------------------------------------------------------------
def test_rotate_rays_kernel_bits_and_float64():
    rs = np.random.RandomState(0)
    rays = np.concatenate([rs.normal(size=(5000, 3)) * 4, rs.normal(size=(5000, 3)), rs.uniform(0, 30, (5000, 3))], 1)
    rays = rays.astype(np.float32)
    rays[:, 3:6] /= np.linalg.norm(rays[:, 3:6], axis=1, keepdims=True)
    got = N.rotate_rays(torch.from_numpy(rays).to(DEV), R_GEN, C_GEN).cpu().numpy()
    want = rotate_rays_f32(rays, R_GEN, C_GEN)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    R64, c64, r64 = R_GEN.astype(np.float64), C_GEN.astype(np.float64), rays.astype(np.float64)
    o64 = (R64.T @ (r64[:, :3] - c64).T).T + c64
    d64 = (R64.T @ r64[:, 3:6].T).T
    scale = np.abs(r64[:, :3]).max() + np.abs(c64).max()
    assert np.abs(got[:, :3] - o64).max() <= 8 * np.finfo(np.float32).eps * scale
    assert np.abs(got[:, 3:6] - d64).max() <= 8 * np.finfo(np.float32).eps


@pytest.mark.parametrize("columns", [9, 7])
@pytest.mark.parametrize("precision", ["fp32", "exact"])
def test_camera_equivalence_forward(precision, columns):
    rays = _rays(columns)
    uni = C.uniforms_for(SYN)
    rot = _model(SYN, precision, rotation=[(R_GEN, C_GEN)] * 3)
    got = _forward(rot, rays, uni)
    plain = _model(SYN, precision)
    want = _forward(plain, torch.from_numpy(rotate_rays_f32(rays.numpy(), R_GEN, C_GEN)), uni)
    _equal(got, want)
    assert got["ray_mask.1"].any() and got["ray_mask.2"].any()
    # and the rotation does something
    base = _forward(plain, rays, uni)
    assert not np.array_equal(base["fine_mixed.rgb"], got["fine_mixed.rgb"])


def test_camera_equivalence_render_views_and_pose_renderer():
    from stnerf_b200 import PoseRenderer
    H, W = 48, 64
    K, T = O.synthetic_camera(3, 16, H, W)
    ids = [0.0, 10.0, 11.0]
    rot = _model(SYN, "exact", rotation=[(R_GEN, C_GEN)] * 3)
    pr = PoseRenderer(rot, H, W, far=20.0)
    seed = rot.seed + 1
    img = pr.render_images(T, K, [(0, 0), (1, 10), (2, 11)])                  # (l+1, H, W, 5)
    plain = _model(SYN, "exact")
    nat = plain._ensure_native(torch.device(DEV))
    plain.retiming = True
    nat.set_scene(plain._resolve_scene(torch.tensor(ids), 0.0, 0.0))
    rays = ops.generate_rays(K, T, H, W, frame_ids=ids).cpu().numpy()
    out, _ = nat.render(torch.from_numpy(rotate_rays_f32(rays, R_GEN, C_GEN)).to(DEV), 64, 128, seed=seed)
    fm, _, fl, _ = split_planes(out, 3)
    assert torch.equal(fm[0].reshape(H, W, 3), img[0, ..., :3]) and torch.equal(fm[1].reshape(H, W), img[0, ..., 3])
    for i in range(3):
        assert torch.equal(fl[i][0].reshape(H, W, 3), img[1 + i, ..., :3]) and torch.equal(fl[i][2].reshape(H, W), img[1 + i, ..., 4])


def test_default_centre_is_each_calls_box_centre():
    """A rotation without a centre turns each layer about its edited box's centre: the same render as the explicit centres."""
    rays, uni = _rays(9), C.uniforms_for(SYN)
    a = _model(SYN, "exact", rotation=[None, R_GEN, R_GEN])
    got = _forward(a, rays, uni)
    sc = a._resolve_scene(torch.tensor(SYN["frame_ids"], dtype=torch.float32), 0.0, 0.0)
    cen = [ROT.default_centre(sc.bmin[i][:], sc.bmax[i][:]) for i in range(3)]
    b = _model(SYN, "exact", rotation=[None, (R_GEN, cen[1]), (R_GEN, cen[2])])
    _equal(got, _forward(b, rays, uni))


def test_selectivity_and_hidden_layers():
    rays, uni = _rays(9), C.uniforms_for(SYN)
    plain = _model(SYN, "exact")
    base = _forward(plain, rays, uni)
    one = _model(SYN, "exact", rotation=[None, (R_GEN, C_GEN), None])
    got = _forward(one, rays, uni)
    _equal(got, base, [k for k in base if k.startswith(("fine_layer.2", "coarse_layer.2", "fine_layer.0", "coarse_layer.0"))
                       or k in ("ray_mask.0", "ray_mask.2")])
    assert not np.array_equal(got["fine_layer.1.rgb"], base["fine_layer.1.rgb"])
    one.hide_layer(1)
    plain.hide_layer(1)
    _equal(_forward(one, rays, uni), _forward(plain, rays, uni))


def _slab64(o, d, lo, hi):
    """float64 slab test of the box [lo, hi] along o + t d: (hit, t_near, t_far)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (lo - o) / d, (hi - o) / d
    tn, tf = np.nanmax(np.minimum(t1, t2), 1), np.nanmin(np.maximum(t1, t2), 1)
    return tf > tn, tn, tf


def test_oriented_box_clipping_against_float64():
    """Rays at face centres, edges and corners of an oriented box: the kernel's clip of the rotated rays against the edited box
    agrees with a float64 slab test of the oriented box (hit and t_near / t_far), away from edges by a margin."""
    lo, hi = np.float64([-0.4, -0.7, -1.1]), np.float64([0.5, 0.6, 0.9])
    R64 = R_GEN.astype(np.float64)
    c = ((lo + hi) / 2).astype(np.float32)
    rs = np.random.RandomState(3)
    fams = {}
    ctr = (lo + hi) / 2
    half = (hi - lo) / 2
    # local targets: face interiors (inset), edge midpoints pulled inward, corners pulled inward, and points outside (misses)
    face = np.stack([ctr + half * np.eye(3)[k % 3] * (1 if k < 3 else -1) * 0.999 + rs.uniform(-0.6, 0.6, 3) * half
                     * (1 - np.eye(3)[k % 3]) for k in range(6) for _ in range(50)])
    edge = np.stack([ctr + half * np.array(s) * 0.97 for s in [(1, 1, 0), (1, -1, 0), (-1, 0, 1), (0, 1, -1), (0, -1, -1)]
                     for _ in range(20)])
    corner = np.stack([ctr + half * np.array([sx, sy, sz]) * 0.97 for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)
                       for _ in range(10)])
    miss = np.stack([ctr + half * (2.0 + rs.uniform(0, 1, 3)) * rs.choice([-1, 1], 3) for _ in range(200)])
    fams = dict(face=face, edge=edge, corner=corner, miss=miss)
    counts = {}
    for name, tgt in fams.items():
        w_tgt = (R64 @ (tgt - c).T).T + c                                 # targets on the oriented box in the world
        eye = rs.normal(size=(len(tgt), 3))
        eye = ctr + 6 * eye / np.linalg.norm(eye, axis=1, keepdims=True)
        eye = (R64 @ (eye - c).T).T + c
        dvec = w_tgt - eye
        dvec /= np.linalg.norm(dvec, axis=1, keepdims=True)
        rays = np.concatenate([eye, dvec, np.zeros((len(tgt), 3))], 1).astype(np.float32)
        rr = N.rotate_rays(torch.from_numpy(rays).to(DEV), R_GEN, c)
        n1 = 4
        tt = torch.empty((len(rays), 2), dtype=torch.float32, device=DEV)
        mask = torch.empty(len(rays), dtype=torch.uint8, device=DEV)
        jit = torch.zeros((len(rays), n1), dtype=torch.float32, device=DEV)
        lo32, hi32 = torch.tensor(lo, dtype=torch.float32), torch.tensor(hi, dtype=torch.float32)
        from stnerf_b200 import _lib as L
        L.check(L.lib().stnerf_intersect_sample(L.ptr(rr), len(rays), 9, L.ptr(lo32), L.ptr(hi32), 0, n1, L.ptr(jit), None,
                                                None, L.ptr(mask), L.ptr(tt), L.stream_ptr()), "intersect")
        torch.cuda.synchronize()
        m, tt = mask.cpu().numpy().astype(bool), tt.cpu().numpy().astype(np.float64)
        # float64: rotate the rays back exactly and slab-test the edited box
        o64 = (R64.T @ (rays[:, :3].astype(np.float64) - c).T).T + c
        d64 = (R64.T @ rays[:, 3:6].astype(np.float64).T).T
        hit, tn, tf = _slab64(o64, d64, lo, hi)
        assert np.array_equal(m, hit), name
        # depths away from edges: where the entry or exit point lies within 1e-4 of two faces the fp32 face tests may pick another
        # face of the same corner region, as for an axis-aligned box (test_gpu_sampling_f64)
        def near_edge(t):
            p = o64 + t[:, None] * d64
            return ((np.abs(p - lo) < 1e-4) | (np.abs(p - hi) < 1e-4)).sum(1) >= 2
        ok = hit & ~near_edge(np.where(hit, tn, 0)) & ~near_edge(np.where(hit, tf, 0))
        assert ok.sum() >= 0.9 * hit.sum(), name
        # the fp32 rotation moves o' by a few ulp of |o|; a depth moves by that over the direction's component across the face
        with np.errstate(divide="ignore", invalid="ignore"):
            t1, t2 = (lo - o64) / d64, (hi - o64) / d64
        a_near, a_far = np.argmax(np.minimum(t1, t2), 1), np.argmin(np.maximum(t1, t2), 1)
        rows = np.arange(len(rays))
        for col, t64, ax in ((1, tn, a_near), (0, tf, a_far)):
            tol = 2e-5 + 1e-5 * np.abs(t64) + 8e-7 * 6 / np.abs(d64[rows, ax])
            assert (np.abs(tt[ok, col] - t64[ok]) <= tol[ok]).all(), name
        counts[name] = int(hit.sum())
    assert counts["face"] == 300 and counts["edge"] == 100 and counts["corner"] == 80 and counts["miss"] < 200, counts


def _field_pair(case, frame):
    R90 = Rotation.from_rotvec([0, 0, np.pi / 2]).as_matrix().astype(np.float32)      # vertical axis here is z; R != R^T
    rot = _model(case, "exact", rotation=[None, R90] + [None] * (case["L"] - 1))
    plain = _model(case, "exact")
    return R90, rot, plain


@pytest.mark.parametrize("frame", [10.0, 10.5])
def test_field_convention_bits(frame):
    """The rotated field at world points w equals, bit for bit, the unrotated field at the fp32 c + R^T (w - c) (colour seen
    along R^T d), with c the default centre."""
    R90, rot, plain = _field_pair(SYN, frame)
    sc = X._scene(rot, frame)
    c = ROT.default_centre(sc.bmin[1][:], sc.bmax[1][:])
    rs = np.random.RandomState(5)
    lo, hi = np.float32(sc.bmin[1][:]), np.float32(sc.bmax[1][:])
    w = (lo + (hi - lo) * rs.uniform(-0.2, 1.2, (3000, 3))).astype(np.float32)
    d = rs.normal(size=(3000, 3)).astype(np.float32)
    packed = np.concatenate([w, d], 1)
    back = rotate_rays_f32(packed, R90, c)
    X._scene_at(rot, frame)
    rgb_r, sig_r = rot._native.layer_field(1, True, frame, torch.from_numpy(w).to(DEV), torch.from_numpy(d).to(DEV))
    X._scene_at(plain, frame)
    rgb_p, sig_p = plain._native.layer_field(1, True, frame, torch.from_numpy(back[:, :3].copy()).to(DEV),
                                             torch.from_numpy(back[:, 3:6].copy()).to(DEV))
    assert torch.equal(sig_r, sig_p) and torch.equal(rgb_r, rgb_p)


def test_field_convention_centroid_and_mesh():
    """R versus R^T: the sigma centroid of a performer turned 90 degrees about the vertical axis is c + R (centroid0 - c) of
    the unrotated one, within one grid step; the mesh volume agrees within h^2 * area."""
    import test_gpu_networks_f64 as NF
    sd = NF.state_dict("tkd")
    case = dict(weights="taekwondo", L=1, space_time=True, n1=64, n2=128) if sd is not None else SYN
    frame = 1.0 if sd is not None else 10.0
    R90, rot, plain = _field_pair(case, frame) if sd is None else (None, None, None)
    if sd is not None:
        import modeling
        R90 = Rotation.from_rotvec([0, 0, np.pi / 2]).as_matrix().astype(np.float32)
        mk = []
        for r in ([None, R90], None):
            cfg = make_cfg(1, 64, 128, True, "exact")
            m = modeling.build_layered_model(cfg, 0, None, None, rotation=r)
            m.load_state_dict(sd)
            bk, fr = C.boxes_for(case)
            m.set_bkgd_bbox(bk)
            m.set_bboxes(fr)
            mk.append(m.cuda())
        rot, plain = mk
    sc = X._scene(plain, frame)
    c = ROT.default_centre(sc.bmin[1][:], sc.bmax[1][:]).astype(np.float64)

    def centroid(d):
        s = np.maximum(d.sigma.cpu().numpy().astype(np.float64), 0)
        ijk = np.stack(np.meshgrid(*[np.arange(n) for n in s.shape], indexing="ij"), -1).reshape(-1, 3)
        p = np.asarray(d.origin) + ijk * np.asarray(d.step)
        return (p * s.reshape(-1, 1)).sum(0) / s.sum(), max(d.step)

    d0 = X.layer_density(plain, 1, frame, resolution=64)
    d1 = X.layer_density(rot, 1, frame, resolution=64)
    c0, h0 = centroid(d0)
    c1, h1 = centroid(d1)
    want = c + R90.astype(np.float64) @ (c0 - c)
    assert np.abs(c1 - want).max() <= max(h0, h1), (c1, want)
    level = 0.25 * float(d0.sigma.max())
    m0 = X.extract_mesh(plain, 1, frame, level, resolution=64, colors=False)
    m1 = X.extract_mesh(rot, 1, frame, level, resolution=64, colors=False)

    def vol_area(m):
        v = m.verts.cpu().double().numpy()
        f = m.faces.cpu().numpy()
        a, b, cc = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
        return abs(np.einsum("ij,ij->i", a, np.cross(b, cc)).sum()) / 6, 0.5 * np.linalg.norm(np.cross(b - a, cc - a), axis=1).sum()
    v0, a0 = vol_area(m0)
    v1, a1 = vol_area(m1)
    h = max(h0, h1)
    assert abs(v0 - v1) <= h * h * max(a0, a1), (v0, v1, h * h * max(a0, a1))


def test_training_forward_with_a_rotated_performer():
    rays, uni = _rays(9), C.uniforms_for(SYN)
    rotation = [None, (R_GEN, C_GEN), None]
    tr = _model(SYN, "fp32", rotation=rotation, trainable=True)
    plain = _model(SYN, "fp32", rotation=rotation)
    jit, u = uni

    def run(m, grad):
        m.inject_uniforms(jit.to(DEV).contiguous(), u.to(DEV).contiguous())
        with torch.set_grad_enabled(grad):
            return m(rays.to(DEV), None, None, density_threshold=0.0, bkgd_density_threshold=0.0)

    got = run(tr, True)
    want = C.flatten_outputs(*run(plain, False))
    flat = C.flatten_outputs(*got)
    for k in want:
        if k.startswith("ray_mask"):
            assert np.array_equal(flat[k], want[k]), k
        else:
            assert float(np.abs(flat[k].astype(np.float64) - want[k]).max()) <= 1e-5, k
    # identical calls, identical gradient bits; an Adam step changes the image
    grads = []
    for _ in range(2):
        tr.zero_grad()
        out = run(tr, True)
        loss = sum(o.square().mean() for o in out[0])
        loss.backward()
        grads.append({k: p.grad.detach().clone() for k, p in tr.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys() and all(torch.equal(grads[0][k], grads[1][k]) for k in grads[0])
    opt = torch.optim.Adam(tr.parameters(), lr=1e-3)
    opt.step()
    with torch.no_grad():
        after = C.flatten_outputs(*run(tr, False))
    assert not np.array_equal(after["fine_layer.1.rgb"], flat["fine_layer.1.rgb"])
