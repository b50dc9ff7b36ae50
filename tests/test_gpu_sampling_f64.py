"""The sampling stage ray by ray: geometry.cu (ray generation, clipping, stratified sampling, positional encoding) and
train_march.cu (ordered hit lists, training points, masked scatter / gather, fine uniforms) against the reference's outputs
on adversarial rays (tests/golden/geometry.npz), the CPU oracle's fp32 restatement and float64.

Comparisons are bit for bit unless stated.  The one leniency: where two candidates of the top-2 are +0 and -0 (an origin on
an edge or corner), torch's topk orders the tie differently with the row's width and the kernel keeps the first face, so a
zero may differ in sign (`same` below).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import make_golden_geometry as G
import tests_support as TS
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

GOLD = TS.C.load_golden("geometry")
IN = G.geometry_inputs()
RAYS = IN["rays"]
N = RAYS.shape[0]
F32 = torch.float32
EINVAL = -1


def _np(x):
    return (x.detach().cpu() if torch.is_tensor(x) else torch.as_tensor(x)).numpy()


def same(a, b, what=""):
    """Equal bits, or both zero."""
    a, b = np.asarray(_np(a), np.float32), np.asarray(_np(b), np.float32)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    ok = (a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0))
    assert ok.all(), "%s: %d differ, first at %s: %r vs %r" % (what, (~ok).sum(), np.argwhere(~ok)[0], a[~ok][0], b[~ok][0])


def L():
    from stnerf_b200 import _lib
    return _lib


def intersect(rays, box, n1, jitter, is_bkgd, stride=None):
    """stnerf_intersect_sample through the C ABI; rays (n, >= 6) CUDA, `stride` floats per row (default its width)."""
    lib = L()
    rays = rays.contiguous()
    n = rays.shape[0] if stride is None else rays.numel() // stride
    stride = rays.shape[1] if stride is None else stride
    bmin = torch.tensor(box[0], dtype=F32)
    bmax = torch.tensor(box[1], dtype=F32)
    t = torch.empty((n, n1), dtype=F32, device="cuda")
    xyz = torch.empty((n, n1, 3), dtype=F32, device="cuda")
    mask = torch.empty((n,), dtype=torch.uint8, device="cuda")
    tt = torch.empty((n, 2), dtype=F32, device="cuda")
    lib.check(lib.lib().stnerf_intersect_sample(lib.ptr(rays), n, stride, lib.ptr(bmin), lib.ptr(bmax), int(is_bkgd), n1,
                                                lib.ptr(jitter.contiguous()), lib.ptr(t), lib.ptr(xyz), lib.ptr(mask),
                                                lib.ptr(tt), lib.stream_ptr()), "stnerf_intersect_sample")
    torch.cuda.synchronize()
    return t.cpu(), xyz.cpu(), mask.cpu(), tt.cpu()


def restated(rays, bmin, bmax, n1, jitter, is_bkgd, cols):
    r = torch.as_tensor(rays)
    far, near = O.ray_box_intersect(r[:, :3], r[:, 3:6], torch.as_tensor(bmin), torch.as_tensor(bmax), cols)
    t, xyz, m = O.stratified_samples(r[:, :3], r[:, 3:6], torch.as_tensor(bmin), torch.as_tensor(bmax), n1,
                                     torch.as_tensor(jitter), is_bkgd, cols)
    return t, xyz, m.to(torch.uint8), torch.stack([far, near], 1)


# ---------------------------------------------------------------------------------------------------------- intersect_sample
@pytest.mark.parametrize("cols", G.COLUMNS)
def test_intersect_sample_equals_the_reference(cols):
    rays = torch.from_numpy(G.widen(RAYS, cols))
    for n1 in G.GOLDEN_N1:
        for layer in (0, 1):
            jit = torch.from_numpy(G.jitter_for(N, n1, 10 * layer))
            got_t = torch.empty((N, n1)); got_m = torch.empty((N,), dtype=torch.uint8); got_tt = torch.empty((N, 2))
            got_x = torch.empty((N, n1, 3))
            for b in np.unique(IN["box_id"]):
                sel = torch.from_numpy(np.flatnonzero(IN["box_id"] == b))
                t, xyz, m, tt = intersect(rays[sel].cuda(), IN["boxes"][b], n1, jit[sel].cuda(), layer == 0)
                got_t[sel], got_x[sel], got_m[sel], got_tt[sel] = t, xyz, m, tt
            same(got_tt, GOLD["isect.%d" % cols], "tfar_tnear cols=%d" % cols)
            assert np.array_equal(_np(got_m), GOLD["mask.%d.%d.%d" % (cols, layer, n1)]), (cols, layer, n1)
            if n1 == 3:
                same(got_t, GOLD["t.%d.%d.3" % (cols, layer)], "t")
                if cols == 7:
                    same(got_x, GOLD["xyz.7.%d.3" % layer], "xyz")


@pytest.mark.parametrize("n1", [1, 2, 3, 47, 64, 128, 129])
def test_intersect_sample_equals_the_restatement(n1):
    box_ids = IN["box_id"]
    for cols in G.COLUMNS:
        rays = G.widen(RAYS, cols)
        jit = G.jitter_for(N, n1, 7)
        for b in np.unique(box_ids):
            sel = np.flatnonzero(box_ids == b)
            for is_bkgd in (True, False):
                got = intersect(torch.from_numpy(rays[sel]).cuda(), IN["boxes"][b], n1, torch.from_numpy(jit[sel]).cuda(), is_bkgd)
                want = restated(rays[sel], IN["boxes"][b][0], IN["boxes"][b][1], n1, jit[sel], is_bkgd, cols)
                for g, w, what in zip(got, want, ("t", "xyz", "mask", "tfar_tnear")):
                    same(g, w, "%s n1=%d cols=%d box=%d" % (what, n1, cols, b))


def test_wide_ray_stride_through_the_c_abi():
    """A row of 12 floats: the columns of the top-2 are the stride's (two sentinels), whatever the extra floats hold."""
    rays = np.concatenate([RAYS, np.full((N, 6), np.nan, np.float32)], 1)
    jit = G.jitter_for(N, 3, 0)
    b = 1
    sel = np.flatnonzero(IN["box_id"] == b)
    got = intersect(torch.from_numpy(rays[sel]).reshape(-1).cuda(), IN["boxes"][b], 3, torch.from_numpy(jit[sel]).cuda(), True,
                    stride=12)
    same(got[3], GOLD["isect.9"][sel], "tfar_tnear")
    same(got[0], GOLD["t.9.0.3"][sel], "t")


# ---------------------------------------------------------------------------------------------------------- contexts
def make_scene(boxes, shared=False, **kw):
    lib = L()
    sc = lib.Scene()
    for i, (lo, hi) in enumerate(boxes):
        for a in range(3):
            sc.bmin[i][a], sc.bmax[i][a] = float(lo[a]), float(hi[a])
        sc.shown[i] = 1
        sc.scale[i] = 1.0
    sc.boarder_weight = 1e10
    sc.alpha_layer2 = kw.get("alpha", 1.0)
    sc.near_plane = kw.get("near", 0.0)
    sc.density_threshold = kw.get("thr", 1e-4)
    sc.bkgd_density_threshold = kw.get("thr_bkgd", 0.0)
    sc.apply_thresholds = 1 if kw.get("apply_thr", not shared) else 0
    sc.shared_frame_id = 1 if shared else 0
    return sc


def context(l, sc, chunk_rays=0):
    from stnerf_b200.native import NativeRenderer
    nat = NativeRenderer(l, [False] * l, "fp32", chunk_rays)
    nat.set_scene(sc)
    return nat


def layer_boxes(l):
    return [IN["boxes"][i % 4] if i < 4 else IN["boxes"][4 + i] for i in range(l)]


def tiled_rays(n, cols, fid=1.0):
    r = np.resize(RAYS, (n, 6))
    return np.concatenate([r, np.full((n, cols - 6), fid, np.float32)], 1)


def train_sample(nat, rays, n1, jitter=None, seed=0):
    lib = L()
    l, n = nat.l, rays.shape[0]
    t = torch.empty((l, n, n1), dtype=F32, device="cuda")
    mask = torch.empty((l, n), dtype=torch.uint8, device="cuda")
    hit = torch.full((l, n), -7, dtype=torch.int32, device="cuda")
    counts, frac = (C.c_int32 * l)(), (C.c_int32 * l)()
    rc = lib.lib().stnerf_train_sample(nat._h, lib.ptr(rays), n, rays.stride(0), n1, lib.ptr(jitter), seed, lib.ptr(t),
                                       lib.ptr(mask), lib.ptr(hit), counts, frac, lib.stream_ptr())
    lib.check(rc, "stnerf_train_sample")
    return t.cpu(), mask.cpu(), hit.cpu(), list(counts), list(frac)


def check_hits(mask, hit, counts, n):
    assert counts[0] == n
    for i in range(1, mask.shape[0]):
        want = np.flatnonzero(_np(mask[i]))
        assert counts[i] == want.size, (i, counts[i], want.size)
        assert np.array_equal(_np(hit[i, :counts[i]]), want), i


# ---------------------------------------------------------------------------------------------------------- sample_kernel
@pytest.mark.parametrize("l", [2, 3, 8])            # a context has the background and at least one performer
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 4097])
def test_train_sample_equals_intersect_sample_per_layer(l, n):
    n1 = (3, 64, 90, 128)[(l + n) % 4]
    cols = 6 + l
    boxes = layer_boxes(l)
    nat = context(l, make_scene(boxes))
    rays = tiled_rays(n, cols)
    jit = np.stack([G.jitter_for(n, n1, 3 + i) for i in range(l)])
    t, mask, hit, counts, frac = train_sample(nat, torch.from_numpy(rays).cuda(), n1, torch.from_numpy(jit).cuda())
    for i in range(l):
        g = intersect(torch.from_numpy(rays).cuda(), boxes[i], n1, torch.from_numpy(jit[i]).cuda(), i == 0)
        same(t[i], g[0], "t layer %d vs intersect_sample" % i)
        assert torch.equal(mask[i], g[2])
        w = restated(rays, boxes[i][0], boxes[i][1], n1, jit[i], i == 0, cols)
        same(t[i], w[0], "t layer %d vs restatement" % i)
        assert torch.equal(mask[i], w[2])
    check_hits(mask, hit, counts, n)
    assert frac == [0] * l


@pytest.mark.parametrize("n1", [3, 64, 90, 128])
def test_train_sample_shared_frame_id_and_philox(n1):
    """7-column rays (one sentinel slot), no jitter: the draws of Philox stream i keyed by the mapped ray id, including ids
    past 2^32 (the counter's high word)."""
    l, n = 3, 1000
    boxes = layer_boxes(l)
    nat = context(l, make_scene(boxes, shared=True))
    base, width, row_stride = (1 << 32) - 300, 37, 1000
    nat.set_ray_ids(base, width, row_stride)
    rays = tiled_rays(n, 7)
    t, mask, hit, counts, _ = train_sample(nat, torch.from_numpy(rays).cuda(), n1, None, seed=0x123456789)
    j = np.arange(n)
    ids = (base + (j // width) * row_stride + j % width).astype(np.uint64)
    assert (ids >= 1 << 32).any() and (ids < 1 << 32).any()
    for i in range(l):
        u = TS.philox_uniforms(0x123456789, i, ids, n1)
        w = restated(rays, boxes[i][0], boxes[i][1], n1, u, i == 0, 7)
        same(t[i], w[0], "t layer %d" % i)
        assert torch.equal(mask[i], w[2])
    check_hits(mask, hit, counts, n)


@pytest.mark.parametrize("shared", [False, True])
def test_fractional_frame_ids_count_on_hit_rays_only(shared):
    l, n, n1 = 3, N, 3
    boxes = layer_boxes(l)
    nat = context(l, make_scene(boxes, shared=shared))
    cols = 7 if shared else 6 + l
    rays = tiled_rays(n, cols, fid=2.0)
    _, mask, _, _, frac = train_sample(nat, torch.from_numpy(rays).cuda(), n1)
    m = _np(mask).astype(bool)
    assert frac == [0] * l
    for i in range(1, l):
        col = 6 if shared else 6 + i
        missed, hitr = np.flatnonzero(~m[i]), np.flatnonzero(m[i])
        assert missed.size and hitr.size
        r2 = rays.copy()
        r2[missed, col] = 2.5                                   # a fractional id on every missed ray: ignored
        _, _, _, _, frac = train_sample(nat, torch.from_numpy(r2).cuda(), n1)
        want = [0] * l
        if shared:                                              # one column for every layer: other layers' hits see it
            want = [0] + [int((m[k] & ~m[i]).any()) for k in range(1, l)]
        assert frac == want, (i, frac, want)
        r2[hitr[-1], col] = 3.25                                # ... and one on a hit ray
        _, _, _, _, frac = train_sample(nat, torch.from_numpy(r2).cuda(), n1)
        assert frac[i] == 1


def test_box_table_rows_per_ray():
    """7-column mixed-frame rays clip against the row of their own frame id: ids 1 and F, fractional (truncated), and out
    of range (clamped)."""
    l, F, n1 = 3, 4, 64
    table = np.stack([np.stack([IN["boxes"][(f + i) % 4] for i in range(l)]) for f in range(F)]).astype(np.float32)
    nat = context(l, make_scene([table[0, i] for i in range(l)], shared=True))
    nat.set_box_table(torch.from_numpy(table))
    ids = np.array([1.0, F, 2.5, 3.99, 0.0, -3.7, F + 1.0, 100.0], np.float32)
    rays = tiled_rays(2048, 7)
    rays[:, 6] = np.resize(ids, 2048)
    jit = np.stack([G.jitter_for(2048, n1, 20 + i) for i in range(l)])
    t, mask, hit, counts, _ = train_sample(nat, torch.from_numpy(rays).cuda(), n1, torch.from_numpy(jit).cuda())
    row = np.clip(np.trunc(rays[:, 6]).astype(np.int64) - 1, 0, F - 1)
    assert set(row.tolist()) == set(range(F))
    for i in range(l):
        bx = torch.from_numpy(table[row, i])
        w = restated(rays, bx[:, 0], bx[:, 1], n1, jit[i], i == 0, 7)
        same(t[i], w[0], "t layer %d" % i)
        assert torch.equal(mask[i], w[2])
    check_hits(mask, hit, counts, 2048)


def test_hit_lists_at_the_size_cap():
    """n * 512 < 2^31: 16 384 blocks in the hit scan, 32-bit indices; one more ray is EINVAL."""
    l, n1, n = 2, 3, (1 << 31) // 512 - 1
    boxes = layer_boxes(l)
    nat = context(l, make_scene(boxes))
    rays = torch.from_numpy(tiled_rays(n, 6 + l)).cuda()
    t, mask, hit, counts, _ = train_sample(nat, rays, n1, None, seed=5)
    check_hits(mask, hit, counts, n)
    assert 0 < counts[1] < n
    tail = slice(n - 5000, n)
    w = restated(_np(rays[tail].cpu()), boxes[1][0], boxes[1][1], n1, TS.philox_uniforms(5, 1, np.arange(n - 5000, n), n1), False, 8)
    same(t[1, tail], w[0], "t of the last rays")
    del t, mask, hit
    lib = L()
    big = torch.empty((l, 1), dtype=F32, device="cuda")
    cnt, frac = (C.c_int32 * l)(), (C.c_int32 * l)()
    rc = lib.lib().stnerf_train_sample(nat._h, lib.ptr(rays), n + 1, rays.stride(0), n1, None, 0, lib.ptr(big), lib.ptr(big),
                                       lib.ptr(big), cnt, frac, lib.stream_ptr())
    assert rc == EINVAL


# ---------------------------------------------------------------------------------------------------------- render path
def test_render_chunks_sample_like_intersect_sample():
    """chunk_rays = 64 and a partial last chunk: the ray masks of every chunk and the coarse depths of the last one equal
    intersect_sample on the same rays and jitter (jitter offset c0*n1, layer stride N*n1, capacity strides)."""
    lib = L()
    l, n, n1 = 3, 1000, 5
    boxes = layer_boxes(l)
    nat = context(l, make_scene(boxes, apply_thr=False), chunk_rays=64)
    nat.load_state_dict(O.synthetic_state_dict(l - 1, False))
    rays = tiled_rays(n, 6 + l)
    jit = np.stack([G.jitter_for(n, n1, 40 + i) for i in range(l)])
    _, ray_mask = nat.render(torch.from_numpy(rays).cuda(), n1, 4, only_coarse=True, jitter=torch.from_numpy(jit).cuda())
    c0 = (n // 64) * 64
    for i in range(l):
        g = intersect(torch.from_numpy(rays).cuda(), boxes[i], n1, torch.from_numpy(jit[i]).cuda(), i == 0)
        assert torch.equal(ray_mask[i].cpu(), g[2]), i
        dst = torch.empty((n - c0, n1), dtype=F32, device="cuda")
        lib.check(lib.lib().stnerf_debug_read_depths(nat._h, 0, i, lib.ptr(dst), n - c0, n1, lib.stream_ptr()), "read_depths")
        hitr = _np(g[2][c0:]).astype(bool) if i > 0 else np.ones(n - c0, bool)
        same(dst.cpu()[hitr], g[0][c0:][hitr], "coarse depths of the last chunk, layer %d" % i)


# ---------------------------------------------------------------------------------------------------------- training points
def edit_scene(sc, l, scale, shift, pivot):
    for i in range(l):
        entry = shift[i] if shift is not None else None
        sc.shift_on[i] = 1 if entry is not None else 0
        if entry is not None:
            for a in range(3):
                sc.shift[i][a] = float(np.float32(entry[a]))
        sc.scale_coarse_on[i] = 1 if scale is not None else 0
        sc.scale_fine_on[i] = 1 if (scale is not None and not (shift is not None and entry is None)) else 0
        sc.scale[i] = float(np.float32(scale[i])) if scale is not None else 1.0
    for a in range(3):
        sc.pivot[a] = float(pivot[a])


EDITS = {"none": (None, None),
         "shift": (None, [[0.5, -0.25, 1.0], [0.1, 0.2, -0.3], None]),
         "scale": ([1.0, 0.7, 1.5], None),
         "both": ([0.75, 1.25, 0.6], [[0.0, 0.0, 0.0], None, [-1.5, 0.25, 0.125]])}


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("edit", list(EDITS))
def test_train_points_equal_the_restatement(edit, shared):
    lib = L()
    l, n, n1 = 3, 700, 64
    scale, shift = EDITS[edit]
    pivot = torch.tensor([0.3, -0.2, 0.9], dtype=F32)
    boxes = layer_boxes(l)
    sc = make_scene(boxes, shared=shared)
    edit_scene(sc, l, scale, shift, pivot)
    nat = context(l, sc)
    cols = 7 if shared else 6 + l
    rays = tiled_rays(n, cols)
    rays[:, 6:] = np.arange(cols - 6, dtype=np.float32)[None] + 1.5 + (np.arange(n) % 3)[:, None]
    rd = torch.from_numpy(rays).cuda()
    t, mask, hit, counts, _ = train_sample(nat, rd, n1, torch.from_numpy(np.stack([G.jitter_for(n, n1, i) for i in range(l)])).cuda())
    rt = torch.from_numpy(rays)
    for fine in (0, 1):
        S = n1 if not fine else 90
        tf = t if not fine else torch.sort(torch.rand((l, n, S), generator=torch.Generator().manual_seed(9)) * 6 - 1, -1)[0]
        for i in range(l):
            m = n if i == 0 else counts[i]
            slots = np.arange(n) if i == 0 else _np(hit[i, :m])
            out = [torch.empty((m * S, k), dtype=F32, device="cuda") for k in (3, 3, 1, 4)]
            hp = None if i == 0 else hit[i].cuda()
            td = tf[i].contiguous().cuda()
            lib.check(lib.lib().stnerf_train_points(nat._h, i, fine, lib.ptr(rd), n, cols, lib.ptr(td), S,
                                                    lib.ptr(hp), m, *[lib.ptr(x) for x in out], lib.stream_ptr()),
                      "stnerf_train_points")
            r = rt[slots]
            o, d = r[:, :3], r[:, 3:6]
            xyz = tf[i][slots][..., None] * d[:, None, :] + o[:, None, :]
            pos = O._inverse_edit(xyz, i, scale, shift, pivot, fine=bool(fine)).reshape(-1, 3)
            tm = r[:, 6 + (0 if shared else i)][:, None].expand(m, S).reshape(-1, 1)
            what = "%s layer %d fine %d" % (edit, i, fine)
            same(out[0], pos, "pos " + what)
            same(out[1], d[:, None, :].expand(m, S, 3).reshape(-1, 3), "dirs " + what)
            same(out[2], tm, "times " + what)
            same(out[3], torch.cat([pos, tm], 1), "xyzt " + what)
            # float64: the marched and edited point, to a few ulps of the magnitudes involved
            x64 = tf[i][slots].double()[..., None] * d.double()[:, None, :] + o.double()[:, None, :]
            sh = shift[i] if shift is not None else None
            if sh is not None:
                x64 = x64 - torch.tensor(sh, dtype=F32).double()
            if scale is not None and not (fine and shift is not None and sh is None):
                x64 = (x64 - pivot.double()) / float(np.float32(scale[i])) + pivot.double()
            if fine and shift is not None and sh is None:
                x64 = tf[i][slots].double()[..., None] * d.double()[:, None, :] + o.double()[:, None, :]
            mag = (tf[i][slots].double().abs()[..., None] * d.double().abs()[:, None, :] + o.double().abs()[:, None, :] + 4.0) * 3.0
            assert ((out[0].cpu().double().reshape(m, S, 3) - x64).abs() <= mag * 2.0 ** -21).all(), what


# ---------------------------------------------------------------------------------------------------------- scatter / gather
def pass_restated(layer, fine, t, sg, near, thr, thr_bkgd, apply_thr, alpha2):
    """layered_rfrender.py:414-422 (coarse) / :538-547, :564-576 (fine) on one layer's samples: the kept sigma and the factor."""
    zero = torch.zeros_like(sg)
    off = float("-inf")
    if not fine:
        if layer > 0:
            v = torch.where(t < 0, zero, sg)
            v = torch.where(v < (thr if apply_thr else off), zero, v)
            keep = ~(t < 0) & ~(sg < (thr if apply_thr else off))
        else:
            v = torch.where(t < near, zero, sg)
            keep = ~(t < near)
        return v, keep.to(F32)
    th = thr_bkgd if layer == 0 else thr
    keep = ~(sg < (th if apply_thr else off))
    v = torch.where(keep, sg, zero)
    f = keep.to(F32)
    if layer == 2:
        v = v * alpha2
        f = torch.where(keep, torch.full_like(sg, alpha2), f)
    return v, f


@pytest.mark.parametrize("apply_thr", [True, False])
def test_train_scatter_and_gather(apply_thr):
    lib = L()
    l, n, S = 3, 300, 16
    near, thr, thr_bkgd, alpha2 = 0.5, 0.25, -0.125, 0.375
    nat = context(l, make_scene(layer_boxes(l), near=near, thr=thr, thr_bkgd=thr_bkgd, alpha=alpha2, apply_thr=apply_thr))
    g = torch.Generator().manual_seed(3)
    specials_t = torch.tensor([0.0, -0.0, near, np.nextafter(np.float32(near), np.float32(0)), -1e-30, 1e-30])
    specials_s = torch.tensor([thr, np.nextafter(np.float32(thr), np.float32(-1)), thr_bkgd,
                               np.nextafter(np.float32(thr_bkgd), np.float32(-1)), 0.0, -0.0])
    for fine in (0, 1):
        for i in range(l):
            t = torch.rand((n, S), generator=g) * 4 - 1
            t.view(-1)[:len(specials_t) * 7] = specials_t.repeat(7)
            hitl = None if i == 0 else torch.from_numpy(np.sort(np.random.RandomState(i).choice(n, 170, replace=False))).int()
            m = n if i == 0 else 170
            sg = torch.randn((m * S,), generator=g)
            sg[:len(specials_s) * 5] = specials_s.repeat(5)
            sg[-len(specials_s) * 5:] = specials_s.repeat(5)
            rgb_c = torch.randn((m * S, 3), generator=g)
            rgb = torch.full((n, S, 3), 7.0, device="cuda")
            sigma = torch.full((n, S), 7.0, device="cuda")
            factor = torch.empty((m * S,), device="cuda")
            hp = None if hitl is None else hitl.cuda()
            td, rgb_cd, sgd = t.cuda(), rgb_c.cuda(), sg.cuda()        # held: a freed temporary's block is reused at once
            lib.check(lib.lib().stnerf_train_scatter(nat._h, i, fine, lib.ptr(td), n, S, lib.ptr(hp), m, lib.ptr(rgb_cd),
                                                     lib.ptr(sgd), lib.ptr(rgb), lib.ptr(sigma), lib.ptr(factor),
                                                     lib.stream_ptr()), "stnerf_train_scatter")
            slots = torch.arange(n) if hitl is None else hitl.long()
            tk = t[slots].reshape(-1)
            v, f = pass_restated(i, fine, tk, sg, near, thr, thr_bkgd, apply_thr, alpha2)
            want_sigma = torch.zeros((n, S)); want_sigma[slots] = v.reshape(m, S)
            want_rgb = torch.zeros((n, S, 3)); want_rgb[slots] = rgb_c.reshape(m, S, 3)
            what = "layer %d fine %d" % (i, fine)
            same(sigma, want_sigma, "sigma " + what)
            same(rgb, want_rgb, "rgb " + what)
            same(factor, f, "factor " + what)
            if fine and i == 2:
                assert (f == alpha2).any()
            # gather: d_sigma * factor and d_rgb, in hit order; the adjoint of the scatter in float64
            d_rgb = torch.randn((n, S, 3), generator=g)
            d_sigma = torch.randn((n, S), generator=g)
            d_rgb_c = torch.empty((m * S, 3), device="cuda")
            d_sigma_c = torch.empty((m * S,), device="cuda")
            d_rgbd, d_sigmad = d_rgb.cuda(), d_sigma.cuda()
            lib.check(lib.lib().stnerf_train_gather(nat._h, S, lib.ptr(hp), m, lib.ptr(factor), lib.ptr(d_rgbd),
                                                    lib.ptr(d_sigmad), lib.ptr(d_rgb_c), lib.ptr(d_sigma_c), lib.stream_ptr()),
                      "stnerf_train_gather")
            ds = d_sigma[slots].reshape(-1)
            same(d_sigma_c, torch.where(f != 0, ds * f, torch.zeros_like(ds)), "d_sigma_c " + what)
            same(d_rgb_c, d_rgb[slots].reshape(-1, 3), "d_rgb_c " + what)
            lhs = (sigma.cpu().double() * d_sigma.double()).sum()
            kept = f != 0
            rhs = (sg.double()[kept] * d_sigma_c.cpu().double()[kept]).sum()
            assert abs(float(lhs - rhs)) <= 1e-5 * float((sg.double().abs() * ds.double().abs()).sum()), what


def test_train_uniforms_follow_the_ray_id_map():
    lib = L()
    l, n, n2 = 3, 777, 33
    nat = context(l, make_scene(layer_boxes(l)))
    base, width, row_stride = (1 << 32) - 500, 100, 4096
    nat.set_ray_ids(base, width, row_stride)
    u = torch.empty((l, n, n2), device="cuda")
    lib.check(lib.lib().stnerf_train_uniforms(nat._h, n, n2, 0xABCDEF0123, lib.ptr(u), lib.stream_ptr()), "stnerf_train_uniforms")
    j = np.arange(n)
    ids = (base + (j // width) * row_stride + j % width).astype(np.uint64)
    for i in range(l):
        same(u[i], TS.philox_uniforms(0xABCDEF0123, 64 + i, ids, n2), "u layer %d" % i)


# ---------------------------------------------------------------------------------------------------------- ray generation
def raygen(Kinv, T, H, W, row0, row_step, n_rows, fids, stride):
    lib = L()
    rays = torch.full((n_rows * W * stride,), -9.0, device="cuda")
    fid = torch.tensor(fids, dtype=F32) if fids else None
    rc = lib.lib().stnerf_raygen(lib.ptr(Kinv), lib.ptr(T), H, W, row0, row_step, n_rows, lib.ptr(fid), len(fids),
                                 lib.ptr(rays), stride, lib.stream_ptr())
    return rc, rays.reshape(n_rows * W, stride)


# max |d - d64| in units of 2^-24 (one ulp just below |d| = 1): 2.74 measured on one H100 80GB HBM3 at 700 W (2160x3840)
RAYGEN_ULPS = 3.0


@pytest.mark.parametrize("H,W,row0,row_step", [(2160, 3840, 3, 8), (480, 640, 0, 1), (37, 53, 2, 5)])
def test_raygen_against_float64(H, W, row0, row_step):
    a = 0.7 + 0.1 * row_step
    R64 = torch.tensor([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    R64 = R64 @ torch.tensor([[1.0, 0.0, 0.0], [0.0, np.cos(1.1), -np.sin(1.1)], [0.0, np.sin(1.1), np.cos(1.1)]], dtype=torch.float64)
    T = torch.eye(4, dtype=F32)
    T[:3, :3] = R64.to(F32)
    T[:3, 3] = torch.tensor([1.5, -2.25, 3.0])
    K = torch.tensor([[0.81 * W, 0.0, 0.43 * W], [0.0, 0.79 * W, 0.57 * H], [0.0, 0.0, 1.0]], dtype=F32)
    Kinv = torch.inverse(K).contiguous()
    n_rows = (H + row_step - 1 - row0) // row_step + 1          # the last row lies past H-1 when row_step > 1
    fids = [1.0, 2.5, 7.0]
    rc, rays = raygen(Kinv, T, H, W, row0, row_step, n_rows, fids, 10)
    assert rc == 0
    rows = row0 + row_step * np.arange(n_rows)
    if row_step > 1:
        assert rows[-1] >= H
    jj, ii = np.meshgrid(np.arange(W, dtype=np.float64), rows.astype(np.float64))
    pix = np.stack([jj.ravel(), ii.ravel(), np.ones(jj.size)], 0)
    c = Kinv.double().numpy() @ pix
    c /= np.linalg.norm(c, axis=0)
    d64 = (T[:3, :3].double().numpy() @ c).T
    got = rays.cpu().numpy()
    assert np.array_equal(got[:, :3], np.broadcast_to(T[:3, 3].numpy(), (got.shape[0], 3)))
    assert np.array_equal(got[:, 6:9], np.broadcast_to(np.float32(fids), (got.shape[0], 3)))
    assert (got[:, 9] == -9.0).all()
    ulps = np.abs(got[:, 3:6] - d64).max() / 2.0 ** -24
    print("raygen %dx%d: max |d - d64| = %.2f ulps of |d|" % (H, W, ulps))
    assert ulps <= RAYGEN_ULPS


def test_raygen_rejects_bad_arguments():
    Kinv, T = torch.eye(3), torch.eye(4)
    assert raygen(Kinv, T, 10, 4, 0, 1, 10, [1.0] * 9, 16)[0] == EINVAL          # more than 8 frame ids
    assert raygen(Kinv, T, 10, 4, 0, 1, 10, [1.0, 2.0], 7)[0] == EINVAL          # stride < 6 + ids
    assert raygen(Kinv, T, 10, 4, 10, 1, 1, [], 6)[0] == EINVAL                  # row0 past the image
    assert raygen(Kinv, T, 10, 4, 1, 3, 5, [], 6)[0] == EINVAL                   # last row 13 >= H + row_step
    assert raygen(Kinv, T, 10, 4, 1, 3, 4, [], 6)[0] == 0                        # last row 10: one padding row


# ---------------------------------------------------------------------------------------------------------- positional encoding
# max ulps of sin / cos against float64 over |v| <= 1e4: 1.46 measured on one H100 80GB HBM3 at 700 W (dim 1 and 4,
# n_freq 10), inside the 2 ulps CUDA documents for full-range sincosf
PE_ULPS = 1.5


@pytest.mark.parametrize("dim", [1, 3, 4])
@pytest.mark.parametrize("n_freq", [0, 1, 4, 10])
def test_positional_encoding_against_float64(dim, n_freq):
    from stnerf_b200 import ops
    rs = np.random.RandomState(dim * 16 + n_freq)
    for P in (1, 255, 256, 257, 20000 // dim):
        x = np.clip(rs.standard_normal((P, dim)) * np.exp(rs.uniform(-8, np.log(1e4), (P, dim))), -1e4, 1e4).astype(np.float32)
        x.ravel()[:4] = [1e4, -1e4, 0.0, -0.0][:x.size]
        out = ops.positional_encoding(torch.from_numpy(x).cuda(), n_freq).cpu().numpy()
        assert out.shape == (P, dim * (1 + 2 * n_freq))
        assert np.array_equal(out[:, :dim].view(np.uint32), x.view(np.uint32))
        worst = 0.0
        for k in range(n_freq):
            arg = (x * np.float32(2.0 ** k)).astype(np.float64)          # exact in fp32
            for j, fn in ((1 + 2 * k, np.sin), (2 + 2 * k, np.cos)):
                ref = fn(arg)
                got = out[:, j * dim:(j + 1) * dim].astype(np.float64)
                ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
                worst = max(worst, float((np.abs(got - ref) / ulp).max()))
        print("posenc dim=%d n_freq=%d P=%d: %.2f ulps" % (dim, n_freq, P, worst))
        assert worst <= PE_ULPS
