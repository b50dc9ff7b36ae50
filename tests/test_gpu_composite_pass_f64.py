"""The compositing / resampling pass of the render path (composite_pass_kernel<NT,NZ>, rs::composite_resample_ray<NT,NZ>,
sample_pdf_kernel) against a float64 restatement of the reference's formulas, sample by sample.

Through `ops.composite_pass` (stnerf_composite_pass: the kernel stnerf_render launches, on explicit inputs):
  (a) exact properties of the placement -- t_fine is sort(cat(t, z_new)) bit for bit, the origin map is the permutation that
      says so, ties put the coarse depth first -- over a grid of (n1, n2) that reaches all 16 register instantiations and the
      generic path, on both sides of every multiple of 32; the register path, the generic path and ops.sample_pdf are three
      implementations of one function and must agree bit for bit;
  (b) every image and every new depth against float64, held to a small multiple of the error of the same formulas in torch
      fp32 on the CPU;
  (c) the merged order where depths tie, the single-list shortcut and the brute-force order of a list that does not ascend;
  (d) the SpaceNet kernel's fused warps: a tensor-core render's own t_fine / z_new / src_map obey (a) and do not change when
      the fusion is switched off.
The restatement lives in tests/composite_pass_restatement.py and is pinned to the reference's outputs on the CPU
(tests/test_composite_pass_restatement.py).  Nothing here reads the reference or the oracle."""
import os

import numpy as np
import pytest
import torch

import composite_pass_restatement as R

gpu = pytest.mark.gpu

N1S = [3, 4, 31, 32, 33, 64, 65, 90, 96, 97, 127, 128]
N2S = [1, 31, 32, 33, 64, 65, 96, 128, 129, 192, 256, 257, 320]
LS, NS = [1, 3, 8], [1, 7, 257]


def dispatch(n1, n2, fine=False):
    """The instantiation launch_composite_pass picks (composite.cu): <NT, NZ> register slots per lane, or <0, 0> generic."""
    if fine or n1 > 128 or n2 > 256:
        return (0, 0)
    nzr = (max(n2, 1) + 31) // 32
    return ((n1 + 31) // 32, 1 if nzr <= 1 else 2 if nzr <= 2 else 4 if nzr <= 4 else 8)


def test_grid_reaches_every_instantiation():
    hit = {dispatch(a, b) for a in N1S for b in N2S}
    assert hit == {(nt, nz) for nt in (1, 2, 3, 4) for nz in (1, 2, 4, 8)} | {(0, 0)}
    assert all(a + b <= 512 for a in N1S for b in N2S)
    # the tail word of the occupancy mask: n1 + n2 an exact multiple of 32 and not, in the register path
    assert {(a + b) % 32 == 0 for a in N1S for b in N2S if dispatch(a, b) != (0, 0)} == {True, False}


# ---------------------------------------------------------------------------------------------------------------- inputs
def f32(x):
    return float(np.float32(x))


def make_scene(l, near=0.0, alpha2=1.0, thr=None, hidden=(), boarder=1e10):
    """(dict for the restatement, L.Scene for the library), every constant an fp32 value."""
    from stnerf_b200 import _lib as L
    d = dict(near=f32(near), alpha2=f32(alpha2), thr_layer=f32(thr[0]) if thr else 0.0, thr_bkgd=f32(thr[1]) if thr else 0.0,
             boarder=f32(boarder), apply_thr=thr is not None, shown=[i not in hidden for i in range(l)])
    sc = L.Scene()
    for i in range(l):
        sc.shown[i] = 1 if d["shown"][i] else 0
    sc.near_plane, sc.alpha_layer2, sc.boarder_weight = d["near"], d["alpha2"], d["boarder"]
    sc.density_threshold, sc.bkgd_density_threshold, sc.apply_thresholds = d["thr_layer"], d["thr_bkgd"], int(d["apply_thr"])
    return d, sc


def make_inputs(l, n, S, n2, seed):
    """What the kernel sees in a render, and what it gets wrong: background depths sorted, performer depths from the sampler's
    stratified formula (some boxes start behind the camera: t < 0), density mostly <= 0 with a few dense runs, an opaque sample
    mid-ray, a huge density at the border sample, rays of all-zero weights and of one non-zero weight, colours that tell the
    layers apart, rays that miss performers."""
    rs = np.random.RandomState(seed)
    t = np.empty((l, n, S), np.float64)
    t[0] = np.sort(rs.uniform(0.2, 30.0, (n, S)), 1)
    for i in range(1, l):
        tn = rs.uniform(-0.6, 6.0, (n, 1))
        tf = tn + rs.uniform(0.5, 4.0, (n, 1))
        t[i] = tn + (tf - tn) * ((np.arange(S)[None] + rs.uniform(0, 1, (n, S))) / S)
    t = t.astype(np.float32)
    assert (np.diff(t, axis=-1) >= 0).all()
    sig = rs.normal(-6.0, 4.0, (l, n, S))
    for i in range(l):
        for r in range(n):
            a = rs.randint(S)
            sig[i, r, a:a + rs.randint(1, max(2, S // 6) + 1)] = rs.uniform(0.5, 40.0)
            if r % 5 == 2:
                sig[i, r, S // 2] = 1e4
            if r % 7 == 4:
                sig[i, r, S - 1] = 1e6
            if r % 11 in (3, 5):
                sig[i, r] = -1.0
            if r % 11 == 5:
                sig[i, r, S // 3] = 30.0
    logits = rs.normal(0, 0.7, (l, n, S, 3)) + 3.0 * np.cos(2.1 * np.arange(l)[:, None, None, None] + np.arange(3) * 1.3)
    raw = np.concatenate([logits, sig[..., None]], -1).astype(np.float32)
    mask = rs.uniform(0, 1, (l, n)) < 0.7
    mask[:, 0] = True
    if n > 1:
        mask[1:, 1] = False
    mask[0] = True
    u = np.minimum(rs.random_sample((l, n, max(n2, 1))).astype(np.float32), np.float32(0.99999994))[..., :n2]
    return torch.from_numpy(t), torch.from_numpy(raw), torch.from_numpy(mask), torch.from_numpy(u)


def run_gpu(sc, t, raw, mask, fine=False, n2=0, u=None, generic=False, **kw):
    from stnerf_b200 import ops
    old = os.environ.get("STNERF_PASS_GENERIC")
    os.environ["STNERF_PASS_GENERIC"] = "1" if generic else "0"
    try:
        out = ops.composite_pass(sc, t.cuda(), raw.cuda(), mask.cuda(), fine=fine, n2=n2, u=None if u is None else u.cuda(), **kw)
        torch.cuda.synchronize()
    finally:
        if old is None:
            del os.environ["STNERF_PASS_GENERIC"]
        else:
            os.environ["STNERF_PASS_GENERIC"] = old
    return {k: v.cpu() for k, v in out.items()}


def planes(images, n, layout=0):
    """images (l+1, 5n) -> (l+1, n, 5)."""
    if layout:
        return images.reshape(-1, n, 5)
    return torch.cat([images[:, :3 * n].reshape(-1, n, 3), images[:, 3 * n:4 * n, None], images[:, 4 * n:, None]], -1)


def bits(x):
    return np.ascontiguousarray(x.numpy() if torch.is_tensor(x) else x).view(np.int32)


# ------------------------------------------------------------------------------------------------- (a) exact properties
def check_placement(t, t_fine, z_new=None, src_map=None):
    """Rows = hit (ray, layer) pairs.  t (m,n1), t_fine (m,n1+n2), z_new (m,n2), src_map (m,n1+n2) as numpy."""
    m, n1 = t.shape
    S2 = t_fine.shape[1]
    assert (np.diff(t_fine, axis=1) >= 0).all()
    if z_new is None:
        return
    assert (np.diff(z_new, axis=1) >= 0).all(), "z_new ascends"
    cat = np.concatenate([t, z_new], 1)
    assert np.array_equal(bits(t_fine), bits(np.sort(cat, 1))), "t_fine == sort(cat(t, z_new)) bit for bit"
    src = src_map.astype(np.int64)
    assert np.array_equal(np.sort(src, 1), np.broadcast_to(np.arange(S2), src.shape)), "src_map is a permutation"
    assert np.array_equal(bits(np.take_along_axis(cat, src, 1)), bits(t_fine)), "t_fine[p] is the depth src_map[p] names"
    pos = np.argsort(src, 1)                          # inverse permutation: where each source landed
    assert (np.diff(pos[:, :n1], axis=1) > 0).all() and (np.diff(pos[:, n1:], axis=1) > 0).all(), "each list keeps its order"
    # a new depth lands after every coarse depth <= it: equal depths put the coarse one first
    rank = (t[:, None, :] <= z_new[:, :, None]).sum(-1)
    assert np.array_equal(pos[:, n1:], rank + np.arange(S2 - n1)[None]), "ties: coarse first"


def leftover(t, t_fine):
    """t_fine (m,S2) minus the sub-multiset t (m,n1), bitwise -> (m, n2) in ascending order.  Rows ascend."""
    out = []
    for a, b in zip(t, t_fine):
        idx = np.searchsorted(b, a, "left") + np.arange(len(a)) - np.searchsorted(a, a, "left")   # k-th copy of a value -> k-th slot
        assert idx.max() < len(b) and np.array_equal(bits(b[idx]), bits(a)), "t_fine contains every coarse depth"
        keep = np.ones(len(b), bool)
        keep[idx] = False
        out.append(b[keep])
    return np.stack(out)


def z_reference(d, t, raw, mask, u):
    """float64 new depths + the tolerance each deserves, from the restatement in float64 and (the yardstick) in fp32."""
    o64 = R.run_pass(d, False, t.double(), raw.double(), mask, u.double())
    o32 = R.run_pass(d, False, t, raw, mask, u)
    l = t.shape[0]
    z64, tol, aside = [], [], []
    for i in range(l):
        p64, p32 = o64["pdf"][i], o32["pdf"][i]
        eps = (p32["cdf"].double() - p64["cdf"]).abs().amax(-1, keepdim=True).clamp(min=2.0 ** -22)     # per ray
        width = (p64["ba"] - p64["bb"]).abs()
        ulp = torch.maximum(p64["ba"].abs(), p64["bb"].abs()) * 2.0 ** -23
        tol.append(width * (8 * eps + 2.0 ** -23) / p64["den"] + 4 * ulp)
        d_below = (u[i].double() - p64["cb"]).abs()
        d_below[p64["below"] == 0] = 1.0                 # cdf[0] = 0 exactly, in every implementation: no doubt about that knot
        knot = torch.minimum(d_below, (u[i].double() - p64["ca"]).abs())
        aside.append((knot < torch.clamp(8 * eps, min=4e-6)) | ((p64["den_raw"] - 1e-5).abs() < torch.clamp(8 * eps, min=4e-6)))
        z64.append(o64["z"][i])
    return torch.stack(z64).numpy(), torch.stack(tol).numpy(), torch.stack(aside).numpy()


def check_z(z_gpu_sorted, z64, tol, aside):
    """z_gpu_sorted (m,n2) ascending, against float64 draws z64 (m,n2) in draw order.  Rays without a set-aside sample: sorted
    against sorted, one to one.  Rays with one (its `den < 1e-5` or its bin may legitimately go either way, moving it within its
    bin and shifting the ranks between): every other float64 depth has a kernel depth within its tolerance."""
    worst = 0.0
    for zg, zr, tl, sa in zip(z_gpu_sorted.astype(np.float64), z64, tol, aside):
        if not sa.any():
            o = np.argsort(zr, kind="stable")
            tls = tl[o]
            tls = np.maximum(tls, np.maximum(np.roll(tls, 1), np.roll(tls, -1)))
            ratio = np.abs(zg - zr[o]) / tls
        else:
            k = np.clip(np.searchsorted(zg, zr), 1, len(zg) - 1) if len(zg) > 1 else np.zeros(len(zr), int)
            near = np.minimum(np.abs(zg[k] - zr), np.abs(zg[np.maximum(k - 1, 0)] - zr))
            ratio = (near / tl)[~sa]
        if ratio.size:
            worst = max(worst, float(ratio.max()))
    return worst


STATS = {"aside": 0, "z": 0, "z_ratio": 0.0}


def placement_case(n1, n2, l, n, seed, u=None, dup_first=False, count=True):
    from stnerf_b200 import ops
    d, sc = make_scene(l, near=0.8, hidden=(2,) if l > 2 else ())
    t, raw, mask, u0 = make_inputs(l, n, n1, n2, seed)
    u = u0 if u is None else u(u0)
    if dup_first:
        t[:, :, 1] = t[:, :, 0]                       # bins[0] == t[0] == t[1]: a new depth drawn with u = 0 ties with both
    regs = dispatch(n1, n2) != (0, 0)
    origin = regs and n1 + n2 <= 256
    sentinel = -777.0
    tf0 = torch.full((l, n, n1 + n2), sentinel).cuda()
    got = run_gpu(sc, t, raw, mask, n2=n2, u=u, want_origin=origin, t_fine=tf0)
    hit = mask.clone()
    hit[0] = True
    hm = hit.numpy()
    tf = got["t_fine"].numpy()
    assert (tf[~hm] == sentinel).all(), "rows of missed layers stay untouched"
    img = planes(got["images"], n).numpy()
    assert (img[1:][~hm] == 0).all(), "a missed layer's pixel is exactly zero"
    tn = t.numpy()
    check_placement(tn[hm], tf[hm], got["z_new"].numpy()[hm] if origin else None, got["src_map"].numpy()[hm] if origin else None)
    z_sorted = got["z_new"].numpy()[hm] if origin else leftover(tn[hm], tf[hm])
    # new depths stay inside [bins[0], bins[-1]] to one rounding of bb + tt (ba - bb)
    lo, hi = 0.5 * (tn[hm][:, 0] + tn[hm][:, 1]), 0.5 * (tn[hm][:, -1] + tn[hm][:, -2])
    slack = 2.0 ** -22 * np.maximum(np.abs(lo), np.abs(hi))
    assert (z_sorted >= (lo - slack)[:, None]).all() and (z_sorted <= (hi + slack)[:, None]).all()
    z64, tol, aside = z_reference(d, t, raw, mask, u)
    if count:
        STATS["aside"] += int(aside[hm].sum())
        STATS["z"] += int(hm.sum()) * n2
    worst = check_z(z_sorted, z64[hm], tol[hm], aside[hm])
    STATS["z_ratio"] = max(STATS["z_ratio"], worst)
    assert worst <= 1.0, "new depth off float64 by %.2f x its conditioned tolerance (n1=%d n2=%d)" % (worst, n1, n2)
    # three implementations of one function
    if regs:
        gen = run_gpu(sc, t, raw, mask, n2=n2, u=u, generic=True, t_fine=tf0.clone().fill_(sentinel))
        assert np.array_equal(bits(gen["t_fine"]), bits(tf)), "generic path == register path"
        assert np.array_equal(bits(gen["images"]), bits(got["images"]))
    for i in range(l):
        sg = R.mask_density(d, i, False, t[i], raw[i, ..., 3])
        lg = raw[i, ..., :3] if d["shown"][i] else torch.zeros_like(raw[i, ..., :3])
        c, dep, acc, w = ops.composite(t[i].cuda(), lg.cuda(), sg.cuda(), boarder=d["boarder"])
        pix = torch.cat([c, dep, acc], 1).cpu().numpy()
        assert np.array_equal(bits(pix[hm[i]]), bits(img[1 + i][hm[i]])), "stnerf_composite's pixel is the pass kernel's"
        _, tf3 = ops.sample_pdf(t[i].cuda(), w, u[i].cuda(), merge=True)
        assert np.array_equal(bits(tf3.cpu().numpy()[hm[i]]), bits(tf[i][hm[i]])), "stnerf_sample_pdf's merge == the pass kernel's"
    return got, (t, raw, mask, u)


@gpu
@pytest.mark.parametrize("n1", N1S)
def test_placement_grid(n1):
    for k, n2 in enumerate(N2S):
        j = N1S.index(n1) + k
        placement_case(n1, n2, LS[j % 3], NS[(j // 3) % 3], seed=1000 * n1 + n2)
    print("placement n1=%d: worst z / tolerance %.3f, set aside %d of %d" % (n1, STATS["z_ratio"], STATS["aside"], STATS["z"]))
    assert STATS["aside"] < 0.01 * STATS["z"]


@gpu
@pytest.mark.parametrize("kind", ["equal", "zero", "below_one", "ties"])
@pytest.mark.parametrize("n1,n2", [(3, 33), (64, 128), (97, 96), (128, 128), (33, 320)])
def test_degenerate_uniforms(kind, n1, n2):
    one = float(np.nextafter(np.float32(1), np.float32(0)))
    fill = {"equal": 0.37, "zero": 0.0, "below_one": one, "ties": 0.0}[kind]
    placement_case(n1, n2, 3, 7, seed=5 + n1, u=lambda u0: torch.full_like(u0, fill), dup_first=kind == "ties", count=False)


@gpu
def test_uniform_on_a_cdf_knot():
    """Uniforms that sit on the knots of the cdf: a ray of all-zero weights has the uniform pdf, whose knots are k / (n1 - 2).
    Which of the two bins a draw on a knot falls into is round-off's choice; the inverse cdf is continuous there, so the depth
    is the same either way, and the exact properties hold regardless."""
    n1, n2, l, n = 34, 64, 1, 7
    d, sc = make_scene(l)
    t, raw, mask, _ = make_inputs(l, n, n1, n2, 9)
    raw[..., 3] = -1.0
    u = (torch.arange(n2) % (n1 - 1)).float().div(n1 - 2).clamp(max=0.99999994).expand(l, n, n2).contiguous()
    got = run_gpu(sc, t, raw, mask, n2=n2, u=u, want_origin=True)
    check_placement(t[0].numpy(), got["t_fine"][0].numpy(), got["z_new"][0].numpy(), got["src_map"][0].numpy())
    z64 = R.run_pass(d, False, t.double(), raw.double(), mask, u.double())["z"][0].numpy()
    width = np.diff(t[0].numpy().astype(np.float64), axis=1).max()
    assert np.abs(np.sort(z64, 1) - got["z_new"][0].numpy()).max() < 1e-5 * width + 1e-5     # a uniform pdf: continuous across knots


@gpu
def test_position_block_and_layout_do_not_matter():
    n1, n2, l, n = 64, 128, 3, 257
    d, sc = make_scene(l, near=0.8, alpha2=0.5, thr=(0.7, 0.9))
    t, raw, mask, u = make_inputs(l, n, n1, n2, 77)
    a = run_gpu(sc, t, raw, mask, n2=n2, u=u, want_origin=True)
    perm = torch.from_numpy(np.random.RandomState(1).permutation(n))
    b = run_gpu(sc, t[:, perm], raw[:, perm], mask[:, perm], n2=n2, u=u[:, perm], want_origin=True)
    hm = mask.clone()
    hm[0] = True
    for k in ("t_fine", "z_new", "src_map"):
        x, y = a[k][:, perm].numpy(), b[k].numpy()
        assert np.array_equal(x[hm[:, perm].numpy()], y[hm[:, perm].numpy()]), k
    assert np.array_equal(bits(planes(a["images"], n)[:, perm]), bits(planes(b["images"], n)))
    one = run_gpu(sc, t[:, 200:201], raw[:, 200:201], mask[:, 200:201], n2=n2, u=u[:, 200:201])
    assert np.array_equal(bits(planes(one["images"], 1)), bits(planes(a["images"], n)[:, 200:201]))
    c = run_gpu(sc, t, raw, mask, n2=n2, u=u, pixel_layout=1)
    assert np.array_equal(bits(planes(c["images"], n, 1)), bits(planes(a["images"], n)))
    p0 = run_gpu(sc, t, raw, mask, fine=True)
    p1 = run_gpu(sc, t, raw, mask, fine=True, pixel_layout=1)
    assert np.array_equal(bits(planes(p0["images"], n)), bits(planes(p1["images"], n, 1)))


@gpu
def test_philox_draws_are_the_documented_stream():
    from tests_support import philox_uniforms
    n1, n2, l, n, seed = 64, 96, 3, 40, 0x1234567887654321
    d, sc = make_scene(l)
    t, raw, mask, _ = make_inputs(l, n, n1, n2, 3)
    a = run_gpu(sc, t, raw, mask, n2=n2, u=None, seed=seed, want_origin=True)
    u = torch.from_numpy(np.stack([philox_uniforms(seed, 64 + i, np.arange(n, dtype=np.uint64), n2) for i in range(l)]))
    b = run_gpu(sc, t, raw, mask, n2=n2, u=u, want_origin=True)
    for k in ("t_fine", "z_new", "src_map"):
        assert np.array_equal(a[k].numpy(), b[k].numpy()), k


@gpu
def test_arguments_outside_the_abi_are_refused():
    import ctypes
    from stnerf_b200 import _lib as L
    d, sc = make_scene(3)
    buf = torch.zeros(1 << 16, device="cuda")
    p = L.ptr(buf)

    def call(l=3, fine=0, S=64, n2=0, layout=0, images=p, t_fine=None, z=None, src=None, n=2, mask=p):
        return L.lib().stnerf_composite_pass(ctypes.byref(sc), l, fine, p, p, mask, None, 0, n, S, n2, layout, images, t_fine, z, src,
                                             L.stream_ptr())
    assert call(n=0) == 0
    for bad in (dict(S=2), dict(S=129), dict(S=128, n2=385, t_fine=p), dict(l=0), dict(l=9), dict(fine=1, S=513), dict(fine=1, S=0),
                dict(fine=1, n2=8, t_fine=p), dict(n2=-1), dict(n2=8), dict(n2=0, t_fine=p), dict(images=None), dict(layout=2),
                dict(fine=2), dict(n=-1), dict(mask=None), dict(n2=64, t_fine=p, z=p), dict(n2=64, t_fine=p, src=p),
                dict(n2=257, t_fine=p, z=p, src=p), dict(S=128, n2=192, t_fine=p, z=p, src=p), dict(z=p, src=p),
                dict(fine=1, z=p, src=p)):
        assert call(**bad) == -1, bad
    os.environ["STNERF_PASS_GENERIC"] = "1"
    try:
        assert call(n2=64, t_fine=p, z=p, src=p) == -1          # the generic path writes no origin map
    finally:
        del os.environ["STNERF_PASS_GENERIC"]
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- (b) values against float64
OUTPUTS = (("merged rgb", slice(0, 1), slice(0, 3)), ("merged depth", slice(0, 1), slice(3, 4)), ("merged acc", slice(0, 1), slice(4, 5)),
           ("layer rgb", slice(1, None), slice(0, 3)), ("layer depth", slice(1, None), slice(3, 4)), ("layer acc", slice(1, None), slice(4, 5)))
RATIOS = {}
# The kernels scan in shuffle-tree order, sum 32 lane partials and squash colours with 1 / (1 + expf(-x)); ATen's cumprod, sums and
# sigmoid round less.  Measured on an H100, worst over every test of this file, the kernel's error is (rms, max) x the
# yardstick's: merged rgb 5.2, 4.6; merged depth 5.8, 7.4; merged acc 3.7, 3.7; layer rgb 3.0, 4.6; layer depth 2.8, 2.2;
# layer acc 3.5, 4.2 -- under 1e-6 on a colour.  A sample attributed to the wrong layer or composited in the wrong order moves
# a pixel by 1e-3 or more.
BUDGET = 10.0


class Yardstick:
    """Pools |kernel - float64| and |torch fp32 on the CPU - float64| per output over the cases of one test, then holds the
    kernel's rms and max to BUDGET times the yardstick's."""

    def __init__(self):
        self.acc = {name: [0.0, 0.0, 0.0, 0.0, 0, 1.0] for name, _, _ in OUTPUTS}      # k sq, k max, y sq, y max, count, scale

    def add(self, d, sc, t, raw, mask, fine):
        n = t.shape[1]
        got = planes(run_gpu(sc, t, raw, mask, fine=fine)["images"], n).double()
        want = R.run_pass(d, fine, t.double(), raw.double(), mask)["images"]
        yard = R.run_pass(d, fine, t, raw, mask)["images"].double()
        for name, rows, ch in OUTPUTS:
            ek, ey, a = (got - want)[rows, :, ch].abs(), (yard - want)[rows, :, ch].abs(), self.acc[name]
            a[0] += float(ek.pow(2).sum()); a[1] = max(a[1], float(ek.max()))
            a[2] += float(ey.pow(2).sum()); a[3] = max(a[3], float(ey.max()))
            a[4] += ek.numel(); a[5] = max(a[5], float(want[rows, :, ch].abs().max()))
        return got, want

    def hold(self, what):
        for name, (ksq, kmax, ysq, ymax, cnt, scale) in self.acc.items():
            floor = 2.0 ** -23 * scale                # an output the CPU's fp32 happens to get exactly right still rounds once
            krms, yrms = (ksq / cnt) ** 0.5, max((ysq / cnt) ** 0.5, floor / 4)
            r = RATIOS.setdefault(name, [0.0, 0.0])
            r[0], r[1] = max(r[0], krms / yrms), max(r[1], kmax / max(ymax, floor))
            assert krms <= BUDGET * yrms, "%s %s: rms %.3e vs fp32 yardstick %.3e" % (what, name, krms, yrms)
            assert kmax <= BUDGET * max(ymax, floor), "%s %s: max %.3e vs fp32 yardstick %.3e" % (what, name, kmax, ymax)
        print("%s: kernel / yardstick error (rms, max): %s" % (what, {k: "%.2f %.2f" % tuple(v) for k, v in RATIOS.items()}))


def place_thresholds(raw, thr_layer, thr_bkgd):
    """Densities exactly at, one ulp below and one ulp above each threshold, early in the ray where they carry weight."""
    for i, th in [(0, thr_bkgd)] + [(i, thr_layer) for i in range(1, raw.shape[0])]:
        th = np.float32(th)
        for k, v in enumerate((th, np.nextafter(th, np.float32(-1e9)), np.nextafter(th, np.float32(1e9)))):
            raw[i, k::3, 1 + k, 3] = float(v)
    return raw


SCENES = {"plain": dict(), "near": dict(near=6.0), "thresholds": dict(thr=(0.75, 1.25)), "alpha": dict(alpha2=0.3),
          "hidden": dict(hidden=(1, 2)), "all": dict(near=4.0, thr=(0.75, 1.25), alpha2=0.3, hidden=(1,))}


@gpu
@pytest.mark.parametrize("switch", sorted(SCENES))
def test_images_against_float64(switch):
    y = Yardstick()
    for fine, S, l in [(False, 64, 3), (False, 3, 8), (False, 128, 8), (False, 97, 1), (True, 2, 3), (True, 33, 8), (True, 192, 8),
                       (True, 256, 3), (True, 512, 3), (True, 192, 1)]:
        kw = dict(SCENES[switch])
        kw["hidden"] = tuple(i for i in kw.get("hidden", ()) if i < l)
        d, sc = make_scene(l, **kw)
        t, raw, mask, _ = make_inputs(l, 129, S, 0, seed=S + 7 * l + fine)
        if "thr" in kw and S >= 4:
            raw = place_thresholds(raw, *kw["thr"])
        y.add(d, sc, t, raw, mask, fine)
    y.hold(switch)


# ------------------------------------------------------------------------------------------------- (c) the merged order
def tie_inputs(kind, l, n, S, seed):
    t, raw, mask, _ = make_inputs(l, n, S, 0, seed)
    mask[:] = True
    raw[..., 3] = raw[..., 3].clamp(min=0.05, max=3.0)               # every sample absorbs a little: the order shows
    if kind == "performers":                                          # same box, same jitter, different density and colour
        t[1:] = t[1:2]
    elif kind == "background":                                        # a performer shares every other depth with the background
        t[1] = t[0]
        t[1, :, 1:-1:2] = 0.5 * (t[0, :, 0:-2:2] + t[0, :, 2::2])
        t[1] = torch.sort(t[1], -1)[0]
    elif kind == "all_equal":
        t[:] = 2.0
    return t, raw, mask


@gpu
@pytest.mark.parametrize("fine", [False, True])
@pytest.mark.parametrize("kind,l", [("performers", 3), ("performers", 8), ("background", 3), ("all_equal", 3), ("all_equal", 8)])
def test_ties_follow_concatenation_order(kind, l, fine):
    n, S = 33, 64 if not fine else 96
    d, sc = make_scene(l, near=0.0)
    t, raw, mask = tie_inputs(kind, l, n, S, seed=l + 10 * fine)
    y = Yardstick()
    got, want = y.add(d, sc, t, raw, mask, fine)
    y.hold("ties %s l=%d" % (kind, l))
    got, want = got[0], want[0]
    wrong = R.run_pass(d, fine, t.double(), raw.double(), mask, reverse_ties=True)["images"][0]
    e_right, e_wrong = (got - want)[:, :3].abs().max(), (got - wrong)[:, :3].abs().max()
    assert e_wrong > 1e-2 and e_wrong > 1e3 * e_right, (float(e_right), float(e_wrong))       # the case tells the orders apart


@gpu
@pytest.mark.parametrize("fine", [False, True])
def test_single_list_shortcut_is_the_full_merge(fine):
    """A ray that hits only the background takes the shortcut (its merged pixel is the background's own); with a hit but hidden
    performer parked behind the background's last depth the same samples go through the full merge: the same bits, as long as
    the background's last sample has no weight (its delta is then the only thing that changed)."""
    n, S = 65, 96
    d1, sc1 = make_scene(1, near=0.0)
    t, raw, mask, _ = make_inputs(1, n, S, 0, 21)
    raw[0, :, -1, 3] = -1.0
    a = planes(run_gpu(sc1, t, raw, mask, fine=fine)["images"], n)
    assert np.array_equal(bits(a[0]), bits(a[1]))
    d2, sc2 = make_scene(2, near=0.0, hidden=(1,))
    t2 = torch.cat([t, t[:, :, -1:] + 1.0 + torch.arange(S).float()[None, None]], 0)
    raw2 = torch.cat([raw, torch.full_like(raw, 5.0)], 0)
    b = planes(run_gpu(sc2, t2, raw2, torch.ones(2, n, dtype=torch.bool), fine=fine)["images"], n)
    assert np.array_equal(bits(b[0]), bits(a[0])) and np.array_equal(bits(b[1]), bits(a[1]))
    # a sample in front of the near plane: the fine merge cuts it, the layer's own image does not -- no shortcut there
    d3, sc3 = make_scene(1, near=8.0)
    raw3 = raw.clone()
    raw3[0, :, :4, 3] = 2.0
    y = Yardstick()
    c, _ = y.add(d3, sc3, t, raw3, mask, fine)
    y.hold("near plane, one list")
    if fine:
        assert (c[0] - c[1]).abs().max() > 1e-2


@gpu
@pytest.mark.parametrize("signed_zero", [False, True])
def test_a_list_that_does_not_ascend(signed_zero):
    """The brute-force order (a list out of order: degenerate boxes).  The reference's torch.sort is a comparison sort: -0.0 and
    +0.0 are equal there and stay in concatenation order, so the kernel's integer keys must not tell them apart either."""
    l, n, S = 3, 33, 64
    d, sc = make_scene(l, near=0.0)
    t, raw, mask, _ = make_inputs(l, n, S, 0, 31)
    mask[:] = True
    raw[..., 3] = raw[..., 3].clamp(min=0.05, max=3.0)
    t[1:] = t[1:].clamp(min=0.01)
    k = S // 2
    t[1, :, [k, k + 1]] = t[1, :, [k + 1, k]] + torch.tensor([1e-3, 0.0])          # out of order by a hair
    raw[1, :, k:k + 2, 3] = -1.0                                                    # (zero density there: alpha stays in [0, 1])
    assert (t[1, :, k] > t[1, :, k + 1]).all()
    if signed_zero:
        t[1, :, 0], t[2, :, 0] = 0.0, -0.0                                          # +0.0 of list 1, then -0.0 of list 2
        raw[1:, :, 0, 3] = 3.0
        assert bits(t[2, :, 0])[0] != bits(t[1, :, 0])[0]
    y = Yardstick()
    got, want = y.add(d, sc, t, raw, mask, False)
    y.hold("non-ascending list")
    if signed_zero:
        # what ordering -0.0 before +0.0 would composite: the same densities and colours, list 2's zero moved a hair forward
        t64, raw64 = t.double(), raw.double()
        keys = [t64[0], t64[1], t64[2].clone()]
        keys[2][:, 0] = -1e-30
        wrong = R.merged_pixel(d, False, keys, [raw64[i, ..., :3] for i in range(l)],
                               [R.mask_density(d, i, False, t64[i], raw64[i, ..., 3]) for i in range(l)])
        assert (want[0] - wrong)[:, :3].abs().max() > 1e-3
        assert (got[0] - want[0])[:, :3].abs().max() < 1e-5


# --------------------------------------------------------------------------------- (d) the fused warps and the render path
def render_placements(no_fuse):
    """t_coarse, t_fine, z_new, src_map, mask of every layer and the images of a tensor-core render with n1 = 64."""
    from stnerf_b200 import NativeRenderer
    from stnerf_b200.synthetic import synthetic_state_dict
    l, n, n1, n2 = 3, 300, 64, 128
    old = os.environ.get("STNERF_NO_FUSE")
    os.environ["STNERF_NO_FUSE"] = "1" if no_fuse else "0"
    try:
        r = NativeRenderer(l, [False, True, True], "exact")
    finally:
        if old is None:
            del os.environ["STNERF_NO_FUSE"]
        else:
            os.environ["STNERF_NO_FUSE"] = old
    r.load_state_dict(synthetic_state_dict(l - 1, True, seed=5))
    _, sc = make_scene(l, near=0.3, thr=(0.2, 0.1), hidden=(2,), alpha2=0.6)
    boxes = [((-4, -4, -4), (4, 4, 4)), ((-1.0, -0.8, -0.6), (0.7, 0.9, 0.8)), ((-0.3, -1.0, -0.9), (1.1, 0.4, 0.5))]
    for i, (lo, hi) in enumerate(boxes):
        for a in range(3):
            sc.bmin[i][a], sc.bmax[i][a] = lo[a], hi[a]
    sc.shared_frame_id = 0
    r.set_scene(sc)
    rs = np.random.RandomState(11)
    o = rs.normal(0, 0.3, (n, 3)) + np.array([0, 0, -3.0])
    dirs = rs.normal(0, 0.25, (n, 3)) + np.array([0, 0, 1.0])
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rays = torch.from_numpy(np.concatenate([o, dirs, np.full((n, l), 3.0)], 1).astype(np.float32)).cuda()
    out, mask = r.render(rays, n1, n2, seed=99)
    res = {"images": out.cpu(), "mask": mask.cpu().bool()}
    for i in range(l):
        res["t%d" % i] = r.read_depths(False, i, n, n1).cpu()
        res["tf%d" % i] = r.read_depths(True, i, n, n1 + n2).cpu()
        z, src = r.read_origin(i, n, n1, n2)
        res["z%d" % i], res["src%d" % i] = z.cpu(), src.cpu()
    r.close()
    return res, l


@gpu
def test_fused_warps_place_the_same_samples():
    fused, l = render_placements(no_fuse=False)
    alone, _ = render_placements(no_fuse=True)
    assert fused["mask"][1].any() and fused["mask"][2].any() and not fused["mask"][1].all()
    for i in range(l):
        hit = fused["mask"][i].numpy() if i else np.ones(fused["mask"].shape[1], bool)
        check_placement(fused["t%d" % i].numpy()[hit], fused["tf%d" % i].numpy()[hit], fused["z%d" % i].numpy()[hit],
                        fused["src%d" % i].numpy()[hit])
        for k in ("t", "tf", "z", "src"):
            a, b = fused["%s%d" % (k, i)].numpy()[hit], alone["%s%d" % (k, i)].numpy()[hit]
            assert np.array_equal(a, b), "layer %d %s differs between the fused and the stand-alone coarse pass" % (i, k)
    assert torch.equal(fused["images"], alone["images"])
