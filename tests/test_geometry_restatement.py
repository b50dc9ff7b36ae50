"""The CPU oracle's ray/box clipping and stratified sampling against the reference on adversarial rays (geometry.npz), and
the reference's fp32 masks against a float64 slab intersection away from faces, edges and corners.

The fixture's rays are built to land exactly on faces, edges and corners (tests/golden/make_golden_geometry.py); the counts
below pin that each family really takes the branch it was built for.
"""
import numpy as np
import pytest
import torch

import cases as C
import make_golden_geometry as G
from oracle import stnerf_oracle as O

GOLD = C.load_golden("geometry")
IN = G.geometry_inputs()
RAYS = torch.from_numpy(IN["rays"])
BOX = torch.from_numpy(IN["boxes"][IN["box_id"]])
N = RAYS.shape[0]


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def oracle_isect(cols):
    far, near = O.ray_box_intersect(RAYS[:, :3], RAYS[:, 3:6], BOX[:, 0], BOX[:, 1], cols)
    return torch.stack([far, near], 1).numpy()


def test_fixture_shape():
    assert GOLD is not None, "tests/golden/geometry.npz missing (run tests/golden/make_golden_geometry.py)"
    assert N == 1136 and IN["boxes"].shape == (22, 2, 3)
    assert np.bincount(IN["family"]).tolist() == [168, 192, 160, 72, 217, 21, 54, 36, 90, 108, 18]


def test_every_family_takes_its_branch():
    cand = O.ray_box_candidates(RAYS[:, :3], RAYS[:, 3:6], BOX[:, 0], BOX[:, 1])
    valid = (cand != -1000.0).sum(1).numpy()
    assert np.bincount(valid, minlength=7).tolist() == [44, 0, 454, 251, 93, 221, 73]
    fam = IN["family"]
    assert (valid[fam == G.FAMILIES.index("diag")] == 6).sum() == 72
    # the sentinel rows: five or six valid faces, every one of them below t = -1000
    deep = ((cand < -1000.0) | (cand == -1000.0)).all(1).numpy()
    assert ((valid == 5) & deep).sum() == 73 and ((valid == 6) & deep).sum() == 24
    den = RAYS[:, 3:6] + torch.tensor(np.finfo(float).eps, dtype=torch.float32)
    assert int((den == 0).any(1).sum()) == 18                 # d = -2.220446e-16f: t = +-inf or NaN
    assert int(((RAYS[:, 3:6] != 0) & (RAYS[:, 3:6].abs() < np.finfo(np.float32).tiny)).any(1).sum()) == 36
    assert int(((RAYS[:, 3:6] == 0) & torch.signbit(RAYS[:, 3:6])).any(1).sum()) == 18
    # |width| one ulp below, at and one ulp above 1e-5f, for both n1 of the fixture and both layers
    far, near = [torch.from_numpy(x) for x in oracle_isect(7).T]
    T = np.float32(1e-5)
    for n1 in G.GOLDEN_N1:
        for layer in (0, 1):
            start = torch.where((near <= 0) & (layer == 0), torch.zeros_like(near), near)
            w = ((far - start) / n1).abs().numpy()
            for target in (np.nextafter(T, np.float32(0)), T, np.nextafter(T, np.float32(1))):
                assert (w == target).sum() == 3, (n1, layer, target)
            assert GOLD["mask.7.%d.%d" % (layer, n1)][w == T].sum() == 0      # |width| > 1e-5 is strict
            assert GOLD["mask.7.%d.%d" % (layer, n1)][w == np.nextafter(T, np.float32(1))].all()


@pytest.mark.parametrize("cols", G.COLUMNS)
def test_oracle_intersection_reproduces_the_reference(cols):
    assert np.array_equal(bits(oracle_isect(cols)), bits(GOLD["isect.%d" % cols]))


def test_sentinel_rows_depend_on_the_column_count():
    """Six face slots without sentinels (6 columns), one sentinel (7) and two (9) give different top-2s on the rays whose
    valid faces all lie below t = -1000 -- the rows a fixed number of sentinel slots gets wrong."""
    g6, g7, g9 = (GOLD["isect.%d" % c] for c in G.COLUMNS)
    assert (g6 != g7).any(1).sum() == 73 + 24 and (g7 != g9).any(1).sum() == 24
    assert (g6[:, 0] < -1000).sum() == 24 and (g9 == -1000).all(1).sum() == 159
    # a ray through a corner and an edge of [0,1]^3 far behind the origin (the last of the corner_edge family)
    assert GOLD["isect.6"][-19].tolist() == [-1000.0, -2998.5] and GOLD["isect.7"][-19].tolist() == [-1000.0, -1000.0]


@pytest.mark.parametrize("cols", G.COLUMNS)
@pytest.mark.parametrize("n1", G.GOLDEN_N1)
@pytest.mark.parametrize("layer", [0, 1])
def test_oracle_samples_reproduce_the_reference(cols, n1, layer):
    jit = torch.from_numpy(G.jitter_for(N, n1, 10 * layer))
    t, xyz, m = O.stratified_samples(RAYS[:, :3], RAYS[:, 3:6], BOX[:, 0], BOX[:, 1], n1, jit, layer == 0, cols)
    assert np.array_equal(m.numpy().astype(np.uint8), GOLD["mask.%d.%d.%d" % (cols, layer, n1)])
    if n1 == 3:
        assert np.array_equal(bits(t), bits(GOLD["t.%d.%d.3" % (cols, layer)]))
        if cols == 7:
            assert np.array_equal(bits(xyz), bits(GOLD["xyz.7.%d.3" % layer]))


def slab_f64(cols, ulps=8.0):
    """Float64 top-2 of the six face candidates and the sentinels, and which rays lie within `ulps` fp32 ulps of a face,
    edge or corner decision (an in-face test, a zero den, or a tie between candidates)."""
    o = IN["rays"][:, :3].astype(np.float64)
    d = IN["rays"][:, 3:6].astype(np.float64)
    lo, hi = IN["boxes"][IN["box_id"]].astype(np.float64).transpose(1, 0, 2)
    u = ulps * 2.0 ** -23
    cand, near_edge = [], np.zeros(N, bool)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for axis in range(3):
            for face in (lo[:, axis], hi[:, axis]):
                t = (face - o[:, axis]) / (d[:, axis] + np.finfo(float).eps)
                ok = np.ones(N, bool)
                for a in range(3):
                    if a == axis:
                        continue
                    p = t * d[:, a] + o[:, a]
                    scale = np.abs(t * d[:, a]) + np.abs(o[:, a]) + np.abs(lo[:, a]) + np.abs(hi[:, a])
                    ok &= (p >= lo[:, a]) & (p <= hi[:, a])
                    near_edge |= ~np.isfinite(p) | (np.abs(p - lo[:, a]) <= u * scale) | (np.abs(p - hi[:, a]) <= u * scale)
                cand.append(np.where(ok, t, -1000.0))
    cand = np.stack(cand + [np.full(N, -1000.0)] * (cols - 6), 1)
    top = -np.sort(-cand, 1)[:, :2]
    gap = np.abs(top[:, 0] - top[:, 1]) <= u * (np.abs(top[:, 0]) + np.abs(top[:, 1]))
    return top, near_edge | (gap & (top[:, 1] != -1000.0))


@pytest.mark.parametrize("cols", G.COLUMNS)
def test_fp32_masks_agree_with_float64_away_from_edges(cols):
    top, unsure = slab_f64(cols)
    g = GOLD["isect.%d" % cols].astype(np.float64)
    far_ok = ~unsure
    assert far_ok.sum() >= 200, far_ok.sum()           # most of the fixture aims at faces, edges and corners on purpose
    err = np.abs(g[far_ok] - top[far_ok]) / np.maximum(np.abs(top[far_ok]), 1e-30)
    assert err.max() <= 2.0 ** -22, err.max()
    for n1 in G.GOLDEN_N1:
        for layer in (0, 1):
            start = np.where((top[:, 1] <= 0) & (layer == 0), 0.0, top[:, 1])
            w = np.abs(top[:, 0] - start) / n1
            sure = far_ok & (np.abs(w - 1e-5) > 1e-5 * 2.0 ** -18)
            m64 = w > 1e-5
            assert np.array_equal(m64[sure], GOLD["mask.%d.%d.%d" % (cols, layer, n1)][sure].astype(bool)), (n1, layer)
