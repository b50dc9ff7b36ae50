"""Geometry extraction on the host: the default grid box of `layer_density` is the render's clipping box, `write_ply` round-trips,
and the marching-cubes table closes and orients every surface of the float64 restatement (tests/mc_restatement.py)."""
import numpy as np
import pytest
import torch

import cases as C
import mc_restatement as M
import train_restatement as TR
from stnerf_b200 import extract as X
from stnerf_b200 import scene_data as SD
from tests_support import make_cfg

SYN = C.CASES["syn_L2_64_128"]
EDITS = {
    "none": {},
    "scale_shift": dict(scale=[1, 0.75, 1.5], shift=[[0, 0, 0], [0, 2, 0], [0, -2, 0]]),
    "none_shift": dict(scale=[1.1, 0.9, 1.2], shift=[[0.5, 0, 0], None, [0, -0.5, 0.25]]),
}


@pytest.mark.parametrize("edit", sorted(EDITS))
@pytest.mark.parametrize("frame", [1.0, 10.0, 10.5, 37.25, 100.0])
def test_default_box_is_the_render_clipping_box(edit, frame):
    case = dict(SYN, **EDITS[edit])
    import modeling
    model = modeling.build_layered_model(make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], "fp32"), 0,
                                         case.get("scale"), case.get("shift"))
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model.retiming = False                          # extraction resolves in the retiming layout whatever the last forward used
    want = TR.scene(dict(case, frame_ids=[0.0] + [frame] * case["L"]), dtype=torch.float32)
    for layer in range(case["L"] + 1):              # layer 0: the background box
        lo, hi = X.layer_box(model, layer, frame)
        assert torch.equal(torch.tensor(lo), want["bmin"][layer]), (layer, lo, want["bmin"][layer])
        assert torch.equal(torch.tensor(hi), want["bmax"][layer]), (layer, hi, want["bmax"][layer])
    assert model.retiming is False


def test_grid_spans_the_box():
    origin, step, dims = X._grid((-1.0, 0.0, 2.0), (1.0, 3.0, 2.5), (5, 7, 2))
    assert dims == (5, 7, 2) and origin == (-1.0, 0.0, 2.0)
    assert step == (0.5, 0.5, 0.5)
    assert X._grid((0, 0, 0), (1, 1, 1), 4)[2] == (4, 4, 4)
    with pytest.raises(ValueError):
        X._grid((0, 0, 0), (1, 1, 1), (4, 1, 4))


@pytest.mark.parametrize("colors", [True, False])
def test_write_ply_round_trips(tmp_path, colors):
    g = torch.Generator().manual_seed(5)
    verts = torch.randn((257, 3), generator=g) * 3.0
    faces = torch.randint(0, 257, (500, 3), generator=g)
    col = torch.rand((257, 3), generator=g) if colors else None
    p = str(tmp_path / "m.ply")
    X.write_ply(p, X.Mesh(verts, faces, col))
    back = SD.read_ply_points(p)
    assert np.array_equal(back, verts.numpy().astype(np.float64))
    raw = open(p, "rb").read()
    head = raw[:raw.index(b"end_header\n") + len(b"end_header\n")].decode()
    assert "element face 500" in head and "format binary_little_endian 1.0" in head
    assert ("property uchar red" in head) == colors
    vsize = 12 + (3 if colors else 0)
    body = raw[len(head):]
    assert len(body) == 257 * vsize + 500 * 13
    fr = np.frombuffer(body[257 * vsize:], dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    assert (fr["n"] == 3).all() and np.array_equal(fr["i"], faces.numpy())
    if colors:
        vr = np.frombuffer(body[:257 * vsize], dtype=np.dtype([("xyz", "<f4", (3,)), ("rgb", "u1", (3,))]))
        assert np.array_equal(vr["rgb"], np.rint(col.numpy().astype(np.float64) * 255).astype(np.uint8))


def test_write_ply_empty_mesh(tmp_path):
    p = str(tmp_path / "e.ply")
    X.write_ply(p, X.Mesh(torch.zeros((0, 3)), torch.zeros((0, 3), dtype=torch.int64), None))
    assert SD.read_ply_points(p).shape == (0, 3)


def test_table_cases_close_and_orient():
    """Every single-cube case of the table: on a 2x2x2 grid padded with an outside layer the surface is closed, wound
    consistently and encloses a positive volume; the 256 cases need at most 5 triangles."""
    ntri, tri = M.load_table()
    assert ntri.max() <= 5 and ntri[0] == 0 and ntri[255] == 0
    for cs in range(1, 256):
        g = np.full((4, 4, 4), -1.0, np.float32)
        for q, (dx, dy, dz) in enumerate(M.CORNERS):
            g[1 + dx, 1 + dy, 1 + dz] = 1.0 if cs >> q & 1 else -1.0
        v, f, _ = M.marching_cubes(g, (0, 0, 0), (1, 1, 1), 0.0)
        assert M.is_closed(f) and M.oriented_consistently(f), cs
        assert M.signed_volume(v, f) > 0, cs


@pytest.mark.parametrize("seed", range(4))
def test_random_fields_close(seed):
    """Sums of random Gaussians that stay below the level on the border: closed, consistently wound, positive volume."""
    rs = np.random.RandomState(seed)
    cs, ws = rs.uniform(-0.5, 0.5, (6, 3)), rs.uniform(0.1, 0.3, 6)

    def fn(x, y, z):
        return sum(np.exp(-((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) / (2 * w * w)) for c, w in zip(cs, ws))

    g = M.grid_values(fn, (-1, -1, -1), (2 / 23,) * 3, (24, 24, 24))
    v, f, _ = M.marching_cubes(g, (-1, -1, -1), (2 / 23,) * 3, 0.4)
    assert len(f) and M.is_closed(f) and M.oriented_consistently(f) and M.signed_volume(v, f) > 0


def test_sphere_and_torus_topology():
    h = (0.05, 0.05, 0.05)
    for fn, dims, chi, vol in ((M.sphere((0.1, -0.05, 0.02), 0.7), (33, 33, 33), 2, 4 / 3 * np.pi * 0.7 ** 3),
                               (M.torus(0.6, 0.25), (40, 40, 20), 0, 2 * np.pi ** 2 * 0.6 * 0.25 ** 2)):
        org = tuple(-(d - 1) * s / 2 for d, s in zip(dims, h))
        v, f, _ = M.marching_cubes(M.grid_values(fn, org, h, dims), org, h, 0.0)
        assert M.is_closed(f) and M.euler_characteristic(v, f) == chi
        assert abs(M.signed_volume(v, f) - vol) <= h[0] ** 2 * M.area(v, f)
