#!/usr/bin/env python
"""Reference outputs of the ray/box clipping and stratified sampling on adversarial rays (tests/golden/geometry.npz).

Run where the reference tree is available:

    python tests/golden/make_golden_geometry.py

It runs the UNMODIFIED reference's `intersection` and `RaySamplePoint.forward` (layers/RaySamplePoint.py:8-105, jitter
injected through oracle.reference_shim) on the rays of `geometry_inputs()` at 6, 7 and 9 columns.  The inputs are a pure
function of this file, so tests rebuild them here and only the outputs are stored.  The archive is written with fixed
member timestamps, so a rerun reproduces it byte for byte.

Every ray is built from dyadic values (origin = target - s * d with dyadic s and d), so fp32 lands exactly on the faces,
edges and corners it aims at.  Families (`FAMILIES`, one id per ray):
  face / edge / corner  through a face interior, an edge, a corner of a box, from in front of and behind the origin;
  diag                  corner to opposite corner: all six faces valid;  corner_edge: a corner and an edge, five valid;
  inside / on_face      origin inside the box / on a face (t = +-0);  behind: the box behind the origin, nearer and farther
                        than t = -1000;
  den0                  a direction component of +0, -0, -2.220446e-16f (d + eps == 0: t = +-inf or NaN) or denormal;
  graze                 parallel to a face, on its plane and one ulp inside and outside;
  width                 chords that put |bin width| one ulp below, at and above 1e-5f for n1 = 3 and 64;
Boxes include one at 1e4 units and one of zero thickness.  Rays with five or six valid faces all below t = -1000 are the
rows where the -1e3 sentinels of tlist (one per ray column beyond the sixth) decide the result.
"""
from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FAMILIES = ("face", "edge", "corner", "diag", "corner_edge", "inside", "on_face", "behind", "den0", "graze", "width")
COLUMNS = (6, 7, 9)
GOLDEN_N1 = (3, 64)
T_1E5 = np.float32(1e-5)                     # `torch.abs(bin_width) > 1e-5` compares in fp32 (:105)
EPS32 = np.float32(np.finfo(float).eps)      # d + eps of :17-22, in fp32

_BOXES = [((-1.0, -0.25, 0.0), (0.5, 1.5, 2.0)),
          ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)),
          ((1e4, -1e4, 1e4), (1e4 + 2.0, -1e4 + 4.0, 1e4 + 1.0)),
          ((-1.0, -1.0, 0.5), (1.0, 1.0, 0.5))]          # zero thickness in z
_DIRS = [(1.0, 0.5, 0.25), (-0.5, 1.0, 0.75), (0.25, -0.75, 1.0), (-1.0, -0.5, -0.25), (0.75, 0.25, -1.0),
         (0.5, 0.5, 0.5), (-0.125, 1.0, -0.5)]


def _f32_exact(v):
    a = np.asarray(v, dtype=np.float64)
    b = a.astype(np.float32)
    assert np.array_equal(b.astype(np.float64), a, equal_nan=True), a
    return b


def _width_box(n1, target, shape):
    """A box whose x chord gives |(t_far - start) / n1| == target in fp32 for a ray along x from the origin."""
    d0 = np.float32(target * n1)
    for k in range(-16, 17):
        D = np.float32(d0 + np.float32(k) * np.spacing(d0))
        if np.float32(D / np.float32(n1)) == target:
            break
    else:
        raise AssertionError("no chord for width %r at n1=%d" % (target, n1))
    D = float(D)
    if shape == 0:                      # d = +x, box [0, D]: t_near = +0, t_far = D
        return (0.0, -1.0, -1.0), (D, 1.0, 1.0), (1.0, 0.0, 0.0)
    if shape == 1:                      # d = -x, box [-D, 0]: t_near = -0.0
        return (-D, -1.0, -1.0), (0.0, 1.0, 1.0), (-1.0, 0.0, 0.0)
    return (-2.0 * D, -1.0, -1.0), (-D, 1.0, 1.0), (1.0, 0.0, 0.0)     # behind: bkgd width -D/n1, performer D/n1


def geometry_inputs() -> dict:
    """rays (N,6) fp32, box_id (N,), boxes (B,2,3) fp32, family (N,) index into FAMILIES."""
    boxes = [b for b in _BOXES]
    rows, fam, bid = [], [], []

    def add(o, d, b, f):
        rows.append(np.concatenate([_f32_exact(o), _f32_exact(d)]))
        fam.append(FAMILIES.index(f))
        bid.append(b)

    def aim(c, d, s, b, f):
        c, d = np.asarray(c, np.float64), np.asarray(d, np.float64)
        add(c - s * d, d, b, f)

    for b, (lo, hi) in enumerate(_BOXES):
        lo, hi = np.asarray(lo), np.asarray(hi)
        mid = (lo + hi) / 2
        quarter = lo + (hi - lo) / 4
        for axis in range(3):
            for face in (lo[axis], hi[axis]):
                c = quarter.copy(); c[axis] = face
                for j, d in enumerate(_DIRS):
                    aim(c, d, (0.5, 2.0, -1.5)[j % 3], b, "face")
                # an edge of this face, and the corners at its ends
                a1 = (axis + 1) % 3
                for e in (lo[a1], hi[a1]):
                    ce = c.copy(); ce[a1] = e
                    for j, d in enumerate(_DIRS[:4]):
                        aim(ce, d, (1.0, -0.5)[j % 2], b, "edge")
        for cx in (lo[0], hi[0]):
            for cy in (lo[1], hi[1]):
                for cz in (lo[2], hi[2]):
                    for j, d in enumerate(_DIRS[:5]):
                        aim((cx, cy, cz), d, (0.75, -0.25)[j % 2], b, "corner")
        if b == 3:
            continue
        ext = hi - lo
        for sx in (1, -1):
            for sy in (1, -1):
                for sz in (1, -1):
                    sg = np.array([sx, sy, sz], np.float64)
                    start = np.where(sg > 0, lo, hi)
                    for s in (0.5, -1.0, -2048.0):                        # -2048: both corners below t = -1000
                        aim(start, sg * ext, s, b, "diag")
                    for half in range(3):                               # ends on the edge opposite `start` at mid-height
                        d = sg * ext
                        d[half] /= 2
                        for s in (0.5, -4.0, -2048.0):
                            aim(start, d, s, b, "corner_edge")
        for j, d in enumerate(_DIRS):
            add(quarter + (hi - lo) * (j % 3) / 4, d, b, "inside")
        for axis in range(3):
            for face, inward in ((lo[axis], 1.0), (hi[axis], -1.0)):
                o = quarter.copy(); o[axis] = face
                for dv in (inward, -inward, 0.0):
                    d = np.array([0.25, 0.5, 0.75]); d[axis] = dv
                    add(o, d, b, "on_face")
                c = mid.copy(); c[axis] = face
                for s in (-4.0, -1500.0):
                    d = np.array([0.5, 0.25, 0.125]); d[axis] = inward
                    aim(c, d, s, b, "behind")
                # parallel to the face plane: on it, one ulp inside, one ulp outside
                for off in (0.0, inward, -inward):
                    o = quarter.copy()
                    o[axis] = face if off == 0 else float(np.nextafter(np.float32(face), np.float32(face + off)))
                    for a1 in range(3):
                        if a1 == axis:
                            continue
                        d = np.zeros(3); d[a1] = 1.0
                        o2 = o.copy(); o2[a1] = lo[a1] - 1.0
                        add(o2, d, b, "graze")
        # direction components whose den = d + eps is 0, denormal or eps itself
        denorm = float(np.float32(1e-40))
        for axis in range(3):
            for dv in (0.0, -0.0, -float(EPS32), denorm, -denorm):
                for on_plane in (False, True):
                    o = quarter.copy()
                    if on_plane:
                        o[axis] = lo[axis]
                    d = np.array([0.5, 0.75, 1.0]); d[axis] = dv
                    o2 = o - 2.0 * d
                    o2[axis] = o[axis]
                    add(o2, d, b, "den0")
    # the example of a ray through a corner and an edge, far behind the origin: o = (2000, 2000, 1000), d = normalize(1, 1, .5)
    d = torch.tensor([1.0, 1.0, 0.5]); d = (d / d.norm()).numpy()
    rows.append(np.concatenate([np.float32([2000.0, 2000.0, 1000.0]), d.astype(np.float32)]))
    fam.append(FAMILIES.index("corner_edge")); bid.append(1)
    for n1 in GOLDEN_N1:
        for target in (np.nextafter(T_1E5, np.float32(0)), T_1E5, np.nextafter(T_1E5, np.float32(1))):
            for shape in range(3):
                lo, hi, d = _width_box(n1, target, shape)
                boxes.append((lo, hi))
                add((0.0, 0.0, 0.0), d, len(boxes) - 1, "width")
    rays = np.stack(rows).astype(np.float32)
    return {"rays": rays, "box_id": np.asarray(bid, np.int64), "family": np.asarray(fam, np.int64),
            "boxes": np.asarray([[lo, hi] for lo, hi in boxes], dtype=np.float32)}


def jitter_for(n: int, n1: int, seed: int) -> np.ndarray:
    """(n, n1) uniforms in [0, 1) with 24 bits; row r % 4 == 0 is all 0, row r % 4 == 1 all nextafter(1, 0)."""
    rs = np.random.RandomState(seed + n1)
    j = (rs.randint(0, 1 << 24, size=(n, n1)).astype(np.float64) / (1 << 24)).astype(np.float32)
    j[0::4] = 0.0
    j[1::4] = np.nextafter(np.float32(1), np.float32(0))
    return j


def widen(rays: np.ndarray, cols: int) -> np.ndarray:
    """The rays with frame-id columns 6.. appended (value 1.0)."""
    return np.concatenate([rays, np.ones((rays.shape[0], cols - 6), np.float32)], 1)


def corners(bmin, bmax) -> torch.Tensor:
    """(N,8,3) corners in the order of data/datasets/frame_dataset.py:187-188 from per-ray min / max (N,3)."""
    lo, hi = torch.as_tensor(bmin), torch.as_tensor(bmax)
    pick = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
    return torch.stack([torch.stack([(hi if p[a] else lo)[:, a] for a in range(3)], -1) for p in pick], 1)


def save_npz(path: str, arrays: dict):
    """np.savez_compressed with fixed member timestamps: the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    from oracle import reference_shim as R
    R.modules()
    from layers.RaySamplePoint import intersection, RaySamplePoint

    g = geometry_inputs()
    n = g["rays"].shape[0]
    box = torch.from_numpy(g["boxes"][g["box_id"]])
    bbox = corners(box[:, 0], box[:, 1])
    out = {}
    for cols in COLUMNS:
        rays = torch.from_numpy(widen(g["rays"], cols))
        out["isect.%d" % cols] = intersection(rays, bbox).numpy()
        for n1 in GOLDEN_N1:
            jit = [torch.from_numpy(jitter_for(n, n1, 10 * layer)) for layer in (0, 1)]
            with R.injected_uniforms(jit):
                ts, pts, masks = RaySamplePoint(n1).forward(rays, torch.stack([bbox, bbox], 1))
            for layer in (0, 1):
                out["mask.%d.%d.%d" % (cols, layer, n1)] = masks[layer].numpy().astype(np.uint8)
                if n1 == 3:
                    out["t.%d.%d.%d" % (cols, layer, n1)] = ts[layer][..., 0].numpy()
                    if cols == 7:
                        out["xyz.%d.%d.%d" % (cols, layer, n1)] = pts[layer].numpy()
    path = os.path.join(HERE, "geometry.npz")
    save_npz(path, out)
    fam = np.bincount(g["family"], minlength=len(FAMILIES))
    print("geometry.npz: %d rays, %d boxes, %d bytes; %s" % (n, len(g["boxes"]), os.path.getsize(path),
                                                             dict(zip(FAMILIES, fam.tolist()))))


if __name__ == "__main__":
    main()
