"""Float64 numpy restatement of the marching cubes of csrc/extract.cu (stnerf_mc_count / stnerf_mc_fill), and mesh checks.

The triangle table is read from csrc/mc_table.cuh; everything else is written out here: inside = v > level (NaN outside),
vertices on the +x/+y/+z edges of each grid point in grid-point-major order, triangles in cell-major order."""
from __future__ import annotations

import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = os.path.join(ROOT, "st-nerf_b200", "csrc", "mc_table.cuh")
# Bourke's cube: corner offsets, and edge e = (corner offset of its lower end, axis)
CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [((0, 0, 0), 0), ((1, 0, 0), 1), ((0, 1, 0), 0), ((0, 0, 0), 1), ((0, 0, 1), 0), ((1, 0, 1), 1),
         ((0, 1, 1), 0), ((0, 0, 1), 1), ((0, 0, 0), 2), ((1, 0, 0), 2), ((1, 1, 0), 2), ((0, 1, 0), 2)]


def load_table():
    src = open(TABLE).read()
    ntri = np.array([int(x) for x in re.search(r"c_mc_ntri\[256\] = \{([^}]*)\}", src).group(1).replace("\n", " ").split(",")
                     if x.strip()], dtype=np.int64)
    body = src[src.index("c_mc_tri[256]"):]
    rows = re.findall(r"\{([-0-9, ]+)\},", body)
    tri = np.array([[int(x) for x in r.split(",")] for r in rows], dtype=np.int64)
    assert ntri.shape == (256,) and tri.shape[0] == 256
    return ntri, tri


def marching_cubes(sigma, origin, step, level):
    """-> verts (V,3) float64, faces (F,3) int64, owner (V,2) = (flat grid point, axis) of every vertex."""
    s = np.asarray(sigma, dtype=np.float64)
    n0, n1, n2 = s.shape
    ntri, tri = load_table()
    inside = s > level
    mask = np.zeros(s.shape, dtype=np.int64)
    mask[:-1] |= (inside[:-1] != inside[1:]).astype(np.int64)
    mask[:, :-1] |= (inside[:, :-1] != inside[:, 1:]).astype(np.int64) << 1
    mask[:, :, :-1] |= (inside[:, :, :-1] != inside[:, :, 1:]).astype(np.int64) << 2
    flat = mask.reshape(-1)
    count = (flat & 1) + ((flat >> 1) & 1) + ((flat >> 2) & 1)
    voff = np.concatenate([[0], np.cumsum(count)[:-1]])
    stride = np.array([n1 * n2, n2, 1])
    o, h = np.asarray(origin, np.float64), np.asarray(step, np.float64)
    verts, owner = [], []
    pts = np.nonzero(flat)[0]
    idx = np.stack([pts // stride[0], (pts // stride[1]) % n1, pts % n2], 1)
    for p, ijk in zip(pts, idx):
        for a in range(3):
            if flat[p] >> a & 1:
                v0, v1 = s.reshape(-1)[p], s.reshape(-1)[p + stride[a]]
                t = (level - v0) / (v1 - v0)
                if not (0.0 <= t <= 1.0):
                    t = 1.0 if v0 > level else 0.0
                x = o + ijk * h
                x[a] += t * h[a]
                verts.append(x)
                owner.append((p, a))
    cases = np.zeros((n0 - 1, n1 - 1, n2 - 1), dtype=np.int64)
    for q, (dx, dy, dz) in enumerate(CORNERS):
        cases |= inside[dx:n0 - 1 + dx, dy:n1 - 1 + dy, dz:n2 - 1 + dz].astype(np.int64) << q
    cflat = cases.reshape(-1)
    faces = []
    for c in np.nonzero(ntri[cflat])[0]:
        i, j, k = c // ((n1 - 1) * (n2 - 1)), (c // (n2 - 1)) % (n1 - 1), c % (n2 - 1)
        cs = cflat[c]
        for t in range(ntri[cs]):
            f = []
            for q in range(3):
                (dx, dy, dz), a = EDGES[tri[cs, 3 * t + q]]
                p = (i + dx) * stride[0] + (j + dy) * stride[1] + (k + dz)
                f.append(voff[p] + sum((flat[p] >> b) & 1 for b in range(a)))
            faces.append(f)
    return (np.array(verts, np.float64).reshape(-1, 3), np.array(faces, np.int64).reshape(-1, 3),
            np.array(owner, np.int64).reshape(-1, 2))


def edge_face_counts(faces):
    """{(a, b) with a < b: number of faces with that edge}."""
    f = np.asarray(faces, np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
    e.sort(1)
    keys, counts = np.unique(e, axis=0, return_counts=True)
    return keys, counts


def is_closed(faces):
    _, counts = edge_face_counts(faces)
    return bool(len(counts)) and bool((counts == 2).all())


def oriented_consistently(faces):
    """Every edge is used once in each direction (a closed, consistently wound surface)."""
    f = np.asarray(faces, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
    fw = {tuple(x) for x in d}
    return len(fw) == len(d) and all((b, a) in fw for a, b in fw)


def euler_characteristic(verts, faces):
    keys, _ = edge_face_counts(faces)
    used = np.unique(np.asarray(faces).reshape(-1))
    return len(used) - len(keys) + len(faces)


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    return float(np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6.0)


def area(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    return float(np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1).sum() / 2.0)


def grid_values(fn, origin, step, dims):
    """fn(x, y, z) on the grid points (float64 coordinates) -> float32 (D0, D1, D2)."""
    ax = [origin[a] + np.arange(dims[a], dtype=np.float64) * step[a] for a in range(3)]
    x, y, z = np.meshgrid(*ax, indexing="ij")
    return fn(x, y, z).astype(np.float32)


def sphere(c, r):
    return lambda x, y, z: r - np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2)


def torus(big, small):
    return lambda x, y, z: small - np.sqrt((np.sqrt(x ** 2 + y ** 2) - big) ** 2 + z ** 2)
