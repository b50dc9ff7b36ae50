"""Writes st-nerf_b200/csrc/mc_table.cuh: the 256-case marching-cubes triangle table of csrc/extract.cu.

Corner and edge numbering are Bourke's (corner k at (k&1 ^ k>>1&1, k>>1&1, k>>2) ... see CORNERS / EDGES below).  Each case is
built from its six faces, so a face shared by two cells is cut the same way from both sides and the surface is closed:
  - a face with one, two adjacent or three inside corners gets one segment between its two crossed edges;
  - an ambiguous face (two diagonal inside corners) gets two segments, each cutting off one INSIDE corner (the inside corners
    are kept apart, the outside region is connected across the face);
  - every segment is directed so that, seen from outside the cube, the inside region lies on its right; the segments of a case
    then join into closed loops (each crossed edge lies on exactly two faces), and each loop is fanned into triangles whose
    right-hand normal points from inside to outside (toward lower density);
  - a loop is fanned from the vertex whose diagonals do not join two vertices of one cube face, so no triangle edge inside a
    cell coincides with an edge the neighbouring cell draws on their common face.
Run `python scripts/gen_mc_table.py` after changing this file; the output is committed.
"""
import os

import numpy as np

CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
# face: corner cycle, outward normal
FACES = [((0, 1, 2, 3), (0, 0, -1)), ((4, 5, 6, 7), (0, 0, 1)), ((0, 1, 5, 4), (0, -1, 0)), ((3, 2, 6, 7), (0, 1, 0)),
         ((0, 3, 7, 4), (-1, 0, 0)), ((1, 2, 6, 5), (1, 0, 0))]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "st-nerf_b200", "csrc", "mc_table.cuh")


def edge_of(a, b):
    for e, (p, q) in enumerate(EDGES):
        if {p, q} == {a, b}:
            return e
    raise KeyError((a, b))


def mid(e):
    p, q = EDGES[e]
    return (np.array(CORNERS[p], float) + np.array(CORNERS[q], float)) / 2


FACE_EDGES = [set(edge_of(c[i], c[(i + 1) % 4]) for i in range(4)) for c, _ in FACES]


def face_segments(case, corners, normal):
    """Directed segments (edge_from, edge_to) of one face."""
    inside = [(case >> c) & 1 for c in corners]
    n = np.array(normal, float)
    segs = []   # (edge a, edge b, g = direction from inside toward outside in the face)
    ins = [c for c, s in zip(corners, inside) if s]
    outs = [c for c, s in zip(corners, inside) if not s]
    if len(ins) in (0, 4):
        return []
    if len(ins) == 2 and inside[0] == inside[2]:          # ambiguous: cut off each inside corner on its own
        for k in range(4):
            if inside[k]:
                c, prev, nxt = corners[k], corners[(k - 1) % 4], corners[(k + 1) % 4]
                a, b = edge_of(prev, c), edge_of(c, nxt)
                g = (mid(a) + mid(b)) / 2 - np.array(CORNERS[c], float)
                segs.append((a, b, g))
    else:
        crossed = [edge_of(corners[k], corners[(k + 1) % 4]) for k in range(4) if inside[k] != inside[(k + 1) % 4]]
        assert len(crossed) == 2
        g = np.mean([CORNERS[c] for c in outs], 0) - np.mean([CORNERS[c] for c in ins], 0)
        segs.append((crossed[0], crossed[1], g))
    out = []
    for a, b, g in segs:
        t = np.cross(g, n)
        d = float(np.dot(mid(b) - mid(a), t))
        assert abs(d) > 1e-9
        out.append((a, b) if d > 0 else (b, a))
    return out


def triangulate(case):
    nxt = {}
    for corners, normal in FACES:
        for a, b in face_segments(case, corners, normal):
            assert a not in nxt, (case, a)
            nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()), case
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            seen.add(loop[-1])
        loops.append(loop)
    tris = []
    for loop in loops:
        k = len(loop)
        best = None
        for s in range(k):
            rot = loop[s:] + loop[:s]
            diags = [(rot[0], rot[j]) for j in range(2, k - 1)]
            if all(not any(a in fe and b in fe for fe in FACE_EDGES) for a, b in diags):
                best = rot
                break
        assert best is not None, (case, loop)
        tris += [(best[0], best[j], best[j + 1]) for j in range(1, k - 1)]
    return tris


def check_orientation(case, tris):
    """Every triangle's normal points down the gradient of the trilinear interpolant of +1 (inside) / -1 (outside)."""
    v = np.array([1.0 if (case >> c) & 1 else -1.0 for c in range(8)])

    def grad(p):
        x, y, z = p
        g = np.zeros(3)
        for c, (cx, cy, cz) in enumerate(CORNERS):
            wx, wy, wz = (x if cx else 1 - x), (y if cy else 1 - y), (z if cz else 1 - z)
            dx, dy, dz = (1 if cx else -1), (1 if cy else -1), (1 if cz else -1)
            g += v[c] * np.array([dx * wy * wz, wx * dy * wz, wx * wy * dz])
        return g

    for t in tris:
        p = [mid(e) for e in t]
        nrm = np.cross(p[1] - p[0], p[2] - p[0])
        assert np.dot(nrm, -grad(np.mean(p, 0))) > 0, (case, t)


def main():
    table = []
    for case in range(256):
        tris = triangulate(case)
        check_orientation(case, tris)
        table.append(tris)
    max_t = max(len(t) for t in table)
    lines = ["// Generated by scripts/gen_mc_table.py -- do not edit.  Marching-cubes triangle table (see that script): per case the",
             "// triangle count, then up to %d triangles as triples of cube edges (Bourke's numbering), unused entries -1." % max_t,
             "#pragma once", "#include <stdint.h>", "",
             "namespace stnerf {", "constexpr int MC_MAX_TRIS = %d;" % max_t,
             "__constant__ uint8_t c_mc_ntri[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in table[r:r + 32]) + ",")
    lines.append("};")
    lines.append("__constant__ int8_t c_mc_tri[256][%d] = {" % (3 * max_t))
    for case, tris in enumerate(table):
        flat = [e for t in tris for e in t] + [-1] * (3 * (max_t - len(tris)))
        lines.append("    {%s},  // %d" % (", ".join(str(e) for e in flat), case))
    lines.append("};")
    lines.append("}  // namespace stnerf")
    with open(OUT, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("wrote %s (max %d triangles per case)" % (OUT, max_t))


if __name__ == "__main__":
    main()
