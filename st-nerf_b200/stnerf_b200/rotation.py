"""The per-layer rotation edit: parsing `model.rotation` and the host side of stnerf_set_rotation (include/stnerf.h).

Layer i (0 = background, indexed like `shift` / `scale`) may carry a rotation R_i about a centre c_i, applied on top of the
scale / shift edit:  world = c + R (edited(p) - c).  An entry of `model.rotation` is
  - None: no rotation;
  - a 3x3 matrix (orthonormal, det +1, to 1e-5);
  - a rotation vector, axis * angle in radians (Rodrigues' formula in float64, then rounded to float32);
  - (R, centre) with R either of the above and centre a 3-vector; without a centre the layer turns about the centre of its
    edited box in the call's scene, (bmin + bmax) * 0.5 in float32.
An entry exactly equal to the identity counts as None: (o - c) + c is not o in float32, and no rotation must stay bit-identical
to no rotation.  Host only.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L

Entry = Optional[Tuple[np.ndarray, Optional[np.ndarray]]]     # (R float32 (3,3), centre float32 (3,) or None)


def rodrigues(v) -> np.ndarray:
    """Rotation matrix (float64) of the rotation vector v = axis * angle (radians)."""
    v = np.asarray(v, dtype=np.float64).reshape(3)
    theta = float(np.linalg.norm(v))
    if theta == 0.0:
        return np.eye(3)
    k = v / theta
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    return np.eye(3) + np.sin(theta) * K + (1.0 - np.cos(theta)) * (K @ K)


def _matrix(x) -> np.ndarray:
    a = np.asarray(x, dtype=np.float64)
    if a.shape == (3,):
        if not np.isfinite(a).all():
            raise ValueError("rotation vector must be finite, got %r" % (a.tolist(),))
        return rodrigues(a).astype(np.float32)
    if a.shape != (3, 3):
        raise ValueError("a rotation is a 3x3 matrix or a rotation vector (3,), got shape %s" % (a.shape,))
    if not np.isfinite(a).all():
        raise ValueError("rotation matrix must be finite")
    if np.abs(a.T @ a - np.eye(3)).max() > 1e-5 or abs(np.linalg.det(a) - 1.0) > 1e-5:
        raise ValueError("rotation matrix must be orthonormal with determinant +1 (to 1e-5)")
    return a.astype(np.float32)


def parse_entry(e) -> Entry:
    """One entry of `model.rotation` -> None or (R float32 (3,3), centre float32 (3,) or None).  Raises ValueError."""
    if e is None:
        return None
    centre = None
    if isinstance(e, (tuple, list)) and len(e) == 2:
        e, centre = e
        centre = np.asarray(centre, dtype=np.float64)
        if centre.shape != (3,) or not np.isfinite(centre).all():
            raise ValueError("rotation centre must be 3 finite numbers")
        centre = centre.astype(np.float32)
    R = _matrix(e)
    if np.array_equal(R, np.eye(3, dtype=np.float32)):
        return None
    return R, centre


def resolve(rotation, l: int) -> List[Entry]:
    """Every layer's parsed entry.  A list shorter than the layer count (background included) raises IndexError, like shift."""
    if rotation is None:
        return [None] * l
    if len(rotation) < l:
        raise IndexError("rotation must have one entry per layer incl. background")
    return [parse_entry(rotation[i]) for i in range(l)]


def default_centre(lo, hi) -> np.ndarray:
    """The centre a rotation without an explicit one turns about: (bmin + bmax) * 0.5 of the edited box, float32."""
    return (np.asarray(lo, dtype=np.float32) + np.asarray(hi, dtype=np.float32)) * np.float32(0.5)


def centre_of(entry: Entry, lo, hi) -> np.ndarray:
    R, c = entry
    return c if c is not None else default_centre(lo, hi)


def oriented_box_aabb(lo, hi, R, c) -> Tuple[Tuple[float, ...], Tuple[float, ...]]:
    """World axis-aligned bounds of the box [lo, hi] turned by R about c: the eight corners c + R (corner - c) in float64,
    rounded outward to float32."""
    lo64, hi64 = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    corners = np.array([[(hi64 if (k >> a) & 1 else lo64)[a] for a in range(3)] for k in range(8)])
    c64 = np.asarray(c, dtype=np.float64)
    w = (np.asarray(R, dtype=np.float64) @ (corners - c64).T).T + c64
    mn, mx = w.min(0), w.max(0)
    mn32, mx32 = mn.astype(np.float32), mx.astype(np.float32)
    mn32 = np.where(mn32.astype(np.float64) > mn, np.nextafter(mn32, np.float32(-np.inf)), mn32)
    mx32 = np.where(mx32.astype(np.float64) < mx, np.nextafter(mx32, np.float32(np.inf)), mx32)
    return tuple(float(v) for v in mn32), tuple(float(v) for v in mx32)


def abi_arrays(entries: Sequence[Entry]):
    """(modes int32 (l,), R float32 (l,9), centres float32 (l,3)) for stnerf_set_rotation; entries without a centre use
    STNERF_ROT_BOX, so the library takes each call's (each view's) box centre."""
    l = len(entries)
    modes = np.zeros(l, dtype=np.int32)
    R = np.zeros((l, 9), dtype=np.float32)
    cen = np.zeros((l, 3), dtype=np.float32)
    for i, e in enumerate(entries):
        if e is None:
            continue
        R[i] = e[0].reshape(9)
        if e[1] is None:
            modes[i] = L.ROT_BOX
        else:
            modes[i] = L.ROT_CENTRE
            cen[i] = e[1]
    return modes, R, cen
