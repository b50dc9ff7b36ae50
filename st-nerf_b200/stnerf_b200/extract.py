"""A layer's geometry at any frame: its density field on a grid and a triangle mesh of a level set.

The field is the one the renderer draws (stnerf_layer_field / stnerf_layer_grid, include/stnerf.h): the pass' inverse scale /
shift edit, for a performer the MotionNet flow at the frame, then the layer's SpaceNet with the frame as its time input, in the
model's render precision.  `utils.vis_density` is not that field (no MotionNet, no frame, no edit); use `layer_density`.

    d = layer_density(model, layer=1, frame=37)             # sigma (R0,R1,R2) on the device, grid origin and step
    mesh = extract_mesh(model, layer=1, frame=37, level=10.0)
    write_ply("performer1_f37.ply", mesh)

Works on `LayeredRFRender` and `TrainableLayeredRFRender`; the trainable model's current parameters are used (its
`_ensure_native` re-uploads them when they changed).
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import rotation as ROT
from .native import marching_cubes


class LayerDensity(NamedTuple):
    sigma: torch.Tensor          # (R0, R1, R2) raw sigma, fp32 on the device; [i,j,k] at origin + (i,j,k)*step
    origin: Tuple[float, float, float]
    step: Tuple[float, float, float]


class Mesh(NamedTuple):
    verts: torch.Tensor          # (V, 3) fp32
    faces: torch.Tensor          # (F, 3) int64, wound so that normals point toward lower density
    colors: Optional[torch.Tensor]   # (V, 3) in [0, 1], or None


def _scene(model, frame: float):
    """The scene the render uses when every layer shows frame `frame` (retiming layout: boxes lerped to the frame,
    layered_rfrender.py:195-204, then the scale / shift edits :207-242).  Host only."""
    retiming = model.retiming
    model.retiming = True
    try:
        return model._resolve_scene(torch.full((model.layer_num + 1,), float(frame), dtype=torch.float32), 0.0, 0.0)
    finally:
        model.retiming = retiming


def _scene_at(model, frame: float):
    """The model's context (current weights) with the scene of `frame` set on it."""
    nat = model._ensure_native(torch.device("cuda", torch.cuda.current_device()))
    scene = _scene(model, frame)
    nat.set_scene(scene)
    model._upload_rotation(nat)
    return nat, scene


def layer_box(model, layer: int, frame: float):
    """(lo, hi) corners of the box the render clips `layer` against at `frame` (layer 0: the background box), after the scale /
    shift edits; a rotated layer clips against this box turned by its rotation (see `layer_density`)."""
    scene = _scene(model, frame)
    return tuple(float(v) for v in scene.bmin[layer]), tuple(float(v) for v in scene.bmax[layer])


def _grid(lo, hi, resolution):
    dims = (int(resolution),) * 3 if np.isscalar(resolution) else tuple(int(r) for r in resolution)
    if len(dims) != 3 or min(dims) < 2:
        raise ValueError("resolution must be an int or a 3-tuple, each at least 2, got %r" % (resolution,))
    lo32 = torch.tensor(lo, dtype=torch.float32)
    step = (torch.tensor(hi, dtype=torch.float32) - lo32) / torch.tensor([d - 1 for d in dims], dtype=torch.float32)
    return tuple(float(v) for v in lo32), tuple(float(v) for v in step), dims


def _bbox(bbox):
    b = torch.as_tensor(bbox, dtype=torch.float32).reshape(-1, 3)
    return tuple(float(v) for v in b.min(0).values), tuple(float(v) for v in b.max(0).values)


def layer_density(model, layer: int, frame: float, resolution=128, bbox=None, fine: bool = True) -> LayerDensity:
    """Raw sigma of `layer` at `frame` on a resolution^3 (or R0 x R1 x R2) grid spanning `bbox` -- any corner set, e.g. (2,3)
    or (8,3) -- or, by default, the layer's box at that frame as the render clips it (for a rotated layer the world bounds of
    the turned box, rounded outward).  fine=False: the coarse networks."""
    if not 0 <= int(layer) <= model.layer_num:
        raise ValueError("layer %d out of range [0, %d]" % (layer, model.layer_num))
    nat, scene = _scene_at(model, frame)
    lo, hi = _bbox(bbox) if bbox is not None else (tuple(scene.bmin[layer]), tuple(scene.bmax[layer]))
    entry = model._rotation_entries()[int(layer)]
    if bbox is None and entry is not None:
        lo, hi = ROT.oriented_box_aabb(lo, hi, entry[0], ROT.centre_of(entry, lo, hi))
    origin, step, dims = _grid(lo, hi, resolution)
    sigma = nat.layer_grid(int(layer), bool(fine), float(frame), origin, step, dims)
    return LayerDensity(sigma, origin, step)


def _vertex_view_dirs(verts: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """Negated area-weighted vertex normals, unit length (zero where the normals cancel).  Summed in float64 on the host in
    face order, so the result does not depend on the order atomics land in."""
    v = verts.detach().cpu().double().numpy()
    f = faces.detach().cpu().numpy().astype(np.int64)
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])         # twice the area times the unit normal
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    norm = np.linalg.norm(n, axis=1, keepdims=True)
    d = np.where(norm > 0, -n / np.where(norm > 0, norm, 1.0), 0.0)
    return torch.from_numpy(d.astype(np.float32)).to(verts.device)


def extract_mesh(model, layer: int, frame: float, level: float, resolution=256, bbox=None, fine: bool = True,
                 colors: bool = True) -> Mesh:
    """Marching cubes of {sigma > level} of `layer` at `frame` on the grid of `layer_density`.  `level` is a raw-sigma
    threshold and has no default: it depends on the scene.  Colours are sigmoid(rgb) of the same field at each vertex, seen
    head-on from outside (view direction = the negated area-weighted vertex normal) at time `frame`."""
    d = layer_density(model, layer, frame, resolution, bbox, fine)
    verts, faces = marching_cubes(d.sigma, d.origin, d.step, float(level))
    col = None
    if colors:
        col = torch.zeros_like(verts)
        if verts.shape[0] > 0:
            nat = model._native
            rgb, _ = nat.layer_field(int(layer), bool(fine), float(frame), verts, _vertex_view_dirs(verts, faces))
            col = torch.sigmoid(rgb)
    return Mesh(verts, faces.to(torch.int64), col)


def write_ply(path: str, mesh: Mesh) -> None:
    """Binary little-endian PLY: vertices (x, y, z float, plus red/green/blue uchar with colours) and triangle faces."""
    v = mesh.verts.detach().cpu().numpy().astype("<f4")
    f = mesh.faces.detach().cpu().numpy()
    if f.size and (f.min() < 0 or f.max() >= len(v) or f.max() > np.iinfo(np.int32).max):
        raise ValueError("face indices out of range")
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    header = ["ply", "format binary_little_endian 1.0", "element vertex %d" % len(v)] + \
             ["property float %s" % a for a in "xyz"]
    if mesh.colors is not None:
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        header += ["property uchar %s" % c for c in ("red", "green", "blue")]
    header += ["element face %d" % len(f), "property list uchar int vertex_indices", "end_header"]
    vrec = np.empty(len(v), dtype=np.dtype(props))
    for k, a in enumerate("xyz"):
        vrec[a] = v[:, k]
    if mesh.colors is not None:
        c = np.rint(np.clip(mesh.colors.detach().cpu().numpy().astype(np.float64), 0.0, 1.0) * 255.0).astype(np.uint8)
        for k, a in enumerate(("red", "green", "blue")):
            vrec[a] = c[:, k]
    frec = np.empty(len(f), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    frec["n"] = 3
    frec["i"] = f.astype("<i4")
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())
