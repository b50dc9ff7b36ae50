"""Thin object wrapper over the C ABI: owns a context handle, loads weights, sets the scene, renders.

torch is used only for device memory and the current stream; every arithmetic step happens in libstnerf_b200.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L

SPACENET_KEYS = ["stage1.0", "stage1.2", "stage1.4", "stage1.6", "stage2.0", "stage2.2", "stage2.4",
                 "density_net.0", "rgb_net.1", "rgb_net.3"]
MOTIONNET_KEYS = ["motion_net.%d" % i for i in (0, 2, 4, 6, 8, 10)]


def _blob(sd: Dict[str, torch.Tensor], prefix: str, names: Sequence[str]) -> torch.Tensor:
    parts = []
    for n in names:
        parts.append(sd[prefix + n + ".weight"].detach().to("cpu", torch.float32).reshape(-1))
        parts.append(sd[prefix + n + ".bias"].detach().to("cpu", torch.float32).reshape(-1))
    return torch.cat(parts).contiguous()


def _dev_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise L.StnerfError("%s must be a CUDA tensor (no CPU fallback)" % name)
    if t.dtype != torch.float32:
        raise L.StnerfError("%s must be float32, got %s" % (name, t.dtype))
    return t.detach().contiguous()


class NativeRenderer:
    """One libstnerf context (one GPU, one set of networks)."""

    def __init__(self, n_layers: int, space_time: Sequence[bool], precision: str = "fp32", chunk_rays: int = 0):
        if not torch.cuda.is_available():
            raise L.StnerfError("stnerf_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.l = int(n_layers)
        desc = L.ModelDesc()
        desc.n_layers = self.l
        for i in range(self.l):
            desc.space_time[i] = 1 if space_time[i] else 0
        desc.precision = L.PRECISIONS[precision] if isinstance(precision, str) else int(precision)
        desc.chunk_rays = int(chunk_rays)
        self._h = C.c_void_p()
        L.check(L.lib().stnerf_create(C.byref(self._h), C.byref(desc)), "stnerf_create")
        self._scene = None
        self._rotation = None

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            L.lib().stnerf_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ---------------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Upload a reference-format state_dict (SURVEY App. B key names)."""
        lib = L.lib()
        for fine, pre in ((0, "bkgd_spacenet."), (1, "bkgd_spacenet_fine.")):
            b = _blob(sd, pre, SPACENET_KEYS)
            L.check(lib.stnerf_load_spacenet(self._h, 0, fine, L.ptr(b), b.numel()), "load bkgd spacenet")
        for i in range(1, self.l):
            for fine, grp in ((0, "spacenets"), (1, "spacenets_fine")):
                b = _blob(sd, "%s.%d." % (grp, i - 1), SPACENET_KEYS)
                L.check(lib.stnerf_load_spacenet(self._h, i, fine, L.ptr(b), b.numel()), "load spacenet %d" % i)
            b = _blob(sd, "time_deform_nets.%d." % (i - 1), MOTIONNET_KEYS)
            L.check(lib.stnerf_load_motionnet(self._h, i, L.ptr(b), b.numel()), "load motionnet %d" % i)

    def export_weights(self) -> bytes:
        """Packed image of every loaded network (stnerf_weights_export): what `checkpoint_io.load_checkpoint_cached` stores."""
        need = C.c_size_t(0)
        L.check(L.lib().stnerf_weights_export(self._h, None, 0, C.byref(need)), "stnerf_weights_export(size)")
        buf = (C.c_uint8 * need.value)()
        L.check(L.lib().stnerf_weights_export(self._h, buf, need.value, C.byref(need)), "stnerf_weights_export")
        return bytes(buf)

    def import_weights(self, image: bytes):
        buf = (C.c_uint8 * len(image)).from_buffer_copy(image)
        L.check(L.lib().stnerf_weights_import(self._h, buf, len(image)), "stnerf_weights_import")

    def set_precision(self, precision):
        p = L.PRECISIONS[precision] if isinstance(precision, str) else int(precision)
        L.check(L.lib().stnerf_set_precision(self._h, p), "stnerf_set_precision")

    # ---- scene -----------------------------------------------------------------------------------------
    def set_scene(self, scene: L.Scene):
        self._scene = scene
        L.check(L.lib().stnerf_set_scene(self._h, C.byref(scene)), "stnerf_set_scene")

    def set_box_table(self, table: Optional[torch.Tensor]):
        """table (F, l, 2, 3) host fp32: edited min/max corners per frame and layer, for rays that carry their own frame id
        (stnerf_set_box_table); None removes it."""
        if table is None:
            L.check(L.lib().stnerf_set_box_table(self._h, None, 0), "stnerf_set_box_table")
            return
        t = table.detach().to("cpu", torch.float32).contiguous()
        assert t.dim() == 4 and tuple(t.shape[1:]) == (self.l, 2, 3), tuple(t.shape)
        L.check(L.lib().stnerf_set_box_table(self._h, L.ptr(t), int(t.shape[0])), "stnerf_set_box_table")

    def set_rotation(self, modes=None, R=None, centres=None):
        """Per-layer rotation (stnerf_set_rotation): modes (l,) of L.ROT_*, R (l,9) row-major, centres (l,3); modes=None
        clears it.  Host-side only; skipped when unchanged."""
        key = None if modes is None else tuple(np.ascontiguousarray(a).tobytes() for a in (modes, R, centres))
        if key == self._rotation:
            return
        if modes is None:
            L.check(L.lib().stnerf_set_rotation(self._h, None, None, None), "stnerf_set_rotation")
        else:
            m = np.ascontiguousarray(modes, dtype=np.int32)
            r = np.ascontiguousarray(R, dtype=np.float32)
            c = np.ascontiguousarray(centres, dtype=np.float32)
            assert m.shape == (self.l,) and r.shape == (self.l, 9) and c.shape == (self.l, 3)
            L.check(L.lib().stnerf_set_rotation(self._h, m.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p),
                                                c.ctypes.data_as(C.c_void_p)), "stnerf_set_rotation")
        self._rotation = key

    # ---- render ----------------------------------------------------------------------------------------
    def render(self, rays: torch.Tensor, n1: int, n2: int, only_coarse: bool = False,
               jitter: Optional[torch.Tensor] = None, u: Optional[torch.Tensor] = None, seed: int = 0,
               out: Optional[torch.Tensor] = None, ray_mask: Optional[torch.Tensor] = None):
        """rays (N, >=6+l) fp32 CUDA.  Returns out (2, l+1, 5N) fp32 and ray_mask (l, N) uint8."""
        assert rays.is_cuda and rays.dtype == torch.float32 and rays.dim() == 2
        rays = rays if rays.is_contiguous() else rays.contiguous()
        N = rays.shape[0]
        if out is None:
            out = torch.empty((2, self.l + 1, 5 * N), dtype=torch.float32, device=rays.device)
        if ray_mask is None:
            ray_mask = torch.empty((self.l, N), dtype=torch.uint8, device=rays.device)
        for t, shape in ((jitter, (self.l, N, n1)), (u, (self.l, N, n2))):
            if t is not None:
                assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape, \
                    (tuple(t.shape), shape)
        with torch.cuda.device(rays.device):
            L.check(L.lib().stnerf_render(self._h, L.ptr(rays), N, rays.stride(0), int(n1), int(n2),
                                          1 if only_coarse else 0, L.ptr(jitter), L.ptr(None if only_coarse else u),
                                          int(seed) & (2 ** 64 - 1), L.ptr(out), L.ptr(ray_mask), L.stream_ptr()),
                    "stnerf_render")
        return out, ray_mask

    def render_host(self, rays_host: torch.Tensor, n1: int, n2: int, only_coarse: bool = False, seed: int = 0,
                    out_host: Optional[torch.Tensor] = None, mask_host: Optional[torch.Tensor] = None):
        """Host-buffer entry (H2D + render + D2H inside the call): the end-to-end path."""
        assert not rays_host.is_cuda and rays_host.dtype == torch.float32 and rays_host.is_contiguous()
        N = rays_host.shape[0]
        if out_host is None:
            out_host = torch.empty((2, self.l + 1, 5 * N), dtype=torch.float32).pin_memory()
        if mask_host is None:
            mask_host = torch.empty((self.l, N), dtype=torch.uint8).pin_memory()
        L.check(L.lib().stnerf_render_host(self._h, L.ptr(rays_host), N, rays_host.stride(0), int(n1), int(n2),
                                           1 if only_coarse else 0, int(seed) & (2 ** 64 - 1), L.ptr(out_host),
                                           L.ptr(mask_host), L.stream_ptr()), "stnerf_render_host")
        return out_host, mask_host

    def reserve_host(self, max_rays: int, ray_stride: int):
        """Pre-size the device staging of render_host / render_views_host (stnerf_reserve_host): those calls then allocate nothing."""
        L.check(L.lib().stnerf_reserve_host(self._h, int(max_rays), int(ray_stride)), "stnerf_reserve_host")

    # ---- renderer-facing fast path: a batch of poses per native call (stnerf_render_views) -----------------------------------
    @staticmethod
    def make_view(K, T, frame_ids, scene: "L.Scene", seed: int) -> "L.View":
        """K (3,3), T (4,4) host tensors / arrays; frame_ids: one per layer; scene: the prologue's constants for this frame."""
        v = L.View()
        Kinv = torch.inverse(torch.as_tensor(K, dtype=torch.float32, device="cpu")).contiguous().reshape(-1)
        Th = torch.as_tensor(T, dtype=torch.float32, device="cpu").contiguous().reshape(-1)
        for i in range(9):
            v.Kinv[i] = float(Kinv[i])
        for i in range(16):
            v.T[i] = float(Th[i])
        for i, f in enumerate(frame_ids):
            v.frame_ids[i] = float(f)
        C.memmove(C.byref(v.scene), C.byref(scene), C.sizeof(L.Scene))
        v.seed = int(seed) & (2 ** 64 - 1)
        return v

    def render_views(self, views: Sequence["L.View"], H: int, W: int, n1: int, n2: int, row0: int = 0, row_step: int = 1,
                     n_rows: Optional[int] = None, out: Optional[torch.Tensor] = None,
                     coarse_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Fine images of every view, (n_views, l+1, n_rows*W, 5) = rgb, depth, acc per pixel, on the device.  Rays are generated
        on the device; `out` may be any contiguous CUDA fp32 tensor with that many elements per view (e.g. a slice of an
        all-gather buffer).  `coarse_out` (same shape): also produce the coarse images (everything forward() returns).
        Enqueue only."""
        n_rows = (H - row0 + row_step - 1) // row_step if n_rows is None else int(n_rows)
        nv = len(views)
        arr = (L.View * nv)(*views)
        dev = torch.device("cuda", torch.cuda.current_device())
        per = (self.l + 1) * n_rows * W * 5
        if out is None:
            out = torch.empty((nv, self.l + 1, n_rows * W, 5), dtype=torch.float32, device=dev)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == nv * per
        if coarse_out is not None:
            assert coarse_out.is_cuda and coarse_out.dtype == torch.float32 and coarse_out.is_contiguous() and coarse_out.numel() == nv * per
        L.check(L.lib().stnerf_render_views(self._h, arr, nv, int(H), int(W), int(row0), int(row_step), n_rows, int(n1), int(n2),
                                            L.ptr(out), L.ptr(coarse_out), per, L.stream_ptr()), "stnerf_render_views")
        return out

    def render_views_host(self, views: Sequence["L.View"], H: int, W: int, n1: int, n2: int,
                          out_host: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Full frames to pinned host memory, (n_views, l+1, H*W, 5); the copy of view v overlaps the rendering of view v+1.
        Returns after the last copy has landed."""
        nv = len(views)
        arr = (L.View * nv)(*views)
        if out_host is None:
            out_host = torch.empty((nv, self.l + 1, H * W, 5), dtype=torch.float32).pin_memory()
        assert (not out_host.is_cuda) and out_host.dtype == torch.float32 and out_host.is_contiguous()
        assert out_host.numel() == nv * (self.l + 1) * H * W * 5
        L.check(L.lib().stnerf_render_views_host(self._h, arr, nv, int(H), int(W), int(n1), int(n2), L.ptr(out_host),
                                                 L.stream_ptr()), "stnerf_render_views_host")
        return out_host

    # ---- per-stage entry points that need the networks ------------------------------------------------------
    def spacenet(self, layer: int, fine: bool, pos, dirs, times=None, render_schedule: bool = False):
        """rgb logits (P,3), raw sigma (P,1) of layer `layer`'s coarse / fine SpaceNet (stnerf_spacenet).  render_schedule: in the
        weight-stage schedule the render uses for that pass (stnerf_spacenet_pass; differs only in exact_cf's fine pass)."""
        P = pos.shape[0]
        # the contiguous fp32 copies stay bound to locals until the call has been enqueued (a temporary would be
        # released -- and its block reused by the next .contiguous() -- before the kernel runs)
        pos_c, dirs_c = _dev_f32(pos, "pos"), _dev_f32(dirs, "dirs")
        times_c = None if times is None else _dev_f32(times, "times")
        rgb = torch.empty((P, 3), dtype=torch.float32, device=pos_c.device)
        sig = torch.empty((P, 1), dtype=torch.float32, device=pos_c.device)
        with torch.cuda.device(pos_c.device):
            fn = L.lib().stnerf_spacenet_pass if render_schedule else L.lib().stnerf_spacenet
            L.check(fn(self._h, layer, 1 if fine else 0, L.ptr(pos_c), L.ptr(dirs_c), L.ptr(times_c), P, L.ptr(rgb), L.ptr(sig),
                       L.stream_ptr()), "stnerf_spacenet")
        del pos_c, dirs_c, times_c
        return rgb, sig

    def motionnet(self, layer: int, xyzt, lerp_mode: int = -1):
        P = xyzt.shape[0]
        xyzt_c = _dev_f32(xyzt, "xyzt")
        flow = torch.empty((P, 3), dtype=torch.float32, device=xyzt_c.device)
        with torch.cuda.device(xyzt_c.device):
            L.check(L.lib().stnerf_motionnet(self._h, layer, L.ptr(xyzt_c), P, lerp_mode, L.ptr(flow), L.stream_ptr()),
                    "stnerf_motionnet")
        del xyzt_c
        return flow

    def layer_field(self, layer: int, fine: bool, frame: float, xyz, dirs=None, want_rgb: bool = True):
        """The render's field of `layer` (pass `fine`) at frame `frame` at world points xyz (P,3) (stnerf_layer_field):
        rgb logits (P,3) or None, and raw sigma (P,).  want_rgb=False skips the colour; `dirs` (P,3) is needed otherwise."""
        xyz_c = _dev_f32(xyz, "xyz")
        P = xyz_c.shape[0]
        dirs_c = None if dirs is None else _dev_f32(dirs, "dirs")
        if want_rgb and dirs_c is None:
            raise ValueError("layer_field needs view directions for the colour")
        rgb = torch.empty((P, 3), dtype=torch.float32, device=xyz_c.device) if want_rgb else None
        sig = torch.empty((P,), dtype=torch.float32, device=xyz_c.device)
        with torch.cuda.device(xyz_c.device):
            L.check(L.lib().stnerf_layer_field(self._h, int(layer), 1 if fine else 0, float(frame), L.ptr(xyz_c), L.ptr(dirs_c), P,
                                               L.ptr(rgb), L.ptr(sig), L.stream_ptr()), "stnerf_layer_field")
        del xyz_c, dirs_c
        return rgb, sig

    def layer_grid(self, layer: int, fine: bool, frame: float, origin, step, dims, out: Optional[torch.Tensor] = None):
        """Raw sigma of the same field on the grid origin + (i,j,k)*step, (dims0, dims1, dims2) (stnerf_layer_grid); enqueue only."""
        g = make_grid(origin, step, dims)
        dev = torch.device("cuda", torch.cuda.current_device())
        if out is None:
            out = torch.empty(tuple(int(d) for d in dims), dtype=torch.float32, device=dev)
        assert out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == tuple(int(d) for d in dims)
        with torch.cuda.device(out.device):
            L.check(L.lib().stnerf_layer_grid(self._h, int(layer), 1 if fine else 0, float(frame), C.byref(g), L.ptr(out),
                                              L.stream_ptr()), "stnerf_layer_grid")
        return out

    def read_depths(self, fine: bool, layer: int, n_rays: int, S: int) -> torch.Tensor:
        """Sample depths (n_rays, S) of `layer` from the last chunk rendered (stnerf_debug_read_depths; parity tooling)."""
        out = torch.empty((n_rays, S), dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))
        L.check(L.lib().stnerf_debug_read_depths(self._h, 1 if fine else 0, int(layer), L.ptr(out), int(n_rays), int(S),
                                                 L.stream_ptr()), "stnerf_debug_read_depths")
        return out

    def read_origin(self, layer: int, n_rays: int, n1: int, n2: int):
        """z_new (n_rays, n2) and src_map (n_rays, n1+n2) uint8 of `layer` from the last chunk rendered: the new depths in
        ascending order and where every fine depth came from.  Raises unless that render reused the coarse pass' flow."""
        dev = torch.device("cuda", torch.cuda.current_device())
        z = torch.empty((n_rays, n2), dtype=torch.float32, device=dev)
        src = torch.empty((n_rays, n1 + n2), dtype=torch.uint8, device=dev)
        for what, dst in ((2, z), (3, src)):
            L.check(L.lib().stnerf_debug_read_depths(self._h, what, int(layer), L.ptr(dst), int(n_rays), int(dst.shape[1]),
                                                     L.stream_ptr()), "stnerf_debug_read_depths")
        return z, src

    def set_ray_ids(self, base: int = 0, width: int = 0, row_stride: int = 0):
        """Philox keys of the rays of subsequent render calls (see include/stnerf.h: stnerf_set_ray_ids)."""
        L.check(L.lib().stnerf_set_ray_ids(self._h, int(base), int(width), int(row_stride)), "stnerf_set_ray_ids")

    def profile_begin(self):
        L.check(L.lib().stnerf_profile_begin(self._h), "stnerf_profile_begin")

    def profile_end(self) -> dict:
        """Per kernel class device time (CUDA events on the launching stream): SpaceNet, MotionNet, sampling, compositing."""
        p = L.Profile()
        L.check(L.lib().stnerf_profile_end(self._h, C.byref(p)), "stnerf_profile_end")
        names = ("spacenet", "motionnet", "sample", "composite")
        return {n: {"ms": p.ms[i], "points": p.points[i], "launches": int(p.launches[i])} for i, n in enumerate(names)}

    def workspace_bytes(self) -> int:
        return int(L.lib().stnerf_workspace_bytes(self._h))


def split_planes(out: torch.Tensor, l: int):
    """(2, l+1, 5N) planes -> (fine_mixed, coarse_mixed, fine_layer, coarse_layer) tuples of (rgb, depth, acc)."""
    N = out.shape[2] // 5

    def trip(p):
        return (p[:3 * N].view(N, 3), p[3 * N:4 * N].view(N, 1), p[4 * N:].view(N, 1))

    coarse_mixed, fine_mixed = trip(out[0, 0]), trip(out[1, 0])
    coarse_layer = [trip(out[0, 1 + i]) for i in range(l)]
    fine_layer = [trip(out[1, 1 + i]) for i in range(l)]
    return fine_mixed, coarse_mixed, fine_layer, coarse_layer


def make_grid(origin, step, dims) -> "L.Grid":
    g = L.Grid()
    for a in range(3):
        g.origin[a], g.step[a], g.dims[a] = float(origin[a]), float(step[a]), int(dims[a])
    return g


def marching_cubes(sigma: torch.Tensor, origin, step, level: float):
    """Indexed triangle mesh of the level set `sigma > level` of a CUDA fp32 grid (D0, D1, D2) whose point (i,j,k) lies at
    origin + (i,j,k)*step (stnerf_mc_count / stnerf_mc_fill): verts (V,3) fp32 and faces (F,3) int32 on the device."""
    s = _dev_f32(sigma, "sigma")
    assert s.dim() == 3, tuple(s.shape)
    g = make_grid(origin, step, s.shape)
    lib = L.lib()
    nbytes = int(lib.stnerf_mc_scratch_bytes(C.byref(g)))
    if nbytes == 0:
        raise L.StnerfError("marching_cubes: invalid grid (every dimension >= 2, finite origin, finite positive steps, < 2^31 points)")
    with torch.cuda.device(s.device):
        scratch = torch.empty((nbytes,), dtype=torch.uint8, device=s.device)
        nv, nf = C.c_int64(0), C.c_int64(0)
        L.check(lib.stnerf_mc_count(L.ptr(s), C.byref(g), float(level), L.ptr(scratch), nbytes, C.byref(nv), C.byref(nf),
                                    L.stream_ptr()), "stnerf_mc_count")
        verts = torch.empty((nv.value, 3), dtype=torch.float32, device=s.device)
        faces = torch.empty((nf.value, 3), dtype=torch.int32, device=s.device)
        if nv.value > 0:
            L.check(lib.stnerf_mc_fill(L.ptr(s), C.byref(g), float(level), L.ptr(scratch), nbytes, L.ptr(verts), L.ptr(faces),
                                       L.stream_ptr()), "stnerf_mc_fill")
    del s, scratch
    return verts, faces


def rotate_rays(rays: torch.Tensor, R, centre) -> torch.Tensor:
    """A rotated layer's rays (stnerf_rotate_rays): columns 0..5 -> (c + R^T (o - c), R^T d), the rest copied.  rays (N, C)
    contiguous fp32 CUDA; R (3,3), centre (3,)."""
    r = _dev_f32(rays, "rays")
    assert r.dim() == 2 and r.shape[1] >= 6
    Rh = np.ascontiguousarray(np.asarray(R, dtype=np.float32).reshape(9))
    ch = np.ascontiguousarray(np.asarray(centre, dtype=np.float32).reshape(3))
    out = torch.empty_like(r)
    with torch.cuda.device(r.device):
        L.check(L.lib().stnerf_rotate_rays(L.ptr(r), r.shape[0], r.shape[1], Rh.ctypes.data_as(C.c_void_p),
                                           ch.ctypes.data_as(C.c_void_p), L.ptr(out), L.stream_ptr()), "stnerf_rotate_rays")
    del r
    return out


def launch_count() -> int:
    return int(L.lib().stnerf_launch_count())
