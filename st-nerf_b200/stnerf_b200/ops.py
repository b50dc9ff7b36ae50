"""Per-stage operators (no network weights needed): each mirrors one reference function and calls one C-ABI
entry point.  Inputs are CUDA fp32 tensors; outputs are fresh CUDA tensors.  No CPU fallback."""
from __future__ import annotations

import ctypes

import torch

from . import _lib as L


def _f32(t: torch.Tensor) -> torch.Tensor:
    if not t.is_cuda:
        raise L.StnerfError("stnerf_b200 operators take CUDA tensors (no CPU fallback)")
    return t.detach().to(torch.float32).contiguous()


def _host3(v):
    return torch.as_tensor(v, dtype=torch.float32, device="cpu").reshape(3).contiguous()


def intersect_sample(rays, bmin, bmax, n1: int, jitter, is_bkgd: bool = False, want_xyz: bool = True):
    """layers/RaySamplePoint.py:8-62 + :85-105 for one axis-aligned box.  -> t (N,n1), xyz (N,n1,3), mask (N) bool,
    tfar_tnear (N,2)."""
    rays, jitter = _f32(rays), _f32(jitter)
    N = rays.shape[0]
    bmin, bmax = _host3(bmin), _host3(bmax)
    t = torch.empty((N, n1), dtype=torch.float32, device=rays.device)
    xyz = torch.empty((N, n1, 3), dtype=torch.float32, device=rays.device) if want_xyz else None
    mask = torch.empty((N,), dtype=torch.uint8, device=rays.device)
    tt = torch.empty((N, 2), dtype=torch.float32, device=rays.device)
    L.check(L.lib().stnerf_intersect_sample(L.ptr(rays), N, rays.stride(0), L.ptr(bmin), L.ptr(bmax),
                                            1 if is_bkgd else 0, int(n1), L.ptr(jitter), L.ptr(t), L.ptr(xyz),
                                            L.ptr(mask), L.ptr(tt), L.stream_ptr()), "stnerf_intersect_sample")
    return t, xyz, mask.bool(), tt


def composite(t, rgb, sigma, boarder: float = 1e10, want_weights: bool = True):
    """layers/render_layer.py:25-58.  t (N,S), rgb (N,S,3), sigma (N,S) -> color (N,3), depth (N,1), acc (N,1), w (N,S)."""
    t, rgb, sigma = _f32(t), _f32(rgb), _f32(sigma)
    N, S = t.shape
    color = torch.empty((N, 3), dtype=torch.float32, device=t.device)
    depth = torch.empty((N, 1), dtype=torch.float32, device=t.device)
    acc = torch.empty((N, 1), dtype=torch.float32, device=t.device)
    w = torch.empty((N, S), dtype=torch.float32, device=t.device) if want_weights else None
    L.check(L.lib().stnerf_composite(L.ptr(t), L.ptr(rgb), L.ptr(sigma), N, S, float(boarder), L.ptr(color),
                                     L.ptr(depth), L.ptr(acc), L.ptr(w), L.stream_ptr()), "stnerf_composite")
    return color, depth, acc, w


def sample_pdf(t, w, u, merge: bool = False):
    """utils/sample_pdf.py:18-63 with explicit uniforms.  t (N,n1), w (N,n1) full weights, u (N,n2).
    Returns z (N,n2); with merge=True also sort(cat(t,z)) (N,n1+n2) (layered_rfrender.py:462)."""
    t, w, u = _f32(t), _f32(w), _f32(u)
    N, n1 = t.shape
    n2 = u.shape[1]
    z = torch.empty((N, n2), dtype=torch.float32, device=t.device)
    tf = torch.empty((N, n1 + n2), dtype=torch.float32, device=t.device) if merge else None
    L.check(L.lib().stnerf_sample_pdf(L.ptr(t), L.ptr(w), L.ptr(u), N, n1, n2, L.ptr(z), L.ptr(tf), L.stream_ptr()),
            "stnerf_sample_pdf")
    return (z, tf) if merge else z


def composite_pass(scene: "L.Scene", t, raw, mask, fine: bool = False, n2: int = 0, u=None, seed: int = 0,
                   pixel_layout: int = 0, want_images: bool = True, want_origin: bool = False, t_fine=None):
    """One compositing pass of the render path on explicit network outputs (stnerf_composite_pass): density masks, every hit
    layer's own image, the depth-ordered merge and, in a coarse pass with n2 > 0, the resampling.
    t (l,N,S), raw (l,N,S,4) = rgb logits + raw sigma, mask (l,N) uint8/bool, u (l,N,n2) or None = Philox(seed).
    Returns a dict: images (l+1, 5N) (pixel_layout 0: rgb (N,3) | depth (N) | acc (N) per image; 1: (N,5) interleaved),
    t_fine (l,N,S+n2) when n2 > 0 (`t_fine`: a caller's buffer to write into -- rows of missed layers are left untouched),
    and with want_origin z_new (l,N,n2) and src_map (l,N,S+n2) uint8."""
    t, raw = _f32(t), _f32(raw)
    l, N, S = t.shape
    assert tuple(raw.shape) == (l, N, S, 4), tuple(raw.shape)
    mask = mask.to(device=t.device, dtype=torch.uint8).contiguous()
    assert tuple(mask.shape) == (l, N), tuple(mask.shape)
    if u is not None:
        u = _f32(u)
        assert tuple(u.shape) == (l, N, n2), tuple(u.shape)
    out = {}
    if want_images:
        out["images"] = torch.empty((l + 1, 5 * N), dtype=torch.float32, device=t.device)
    if n2 > 0:
        if t_fine is None:
            t_fine = torch.zeros((l, N, S + n2), dtype=torch.float32, device=t.device)
        assert t_fine.is_cuda and t_fine.dtype == torch.float32 and t_fine.is_contiguous() and tuple(t_fine.shape) == (l, N, S + n2)
        out["t_fine"] = t_fine
    if want_origin:
        out["z_new"] = torch.zeros((l, N, n2), dtype=torch.float32, device=t.device)
        out["src_map"] = torch.zeros((l, N, S + n2), dtype=torch.uint8, device=t.device)
    with torch.cuda.device(t.device):
        L.check(L.lib().stnerf_composite_pass(ctypes.byref(scene), l, 1 if fine else 0, L.ptr(t), L.ptr(raw), L.ptr(mask), L.ptr(u),
                                              int(seed) & (2 ** 64 - 1), N, S, int(n2), int(pixel_layout),
                                              L.ptr(out.get("images")), L.ptr(out.get("t_fine")), L.ptr(out.get("z_new")),
                                              L.ptr(out.get("src_map")), L.stream_ptr()), "stnerf_composite_pass")
    return out


def positional_encoding(x, n_freq: int):
    """utils/dimension_kernel.py:24-33.  x (P,dim) -> (P, dim*(1+2*n_freq))."""
    x = _f32(x)
    P, dim = x.shape
    out = torch.empty((P, dim * (1 + 2 * n_freq)), dtype=torch.float32, device=x.device)
    L.check(L.lib().stnerf_positional_encoding(L.ptr(x), P, dim, int(n_freq), L.ptr(out), L.stream_ptr()),
            "stnerf_positional_encoding")
    return out


def generate_rays(K, T, h: int, w: int, frame_ids=None, device=None, row0: int = 0, row_step: int = 1, n_rows=None):
    """utils/render_helpers.py:96-123 / utils/ray_sampling.py:22-72 on the GPU.  K (3,3), T (4,4) host tensors.
    Returns rays (n_rows*w, 6+len(frame_ids)) for image rows row0, row0+row_step, ..."""
    device = torch.device(device if device is not None else "cuda")
    Kinv = torch.inverse(torch.as_tensor(K, dtype=torch.float32, device="cpu")).contiguous()
    Th = torch.as_tensor(T, dtype=torch.float32, device="cpu").contiguous()
    fid = None if frame_ids is None else torch.as_tensor(frame_ids, dtype=torch.float32, device="cpu").contiguous()
    nf = 0 if fid is None else fid.numel()
    if n_rows is None:
        n_rows = (h - row0 + row_step - 1) // row_step
    rays = torch.empty((n_rows * w, 6 + nf), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        L.check(L.lib().stnerf_raygen(L.ptr(Kinv), L.ptr(Th), int(h), int(w), int(row0), int(row_step), int(n_rows),
                                      L.ptr(fid), nf, L.ptr(rays), rays.stride(0), L.stream_ptr()), "stnerf_raygen")
    return rays
