"""Differentiable volume rendering: layers/render_layer.py:8-58 (gen_weight + VolumeRenderer.forward) and the depth-merged
composite of modeling/layered_rfrender.py:425-448 (coarse) / :587-606 (fine), with gradients in rgb and sigma.

The forward is `ops.composite` (csrc/composite.cu, composite_simple_kernel), so the outputs are its bits.  The backward is
`stnerf_composite_backward`, which recomputes alpha, the transmittance and the weights from (t, rgb, sigma): nothing but the
inputs is saved, and nothing at all when no gradient is wanted.  Identical calls give identical gradients (no atomics).
Depths get no gradient, as in the reference (layered_rfrender.py:314-315,461): a `t` that requires one raises
NotImplementedError.

There is no CPU path: CPU tensors raise StnerfError.
"""
from __future__ import annotations

import torch

from . import _lib as L
from . import ops


def _wants_grad(*xs) -> bool:
    return torch.is_grad_enabled() and any(x.requires_grad for x in xs)


class CompositeFunction(torch.autograd.Function):
    """(t (N,S), rgb (N,S,3) raw, sigma (N,S) raw, boarder) -> color (N,3), depth (N,1), acc (N,1), w (N,S)."""

    @staticmethod
    def forward(ctx, t, rgb, sigma, boarder):
        if ctx.needs_input_grad[0]:
            raise NotImplementedError("compositing has no gradient with respect to the depths (the reference detaches them)")
        ctx.set_materialize_grads(False)
        color, depth, acc, w = ops.composite(t, rgb, sigma, boarder)
        ctx.save_for_backward(*(ops._f32(x) for x in (t, rgb, sigma)))
        ctx.boarder = float(boarder)
        return color, depth, acc, w

    @staticmethod
    def backward(ctx, d_color, d_depth, d_acc, d_w):
        t, rgb, sigma = ctx.saved_tensors
        N, S = t.shape
        d_rgb = torch.empty((N, S, 3), dtype=torch.float32, device=t.device)
        d_sigma = torch.empty((N, S), dtype=torch.float32, device=t.device)
        up = [None if g is None else g.to(torch.float32).contiguous() for g in (d_color, d_depth, d_acc, d_w)]
        with torch.cuda.device(t.device):
            L.check(L.lib().stnerf_composite_backward(L.ptr(t), L.ptr(rgb), L.ptr(sigma), N, S, ctx.boarder,
                                                      *(L.ptr(g) for g in up), L.ptr(d_rgb), L.ptr(d_sigma), L.stream_ptr()),
                    "stnerf_composite_backward")
        return None, d_rgb, d_sigma, None


def composite(t, rgb, sigma, boarder: float = 1e10):
    """layers/render_layer.py:8-58.  t (N,S), rgb (N,S,3) raw, sigma (N,S) raw -> color (N,3), depth (N,1), acc (N,1),
    w (N,S); all differentiable in rgb and sigma."""
    for x in (t, rgb, sigma):
        if not x.is_cuda:
            raise L.StnerfError("stnerf_b200 compositing takes CUDA tensors (no CPU fallback)")
    if _wants_grad(t):
        raise NotImplementedError("compositing has no gradient with respect to the depths (the reference detaches them)")
    N, S = t.shape
    if N == 0:                     # no rays: nothing to launch (an empty tensor has no buffer to hand to the kernel)
        outs = [torch.zeros(s, dtype=torch.float32, device=t.device) for s in ((0, 3), (0, 1), (0, 1), (0, S))]
        if _wants_grad(rgb, sigma):
            keep = (rgb.sum() + sigma.sum()) * 0.0          # sums over no element: joins the graph, adds nothing
            outs = [o + keep for o in outs]
        return tuple(outs)
    if not _wants_grad(rgb, sigma):
        return ops.composite(t, rgb, sigma, boarder)
    return CompositeFunction.apply(t, rgb, sigma, boarder)


def composite_merged(ts, rgbs, sigmas, boarder: float = 1e10, near=None):
    """The depth-merged composite of all layers: layered_rfrender.py:425-448 (coarse) and, with `near`, :587-606 (fine, where
    the merged density is zeroed in front of the near plane).  ts: per layer (N,S_i); rgbs (N,S_i,3); sigmas (N,S_i) or
    (N,S_i,1).  The depths are sorted stably, so ties resolve in (t, concatenation index) order like the render kernels.
    -> color (N,3), depth (N,1), acc (N,1), differentiable in every layer's rgb and sigma (the gather's gradient is a scatter
    that hits each sample once)."""
    n = ts[0].shape[0]
    t_cat = torch.cat([t.reshape(n, -1) for t in ts], 1)
    tm, order = torch.sort(t_cat, dim=1, stable=True)
    rm = torch.cat([r.reshape(n, -1, 3) for r in rgbs], 1).gather(1, order[..., None].expand(-1, -1, 3))
    sm = torch.cat([s.reshape(n, -1) for s in sigmas], 1).gather(1, order)
    if near is not None:
        sm = torch.where(tm < near, torch.zeros_like(sm), sm)
    color, depth, acc, _ = composite(tm, rm, sm, boarder)
    return color, depth, acc
