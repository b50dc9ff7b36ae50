"""Trainable `LayeredRFRender`: network parameters and a differentiable forward on the native kernels.

`TrainableLayeredRFRender` registers the reference's networks as submodules (`spacenets`, `spacenets_fine`,
`bkgd_spacenet`, `bkgd_spacenet_fine`, `time_deform_nets`, in the reference's order, modeling/layered_rfrender.py:59-93), so
`parameters()`, `state_dict()`, `load_state_dict()`, `.cuda()` and `.to()` behave as for the reference module and an
optimiser built by solver/build.py sees every network parameter.

`forward` keeps LayeredRFRender's signature and 5-tuple.  With gradients enabled and a parameter that requires one, it runs
the differentiable forward of layered_rfrender.py:141-734: sampling and ordered hit lists (`stnerf_train_sample`), per layer
and pass the compact network inputs (`stnerf_train_points`), MotionNet and SpaceNet on the training kernels
(`nets.MotionNetFunction` / `nets.SpaceNetFunction`), the masked scatter into the sample grid (`stnerf_train_scatter`, backward
`stnerf_train_gather`), the per-layer and merged composites (`volume`), and the fine depths from `stnerf_sample_pdf`.  Depths,
sample points and rays get no gradient, as in the reference (:314-315,461).  `train_precision` (default
cfg.MODEL.B200_TRAIN_PRECISION, else "fp32") selects the networks' training kernels and is applied to every network submodule:
"fp32" on CUDA cores, or "tf32x3" on tensor cores (nets.py).  `precision` selects only the render path, which every other call
takes (e.g. the evaluator's under `torch.no_grad()`), with the current weights -- re-uploaded when a parameter changed since the
last upload.

Without injected uniforms both paths draw the same Philox streams, so a grad and a no-grad forward with the same `seed` place
the same samples.  Identical calls give bit-identical gradients: the hit lists are in ray order and every kernel on the path
sums in a fixed order.

`trace` (default None) is a debugging and testing hook: a callable `trace(name, x)` that sees the intermediate tensors of a
differentiable forward and may return a replacement for a network output (None keeps `x`).  Names: "t_coarse" (l,N,n1),
"mask" (l,N) uint8, "t_fine.<i>" (N,n1+n2); per network call, in hit order, "flow.<p><i>" (MotionNet), "rgb.<p><i>" and
"sigma.<p><i>" (SpaceNet), with <p> = "c" (coarse pass) or "f" (fine pass) and <i> the layer.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import torch
from torch import nn

from . import _lib as L
from . import ops, volume
from .model import LayeredRFRender
from .native import MOTIONNET_KEYS, SPACENET_KEYS, NativeRenderer
from .nets import MotionNet, MotionNetFunction, SpaceNet, SpaceNetFunction, _params


class _ScatterFunction(torch.autograd.Function):
    """Compact (rgb (P,3), sigma (P,1)) of one layer and pass -> dense masked rgb (N,S,3), sigma (N,S)
    (`rgbs[i][idx] = ...; density[i][idx] = ...` and the density masks, layered_rfrender.py:397-422 / :552-576)."""

    @staticmethod
    def forward(ctx, rgb_c, sigma_c, nat, layer, fine, t, hit, m):
        ctx.set_materialize_grads(False)
        N, S = t.shape
        dev = t.device
        rgb_c, sigma_c = rgb_c.detach().contiguous(), sigma_c.detach().contiguous()
        rgb = torch.empty((N, S, 3), dtype=torch.float32, device=dev)
        sigma = torch.empty((N, S), dtype=torch.float32, device=dev)
        factor = torch.empty((m * S,), dtype=torch.float32, device=dev)
        L.check(L.lib().stnerf_train_scatter(nat._h, layer, int(fine), L.ptr(t), N, S, L.ptr(hit), m, L.ptr(rgb_c),
                                             L.ptr(sigma_c), L.ptr(rgb), L.ptr(sigma), L.ptr(factor), L.stream_ptr()),
                "stnerf_train_scatter")
        ctx.save_for_backward(factor, hit)
        ctx.nat, ctx.S, ctx.m = nat, S, m
        return rgb, sigma

    @staticmethod
    def backward(ctx, d_rgb, d_sigma):
        factor, hit = ctx.saved_tensors
        P, dev = ctx.m * ctx.S, factor.device
        d_rgb = None if d_rgb is None else d_rgb.to(torch.float32).contiguous()
        d_sigma = None if d_sigma is None else d_sigma.to(torch.float32).contiguous()
        d_rgb_c = torch.empty((P, 3), dtype=torch.float32, device=dev)
        d_sigma_c = torch.empty((P, 1), dtype=torch.float32, device=dev)
        L.check(L.lib().stnerf_train_gather(ctx.nat._h, ctx.S, L.ptr(hit), ctx.m, L.ptr(factor), L.ptr(d_rgb), L.ptr(d_sigma),
                                            L.ptr(d_rgb_c), L.ptr(d_sigma_c), L.stream_ptr()), "stnerf_train_gather")
        return d_rgb_c, d_sigma_c, None, None, None, None, None, None


class TrainableLayeredRFRender(LayeredRFRender):
    """LayeredRFRender with the reference's network submodules and a differentiable forward (module docstring)."""

    def __init__(self, cfg, camera_num=0, scale=None, shift=None, precision=None, train_precision=None, rotation=None):
        super().__init__(cfg, camera_num=camera_num, scale=scale, shift=shift, precision=precision, rotation=rotation)
        tp = train_precision or getattr(cfg.MODEL, "B200_TRAIN_PRECISION", "fp32")
        L.train_precision_code(tp)
        self.train_precision = tp
        n = self.layer_num
        # registration order = the reference's (layered_rfrender.py:59-93) = key order of fresh_state_dict / the checkpoints
        self.spacenets = nn.ModuleList([SpaceNet(use_time=self.use_space_time, train_precision=tp) for _ in range(n)])
        self.spacenets_fine = nn.ModuleList([SpaceNet(use_time=self.use_space_time, train_precision=tp) for _ in range(n)])
        self.bkgd_spacenet = SpaceNet(use_time=self.bkgd_use_space_time, train_precision=tp)
        self.bkgd_spacenet_fine = SpaceNet(use_time=self.bkgd_use_space_time, train_precision=tp)
        self.time_deform_nets = nn.ModuleList([MotionNet(c_input=4, input_time=True, train_precision=tp) for _ in range(n)])
        nn.Module.load_state_dict(self, self._sd)       # the reference's initialisation (fresh_state_dict)
        self._weights_key = None
        self._grad_call = False
        self.trace = None

    # ---- a plain nn.Module again: parameters live in the submodules ---------------------------------------------------------
    def state_dict(self, *args, **kwargs):
        return nn.Module.state_dict(self, *args, **kwargs)

    def load_state_dict(self, state_dict, strict=True, assign=False):
        return nn.Module.load_state_dict(self, state_dict, strict=strict, assign=assign)

    def cuda(self, device=None):
        return nn.Module.cuda(self, device)

    def load_packed(self, image: bytes, state_dict_source=None):
        # StnerfError: checkpoint_io.load_checkpoint_cached then falls back to the plain state_dict load
        raise L.StnerfError("a trainable model takes its weights from its parameters, not from a packed image: use load_state_dict")

    def _param_key(self):
        return tuple((p.data_ptr(), p.device, p._version) for p in self.parameters())

    def _sync_weights(self):
        """The render path's weights are the parameters: re-upload when any of them changed since the last upload."""
        key = self._param_key()
        if key != self._weights_key:
            self._sd = OrderedDict((k, v.detach().to("cpu", torch.float32).clone()) for k, v in nn.Module.state_dict(self).items())
            self._uploaded = False
            self._weights_key = key

    def _ensure_native(self, device):
        if self._grad_call:                  # the training kernels read the parameters in place: no upload
            if self._native is None:
                with torch.cuda.device(device):
                    st = [self.bkgd_use_space_time] + [self.use_space_time] * self.layer_num
                    self._native = NativeRenderer(self.layer_num + 1, st, self.precision, self.chunk_rays)
            return self._native
        self._sync_weights()
        return super()._ensure_native(device)

    # ---- forward ---------------------------------------------------------------------------------------------------------------
    def forward(self, rays, labels=None, bboxes=None, only_coarse=False, near_far=None, near_far_points=[],
                density_threshold=0.0001, bkgd_density_threshold=0):
        """layered_rfrender.py:141-734.  `labels`, `bboxes`, `near_far` are ignored, as in the reference's BBOX path (the boxes
        come from set_bboxes, :193-204).  Differentiable when gradients are enabled and a parameter requires one."""
        self._grad_call = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if not self._grad_call:
            return super().forward(rays, labels, bboxes, only_coarse, near_far, near_far_points, density_threshold,
                                   bkgd_density_threshold)
        try:
            return self._train_forward(rays, bool(only_coarse), density_threshold, bkgd_density_threshold)
        finally:
            self._grad_call = False

    def _see(self, name, x):
        if self.trace is None:
            return x
        y = self.trace(name, x)
        return x if y is None else y

    def _train_forward(self, rays, only_coarse, density_threshold, bkgd_density_threshold):
        l = self.layer_num + 1
        nat, rays = self._prologue(rays, density_threshold, bkgd_density_threshold)
        for p in self.parameters():
            if p.device != rays.device:
                raise L.StnerfError("the parameters are on %s and the rays on %s: move the model with .cuda()" %
                                    (p.device, rays.device))
        N, dev = rays.shape[0], rays.device
        n1, n2 = self.coarse_ray_sample, 0 if only_coarse else self.fine_ray_sample
        if n1 + n2 > L.MAX_S:
            raise ValueError("n1 + n2 = %d samples exceed the %d the kernels support" % (n1 + n2, L.MAX_S))
        jitter, u = self._inject if self._inject is not None else (None, None)
        self._inject = None
        self.seed += 1
        for x, shape in ((jitter, (l, N, n1)), (u if n2 > 0 else None, (l, N, n2))):
            if x is not None and not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and tuple(x.shape) == shape):
                raise ValueError("injected uniforms must be contiguous CUDA float32 of shape %s, got %s" % (shape, tuple(x.shape)))
        t_c = torch.empty((l, N, n1), dtype=torch.float32, device=dev)
        mask = torch.empty((l, N), dtype=torch.uint8, device=dev)
        hit = torch.empty((l, N), dtype=torch.int32, device=dev)
        counts, frac = (C.c_int32 * l)(), (C.c_int32 * l)()
        with torch.cuda.device(dev):
            L.check(L.lib().stnerf_train_sample(nat._h, L.ptr(rays), N, rays.stride(0), n1, L.ptr(jitter), self.seed & (2 ** 64 - 1),
                                                L.ptr(t_c), L.ptr(mask), L.ptr(hit), counts, frac, L.stream_ptr()),
                    "stnerf_train_sample")
            self._see("t_coarse", t_c)
            self._see("mask", mask)
            lists = [(None, N, 0)] + [(hit[i], int(counts[i]), int(frac[i])) for i in range(1, l)]
            coarse_layer, coarse_mixed, w_c = self._pass(nat, rays, [t_c[i] for i in range(l)], lists, fine=False)
            if only_coarse:                                                       # :721-722
                ray_mask = [mask[i].bool() for i in range(l)]
                return coarse_mixed, coarse_mixed, coarse_layer, coarse_layer, ray_mask
            if u is None:
                u = torch.empty((l, N, n2), dtype=torch.float32, device=dev)
                L.check(L.lib().stnerf_train_uniforms(nat._h, N, n2, self.seed & (2 ** 64 - 1), L.ptr(u), L.stream_ptr()),
                        "stnerf_train_uniforms")
            # :459-463: resample on the detached coarse weights of each layer, sort(cat(t, z))
            t_f = [ops.sample_pdf(t_c[i], w_c[i], u[i], merge=True)[1] for i in range(l)]
            for i in range(l):
                self._see("t_fine.%d" % i, t_f[i])
            fine_layer, fine_mixed, _ = self._pass(nat, rays, t_f, lists, fine=True)
        ray_mask = [mask[i].bool() for i in range(l)]
        return fine_mixed, coarse_mixed, fine_layer, coarse_layer, ray_mask

    def _pass(self, nat, rays, ts, lists, fine):
        """One pass over every layer: networks, masked scatter, per-layer composites, the merged composite (:379-448 coarse,
        :526-606 fine).  Returns the per-layer (rgb, depth, acc), the merged one and the detached per-layer weights."""
        rgbs, sigmas, layer_out, weights = [], [], [], []
        for i, t in enumerate(ts):
            hit, m, frac = lists[i]
            N, S = t.shape
            if i > 0 and (m == 0 or self.display_layers.get(i, 1) != 1):      # no network: sigma = rgb = 0 (:401, :556)
                rgb = torch.zeros((N, S, 3), dtype=torch.float32, device=t.device)
                sigma = torch.zeros((N, S), dtype=torch.float32, device=t.device)
            else:
                rgb, sigma = self._layer(nat, rays, i, fine, t, hit, m, frac)
            color, depth, acc, w = volume.composite(t, rgb, sigma, self.boarder_weight)
            rgbs.append(rgb)
            sigmas.append(sigma)
            layer_out.append((color, depth, acc))
            weights.append(w.detach())
        mixed = volume.composite_merged(ts, rgbs, sigmas, self.boarder_weight, float(self.near) if fine else None)
        return layer_out, mixed, weights

    def _layer(self, nat, rays, i, fine, t, hit, m, frac):
        N, S = t.shape
        P, dev = m * S, t.device
        use_time = self.bkgd_use_space_time if i == 0 else self.use_space_time
        dirs = torch.empty((P, 3), dtype=torch.float32, device=dev)
        times = torch.empty((P, 1), dtype=torch.float32, device=dev) if use_time else None
        pos = torch.empty((P, 3), dtype=torch.float32, device=dev) if i == 0 else None
        xyzt = torch.empty((P, 4), dtype=torch.float32, device=dev) if i > 0 else None
        L.check(L.lib().stnerf_train_points(nat._h, i, int(fine), L.ptr(rays), N, rays.stride(0), L.ptr(t), S, L.ptr(hit), m,
                                            L.ptr(pos), L.ptr(dirs), L.ptr(times), L.ptr(xyzt), L.stream_ptr()),
                "stnerf_train_points")
        if i > 0:                                                                  # :340-356 / :495-510
            mnet = self.time_deform_nets[i - 1]
            flow = MotionNetFunction.apply(xyzt, frac, mnet.train_precision, *_params(mnet, MOTIONNET_KEYS))
            flow = self._see("flow.%s%d" % ("f" if fine else "c", i), flow)
            pos = xyzt[:, :3] + flow
            net = (self.spacenets_fine if fine else self.spacenets)[i - 1]
        else:
            net = self.bkgd_spacenet_fine if fine else self.bkgd_spacenet
        rgb_c, sigma_c = SpaceNetFunction.apply(pos, dirs, times, use_time, net.train_precision, *_params(net, SPACENET_KEYS))
        tag = "%s%d" % ("f" if fine else "c", i)
        rgb_c, sigma_c = self._see("rgb." + tag, rgb_c), self._see("sigma." + tag, sigma_c)
        return _ScatterFunction.apply(rgb_c, sigma_c, nat, i, fine, t, hit, m)
