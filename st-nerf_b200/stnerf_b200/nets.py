"""Trainable SpaceNet and MotionNet: `torch.nn.Module`s over the native training kernels (csrc/mlp_train.cu, mlp_train_tc.cu).

The modules have the reference's constructors, parameter names and shapes (modeling/spacenet.py:17-86,
modeling/motion_net.py:6-31) and `forward` signatures, so a reference checkpoint's `spacenets.0.*` /
`time_deform_nets.0.*` tensors load into them unchanged.  Forward and backward run in libstnerf_b200.so: fp32 products
with fp32 accumulation, the forward bit-identical to the `fp32` render mode, the weight gradients summed over the points in
a fixed order (identical calls, identical bits).  Directions, times and MotionNet's input get no gradient, as in the
reference (modeling/layered_rfrender.py:272,314-315); `pos` does when it requires one.

`from_layered(model)` collects the networks of a `LayeredRFRender` so that they can be fine-tuned and written back:
`model.load_state_dict(from_layered(model).state_dict())` round-trips.

`train_precision` selects the kernels: "fp32" (default, above) or "tf32x3", which runs every GEMM of the layers with 128 or
more outputs -- forward, input deltas and weight gradients -- on Hopper tensor cores with 3xTF32 products (about 22 significant
bits per product, fp32's exponent range; DESIGN.md section 3.8).  A tf32x3 forward is not bit-identical to any render mode;
its backward runs in the precision its forward ran in.

There is no CPU path: CPU tensors raise StnerfError.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib as L
from .native import MOTIONNET_KEYS, SPACENET_KEYS

SPACENET, MOTIONNET = 0, 1


def _dev_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise L.StnerfError("%s must be a CUDA tensor (no CPU fallback)" % name)
    return t.detach().to(torch.float32).contiguous()


def _blob(params) -> torch.Tensor:
    """The parameters as one stnerf_load_* blob (state_dict order, nn.Linear (out, in) row-major)."""
    for p in params:
        if not p.is_cuda:
            raise L.StnerfError("the network's parameters must be on a CUDA device (no CPU fallback): call .cuda()")
    return torch.cat([p.detach().to(torch.float32).reshape(-1) for p in params])


def _split_grad(d_blob: torch.Tensor, params):
    out, off = [], 0
    for p in params:
        n = p.numel()
        out.append(d_blob[off:off + n].view(p.shape).to(p.dtype))
        off += n
    return out


def _scratch(kind: int, use_time: bool, P: int, device, prec: int) -> torch.Tensor:
    nbytes = L.lib().stnerf_train_scratch_bytes_prec(kind, int(use_time), P, prec)
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


class SpaceNetFunction(torch.autograd.Function):
    """(pos (P,3), dirs (P,3), times (P,1) | None, use_time, train_precision, *parameters) -> rgb (P,3) raw, sigma (P,1) raw."""

    @staticmethod
    def forward(ctx, pos, dirs, times, use_time, train_precision, *params):
        prec = L.train_precision_code(train_precision)
        pos_c, dirs_c = _dev_f32(pos, "pos"), _dev_f32(dirs, "dirs")
        times_c = _dev_f32(times, "times") if use_time else None
        W = _blob(params)
        P, dev = pos_c.shape[0], pos_c.device
        lib = L.lib()
        saved = torch.empty(lib.stnerf_train_saved_floats(SPACENET, int(use_time), P), dtype=torch.float32, device=dev)
        rgb = torch.empty((P, 3), dtype=torch.float32, device=dev)
        sigma = torch.empty((P, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.stnerf_spacenet_train_forward_prec(L.ptr(W), int(use_time), L.ptr(pos_c), L.ptr(dirs_c), L.ptr(times_c),
                                                           P, L.ptr(rgb), L.ptr(sigma), L.ptr(saved), prec, L.stream_ptr()),
                    "stnerf_spacenet_train_forward_prec")
        ctx.save_for_backward(W, saved, *params)
        ctx.use_time, ctx.P, ctx.prec = bool(use_time), P, prec
        return rgb, sigma

    @staticmethod
    def backward(ctx, d_rgb, d_sigma):
        W, saved, *params = ctx.saved_tensors
        P, dev = ctx.P, W.device
        d_rgb = torch.zeros((P, 3), device=dev) if d_rgb is None else d_rgb.to(torch.float32).contiguous()
        d_sigma = torch.zeros((P, 1), device=dev) if d_sigma is None else d_sigma.to(torch.float32).contiguous()
        dW = torch.empty_like(W)
        d_pos = torch.empty((P, 3), dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        scratch = _scratch(SPACENET, ctx.use_time, P, dev, ctx.prec)
        with torch.cuda.device(dev):
            L.check(L.lib().stnerf_spacenet_backward_prec(L.ptr(W), int(ctx.use_time), P, L.ptr(saved), L.ptr(d_rgb),
                                                          L.ptr(d_sigma), L.ptr(dW), L.ptr(d_pos), L.ptr(scratch), scratch.numel(),
                                                          ctx.prec, L.stream_ptr()),
                    "stnerf_spacenet_backward_prec")
        return (d_pos, None, None, None, None, *_split_grad(dW, params))


class MotionNetFunction(torch.autograd.Function):
    """(xyzt (P,4), lerp_mode, train_precision, *parameters) -> flow (P,3).  lerp_mode -1 decides like the reference
    (motion_net.py:53)."""

    @staticmethod
    def forward(ctx, xyzt, lerp_mode, train_precision, *params):
        prec = L.train_precision_code(train_precision)
        x = _dev_f32(xyzt, "xyzt")
        W = _blob(params)
        P, dev = x.shape[0], x.device
        lib = L.lib()
        saved = torch.empty(lib.stnerf_train_saved_floats(MOTIONNET, 0, P), dtype=torch.float32, device=dev)
        flow = torch.empty((P, 3), dtype=torch.float32, device=dev)
        scratch = _scratch(MOTIONNET, False, P, dev, prec)
        with torch.cuda.device(dev):
            L.check(lib.stnerf_motionnet_train_forward_prec(L.ptr(W), L.ptr(x), P, int(lerp_mode), L.ptr(flow), L.ptr(saved),
                                                            L.ptr(scratch), scratch.numel(), prec, L.stream_ptr()),
                    "stnerf_motionnet_train_forward_prec")
        ctx.save_for_backward(W, saved, *params)
        ctx.P, ctx.prec = P, prec
        return flow

    @staticmethod
    def backward(ctx, d_flow):
        W, saved, *params = ctx.saved_tensors
        P, dev = ctx.P, W.device
        d_flow = d_flow.to(torch.float32).contiguous()
        dW = torch.empty_like(W)
        scratch = _scratch(MOTIONNET, False, P, dev, ctx.prec)
        with torch.cuda.device(dev):
            L.check(L.lib().stnerf_motionnet_backward_prec(L.ptr(W), P, L.ptr(saved), L.ptr(d_flow), L.ptr(dW), L.ptr(scratch),
                                                           scratch.numel(), ctx.prec, L.stream_ptr()),
                    "stnerf_motionnet_backward_prec")
        return (None, None, None, *_split_grad(dW, params))


def _params(module, names):
    out = []
    for n in names:
        lin = module.get_submodule(n)
        out += [lin.weight, lin.bias]
    return out


class SpaceNet(nn.Module):
    """modeling/spacenet.py:17-160 on the native training kernels."""

    def __init__(self, c_pos=3, include_input=True, use_dir=True, use_time=False, deep_rgb=False, train_precision="fp32"):
        super().__init__()
        L.train_precision_code(train_precision)
        self.train_precision = train_precision
        if deep_rgb:
            raise NotImplementedError("deep_rgb is not used by any shipped checkpoint and has no native kernel")
        if not use_dir or not include_input or c_pos != 3:
            raise NotImplementedError("the native SpaceNet implements c_pos=3, include_input=True, use_dir=True "
                                      "(both shipped configs)")
        self.c_pos, self.use_dir, self.use_time = c_pos, use_dir, bool(use_time)
        self.pos_dim, self.dir_dim, self.time_dim = 63, 27, 21 if use_time else 0
        bb, head = 256, 128
        self.stage1 = nn.Sequential(nn.Linear(self.pos_dim, bb), nn.ReLU(inplace=True), nn.Linear(bb, bb), nn.ReLU(inplace=True),
                                    nn.Linear(bb, bb), nn.ReLU(inplace=True), nn.Linear(bb, bb), nn.ReLU(inplace=True))
        self.stage2 = nn.Sequential(nn.Linear(bb + self.pos_dim, bb), nn.ReLU(inplace=True), nn.Linear(bb, bb),
                                    nn.ReLU(inplace=True), nn.Linear(bb, bb), nn.ReLU(inplace=True))
        self.density_net = nn.Sequential(nn.Linear(bb, 1))
        self.rgb_net = nn.Sequential(nn.ReLU(inplace=True), nn.Linear(bb + self.dir_dim + self.time_dim, head),
                                     nn.ReLU(inplace=True), nn.Linear(head, 3))

    def forward(self, pos, rays, times=None, maxs=None, mins=None):
        """pos (N,3) or (N,L,3) ("bins mode"), rays (N,>=6), times (N,1) -> rgb (N[,L],3), density (N[,L],1) (:101-160)."""
        if rays is None:
            raise NotImplementedError("the native SpaceNet needs the rays' directions (use_dir=True)")
        dirs = rays[..., 3:6]
        bins = pos.dim() > 2
        if bins:
            n_bins = pos.size(1)
            pos = pos.reshape(-1, self.c_pos)
            dirs = dirs.unsqueeze(1).repeat(1, n_bins, 1).reshape(-1, 3)
            if self.use_time:
                times = times.unsqueeze(1).repeat(1, n_bins, 1).reshape(-1, 1)
        if maxs is not None:
            pos = ((pos - mins) / (maxs - mins) - 0.5) * 2
        if self.use_time and times is None:
            raise ValueError("this SpaceNet consumes PE(time): times is required")
        rgb, density = SpaceNetFunction.apply(pos, dirs, times if self.use_time else None, self.use_time, self.train_precision,
                                              *_params(self, SPACENET_KEYS))
        if bins:
            rgb, density = rgb.reshape(-1, n_bins, 3), density.reshape(-1, n_bins, 1)
        return rgb, density


class MotionNet(nn.Module):
    """modeling/motion_net.py:6-71 on the native training kernels (the configuration LayeredRFRender builds, :90)."""

    def __init__(self, c_input=5, include_input=True, input_time=False, train_precision="fp32"):
        super().__init__()
        L.train_precision_code(train_precision)
        self.train_precision = train_precision
        if c_input != 4 or not input_time or not include_input:
            raise NotImplementedError("the native MotionNet implements c_input=4, include_input=True, input_time=True "
                                      "(the one LayeredRFRender builds)")
        self.c_input, self.input_time = c_input, input_time
        self.pos_dim = 84
        bb, head = 128, 128
        self.motion_net = nn.Sequential(nn.Linear(self.pos_dim, head), nn.ReLU(inplace=False), nn.Linear(head, bb),
                                        nn.ReLU(inplace=True), nn.Linear(bb, bb), nn.ReLU(inplace=True), nn.Linear(bb, bb),
                                        nn.ReLU(inplace=True), nn.Linear(bb, head), nn.ReLU(inplace=True), nn.Linear(head, 3))

    def forward(self, input_0, lerp_mode: int = -1):
        """input_0 (N,4) or (N,L,4) = (x, y, z, t) -> flow (N[,L],3).  lerp_mode -1: lerp the encoding between floor(t) and
        floor(t) + 1 iff any t of the batch is fractional, like the reference (:53); 0 / 1 force it."""
        bins = input_0.dim() > 2
        if bins:
            n_bins = input_0.size(1)
            input_0 = input_0.reshape(-1, self.c_input)
        flow = MotionNetFunction.apply(input_0, lerp_mode, self.train_precision, *_params(self, MOTIONNET_KEYS))
        return flow.reshape(-1, n_bins, 3) if bins else flow


def from_layered(model, train_precision="fp32") -> nn.ModuleDict:
    """The networks of a LayeredRFRender as trainable modules holding its weights, keyed like its state_dict
    (`spacenets.i.*`, `spacenets_fine.i.*`, `bkgd_spacenet.*`, `bkgd_spacenet_fine.*`, `time_deform_nets.i.*`), so that
    `model.load_state_dict(from_layered(model).state_dict())` writes fine-tuned weights back.  Parameters are on the CPU;
    move the result with `.cuda()`.  Every network trains in `train_precision`."""
    n = int(model.layer_num)
    tp = train_precision
    nets = nn.ModuleDict({
        "spacenets": nn.ModuleList([SpaceNet(use_time=model.use_space_time, train_precision=tp) for _ in range(n)]),
        "spacenets_fine": nn.ModuleList([SpaceNet(use_time=model.use_space_time, train_precision=tp) for _ in range(n)]),
        "bkgd_spacenet": SpaceNet(use_time=model.bkgd_use_space_time, train_precision=tp),
        "bkgd_spacenet_fine": SpaceNet(use_time=model.bkgd_use_space_time, train_precision=tp),
        "time_deform_nets": nn.ModuleList([MotionNet(c_input=4, input_time=True, train_precision=tp) for _ in range(n)]),
    })
    nets.load_state_dict(model.state_dict())
    return nets
