#!/usr/bin/env python
"""Forward + backward of one SpaceNet and one MotionNet on the native training kernels (stnerf_b200.nets), against the
same step through torch fp32 autograd (cuBLAS, TF32 off) on the same GPU, and -- for context only -- torch with TF32 on
(arm "torch_1xtf32": one tf32 product per term, less accurate than the native tf32x3 precision).

    python scripts/bench_train_nets.py [--log2p 16 17 18 19 20] [--warmup 3] [--iters 10] [--train-precision fp32|tf32x3]

Per network and batch size P it prints ms per step, points/s and algorithmic FLOP/s, counted from the shapes:
  MACs per point = forward (every Linear: in x out)
                 + delta (every Linear whose input needs a gradient: SpaceNet's trunk down to PE(pos) because d_pos is
                   requested, rgb_net.1 only into its 256 trunk columns; MotionNet down to motion_net.2)
                 + weight gradient (every Linear: in x out)
  FLOP = 2 x MACs x P.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "st-nerf_b200"))

from stnerf_b200 import nets  # noqa: E402

SPACE_LAYERS = [(63, 256), (256, 256), (256, 256), (256, 256), (319, 256), (256, 256), (256, 256), (256, 1), (304, 128),
                (128, 3)]
MOTION_LAYERS = [(84, 128), (128, 128), (128, 128), (128, 128), (128, 128), (128, 3)]


def macs(kind):
    layers = SPACE_LAYERS if kind == "space" else MOTION_LAYERS
    fwd = sum(i * o for i, o in layers)
    if kind == "space":
        delta = fwd - (304 - 256) * 128
    else:
        delta = fwd - 84 * 128
    return fwd + delta + fwd


def pe(x, n):
    return torch.cat([x] + [f(x * 2.0 ** k) for k in range(n) for f in (torch.sin, torch.cos)], -1)


def torch_space(m, pos, dirs, tm):
    x = p = pe(pos, 10)
    for i in (0, 2, 4, 6):
        x = F.relu(m.stage1[i](x))
    x = torch.cat([x, p], 1)
    for i in (0, 2, 4):
        x = F.relu(m.stage2[i](x))
    sig = m.density_net[0](x)
    h = F.relu(torch.cat([x, pe(dirs, 4), pe(tm, 10)], 1))
    return m.rgb_net[3](F.relu(m.rgb_net[1](h))), sig


def torch_motion(m, xyzt):
    x = pe(xyzt, 10)
    for i in (0, 2, 4, 6, 8):
        x = F.relu(m.motion_net[i](x))
    return m.motion_net[10](x)


def time_ms(step, warmup, iters):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2p", type=int, nargs="+", default=[16, 17, 18, 19, 20])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--train-precision", choices=["fp32", "tf32x3"], default="fp32", help="precision of the native arm")
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    card, watts = torch.cuda.get_device_name(dev), power_limit()
    print("# %s, power limit %s W; forward + backward per step, native arm in %s" % (card, "%.0f" % watts if watts else "unknown",
                                                                                  a.train_precision))
    print("%-6s %8s %-12s %10s %14s %10s" % ("net", "P", "arm", "ms/step", "points/s", "TFLOP/s"))
    torch.manual_seed(0)
    sn = nets.SpaceNet(use_time=True, train_precision=a.train_precision).to(dev)
    mn = nets.MotionNet(c_input=4, input_time=True, train_precision=a.train_precision).to(dev)
    rows = []
    for lp in a.log2p:
        P = 1 << lp
        pos = torch.randn((P, 3), device=dev).requires_grad_(True)
        rays = torch.cat([pos.detach(), F.normalize(torch.randn((P, 3), device=dev), dim=1)], 1)
        tm = torch.full((P, 1), 17.0, device=dev)
        xyzt = torch.cat([pos.detach(), tm + 0.5], 1)
        r_rgb, r_sig, r_flow = (torch.randn((P, 3), device=dev), torch.randn((P, 1), device=dev),
                                torch.randn((P, 3), device=dev))

        def space_native():
            rgb, sig = sn(pos, rays, tm)
            ((rgb * r_rgb).sum() + (sig * r_sig).sum()).backward()

        def space_torch():
            rgb, sig = torch_space(sn, pos, rays[:, 3:6], tm)
            ((rgb * r_rgb).sum() + (sig * r_sig).sum()).backward()

        def motion_native():
            (mn(xyzt) * r_flow).sum().backward()

        def motion_torch():
            (torch_motion(mn, xyzt) * r_flow).sum().backward()

        for net, arms in (("space", (("native", space_native), ("torch", space_torch), ("torch_1xtf32", space_torch))),
                          ("motion", (("native", motion_native), ("torch", motion_torch), ("torch_1xtf32", motion_torch)))):
            for arm, step in arms:
                torch.backends.cuda.matmul.allow_tf32 = arm == "torch_1xtf32"
                ms = time_ms(step, a.warmup, a.iters)
                tflops = 2.0 * macs(net) * P / (ms * 1e-3) / 1e12
                print("%-6s %8d %-12s %10.3f %14.4g %10.2f" % (net, P, arm, ms, P / (ms * 1e-3), tflops))
                rows.append({"net": net, "P": P, "arm": arm, "ms": ms, "points_per_s": P / (ms * 1e-3), "tflops": tflops})
        del pos, rays, tm, xyzt, r_rgb, r_sig, r_flow
        sn.zero_grad(set_to_none=True)
        mn.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps({"card": card, "power_limit_w": watts, "train_precision": a.train_precision, "rows": rows}))


if __name__ == "__main__":
    main()
