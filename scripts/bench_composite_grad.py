#!/usr/bin/env python
"""Compositing forward + backward (stnerf_b200.volume) against the same step through torch fp32 autograd on the same GPU.

    python scripts/bench_composite_grad.py [--warmup 5] [--iters 20]

Workloads:
  step    one training step's compositing: 3000 rays (SOLVER.BUNCH), 3 layers, S = 64 and 192 samples per layer.  Per pass:
          three per-layer composites (upstream d_color, d_depth, d_acc) and the depth-merged composite of the three layers
          (torch sort + gather, then the composite; upstream d_color).
  large   one composite of 2^20 rays at S = 192, upstream d_color, d_depth, d_acc and d_w.
For each it prints ms per forward + backward for the native path and for torch autograd of the reference formula
(render_layer.py:8-58).  For the backward kernel alone (stnerf_composite_backward, timed by itself) it prints the achieved
bandwidth from the algorithmic bytes: in 20 B/sample (t, rgb, sigma; +4 with d_w) + 20 B/ray (d_color, d_depth, d_acc),
out 16 B/sample (d_rgb, d_sigma), against the H100 SXM data-sheet 3.35 TB/s.  The card's name and power limit are read in the
same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "st-nerf_b200"))

from stnerf_b200 import _lib as L, volume  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def torch_composite(t, rgb, sigma, boarder=1e10):
    n = t.shape[0]
    delta = torch.cat([t[:, 1:] - t[:, :-1], torch.full((n, 1), boarder, device=t.device)], -1)
    alpha = 1.0 - torch.exp(-torch.relu(sigma) * delta)
    trans = torch.cumprod(torch.cat([torch.ones((n, 1), device=t.device), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    return (torch.sigmoid(rgb) * w[..., None]).sum(1), (w * t).sum(1, keepdim=True), w.sum(1, keepdim=True), w


def torch_merged(ts, rgbs, sigmas):
    tm, order = torch.sort(torch.cat(ts, 1), dim=1, stable=True)
    rm = torch.cat(rgbs, 1).gather(1, order[..., None].expand(-1, -1, 3))
    sm = torch.cat(sigmas, 1).gather(1, order)
    return torch_composite(tm, rm, sm)[:3]


def inputs(N, S, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    t = 2.0 + torch.cumsum(torch.rand((N, S), generator=g, device=dev) * 0.05, 1)
    rgb = torch.randn((N, S, 3), generator=g, device=dev).requires_grad_(True)
    sigma = (torch.randn((N, S), generator=g, device=dev) * 5.0).requires_grad_(True)
    return t, rgb, sigma


def time_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
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


def backward_kernel_row(t, rgb, sigma, ups, warmup, iters):
    """ms and achieved bytes/s of stnerf_composite_backward alone on these inputs."""
    N, S = t.shape
    r, s = rgb.detach(), sigma.detach()
    d_rgb, d_sigma = torch.empty_like(r), torch.empty_like(s)
    args = [ups.get(k) for k in ("color", "depth", "acc", "w")]

    def run():
        L.check(L.lib().stnerf_composite_backward(L.ptr(t), L.ptr(r), L.ptr(s), N, S, 1e10, *(L.ptr(x) for x in args),
                                                  L.ptr(d_rgb), L.ptr(d_sigma), L.stream_ptr()))
    ms = time_ms(run, warmup, iters)
    nbytes = N * S * (20 + (4 if "w" in ups else 0)) + 20 * N + 16 * N * S
    return ms, nbytes / (ms * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda")
    card, watts = torch.cuda.get_device_name(dev), power_limit()
    print("# %s, power limit %s W; compositing forward + backward" % (card, "%.0f" % watts if watts else "unknown"))
    rows = []
    for S in (64, 192):
        N = 3000
        lay = [inputs(N, S, 10 + i, dev) for i in range(3)]
        g = torch.Generator(device=dev).manual_seed(3)
        up = {"color": torch.randn((N, 3), generator=g, device=dev), "depth": torch.randn((N, 1), generator=g, device=dev),
              "acc": torch.randn((N, 1), generator=g, device=dev)}

        def step(comp, merged):
            def run():
                outs, grads = [], []
                for t, r, s in lay:
                    c, d, ac, _ = comp(t, r, s)
                    outs += [c, d, ac]
                    grads += [up["color"], up["depth"], up["acc"]]
                c = merged([x[0] for x in lay], [x[1] for x in lay], [x[2] for x in lay])[0]
                torch.autograd.backward(outs + [c], grads + [up["color"]])
            return run
        ms_nat = time_ms(step(volume.composite, volume.composite_merged), a.warmup, a.iters)
        ms_tor = time_ms(step(torch_composite, torch_merged), a.warmup, a.iters)
        tm, order = torch.sort(torch.cat([x[0] for x in lay], 1), dim=1, stable=True)
        rm = torch.cat([x[1] for x in lay], 1).detach().gather(1, order[..., None].expand(-1, -1, 3)).requires_grad_(True)
        sm = torch.cat([x[2] for x in lay], 1).detach().gather(1, order).requires_grad_(True)

        def merged_only():
            torch.autograd.backward(volume.composite(tm, rm, sm)[0], up["color"])

        def merged_full():
            torch.autograd.backward(volume.composite_merged([x[0] for x in lay], [x[1] for x in lay], [x[2] for x in lay])[0],
                                    up["color"])
        ms_mc = time_ms(merged_only, a.warmup, a.iters)
        ms_mf = time_ms(merged_full, a.warmup, a.iters)
        kb_ms, kb_bw = backward_kernel_row(*lay[0], up, a.warmup, a.iters)
        row = {"workload": "step", "rays": N, "layers": 3, "S": S, "native_ms": ms_nat, "torch_ms": ms_tor,
               "merged_composite_ms": ms_mc, "merged_with_sort_gather_ms": ms_mf,
               "backward_kernel_ms": kb_ms, "backward_kernel_GBps": kb_bw / 1e9, "backward_hbm_share": kb_bw / HBM_BYTES_PER_S}
        rows.append(row)
        print("step  S=%3d  native %.3f ms  torch %.3f ms  | merged: composite %.3f ms, with sort+gather %.3f ms | "
              "backward kernel (per layer) %.4f ms, %.0f GB/s" % (S, ms_nat, ms_tor, ms_mc, ms_mf, kb_ms, kb_bw / 1e9))
        del lay
    N, S = 1 << 20, 192
    t, rgb, sigma = inputs(N, S, 20, dev)
    g = torch.Generator(device=dev).manual_seed(4)
    up = {"color": torch.randn((N, 3), generator=g, device=dev), "depth": torch.randn((N, 1), generator=g, device=dev),
          "acc": torch.randn((N, 1), generator=g, device=dev), "w": torch.randn((N, S), generator=g, device=dev)}

    def big(comp):
        def run():
            outs = comp(t, rgb, sigma)
            torch.autograd.backward(list(outs), [up["color"], up["depth"], up["acc"], up["w"]])
        return run
    ms_nat = time_ms(big(volume.composite), a.warmup, a.iters)
    kb_ms, kb_bw = backward_kernel_row(t, rgb, sigma, up, a.warmup, a.iters)
    rgb.grad = sigma.grad = None
    torch.cuda.empty_cache()
    ms_tor = time_ms(big(torch_composite), a.warmup, a.iters)
    rows.append({"workload": "large", "rays": N, "S": S, "native_ms": ms_nat, "torch_ms": ms_tor, "backward_kernel_ms": kb_ms,
                 "backward_kernel_GBps": kb_bw / 1e9, "backward_hbm_share": kb_bw / HBM_BYTES_PER_S})
    print("large N=2^20 S=%d  native %.3f ms  torch %.3f ms | backward kernel %.3f ms, %.0f GB/s (%.0f%% of 3.35 TB/s)"
          % (S, ms_nat, ms_tor, kb_ms, kb_bw / 1e9, 100 * kb_bw / HBM_BYTES_PER_S))
    print(json.dumps({"card": card, "power_limit_w": watts, "rows": rows}))


if __name__ == "__main__":
    main()
