#!/usr/bin/env python
"""The SpaceNet tensor-core kernel (mlp_tc_kernel<NET_SPACE>) alone, on explicit points through NativeRenderer.spacenet.

    python scripts/bench_spacenet.py [--log2p 21] [--modes exact exact_cf] [--warmup 3] [--iters 20] [--json FILE]

Per network (background: no time input; performer: PE(time)) and precision mode it prints the time per call (CUDA events
around the call: head_bias_kernel + the MLP kernel), the MLP kernel's own time (torch.profiler, in a separate pass), and
from the kernel's time
  algorithmic TFLOP/s = 2 x MACs of the network per point (every Linear, in x out) x points
  executed TFLOP/s    = 2 x MACs the tensor cores execute per point (the GEMM layers at their padded K: PE(pos) is one
                        64-wide chunk; 3 fp16 MMAs per product in exact / exact_cf, 1 in fast; mixed runs rgb_net.1 once).
Weights are random (seeded), the points uniform in [-1, 1]^3.  The card's name, power limit and SM clock (median of
nvidia-smi samples taken while the timed loop runs) are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "st-nerf_b200"))

from stnerf_b200.native import MOTIONNET_KEYS, SPACENET_KEYS, NativeRenderer  # noqa: E402

PE_POS, PE_DIR, PE_TIME, HID, HEAD = 63, 27, 21, 256, 128


def space_shapes(use_time):
    k_rgb = HID + PE_DIR + (PE_TIME if use_time else 0)
    ins = [PE_POS, HID, HID, HID, HID + PE_POS, HID, HID, HID, k_rgb, HEAD]
    outs = [HID] * 7 + [1, HEAD, 3]
    return list(zip(SPACENET_KEYS, ins, outs))


def algorithmic_macs(use_time):
    return sum(i * o for _, i, o in space_shapes(use_time))


def executed_macs(mode):
    # GEMM layers as the kernel runs them: layer 0 = one 64-wide PE chunk, the skip layer 256 + 64, rgb_net.1 its 256 trunk
    # columns (the dir / time columns are a per-ray fp32 bias)
    trunk = 64 * HID + 3 * HID * HID + (HID + 64) * HID + 2 * HID * HID
    head = HID * HEAD
    return {"exact": 3 * (trunk + head), "exact_cf": 3 * (trunk + head), "mixed": 3 * trunk + head,
            "fast": trunk + head}[mode]


def random_state_dict(gen):
    sd = {}

    def lin(prefix, i, o):
        sd[prefix + ".weight"] = (torch.rand((o, i), generator=gen) * 2 - 1) / i ** 0.5
        sd[prefix + ".bias"] = (torch.rand((o,), generator=gen) * 2 - 1) * 0.1

    for pre, use_time in (("bkgd_spacenet.", False), ("bkgd_spacenet_fine.", False), ("spacenets.0.", True),
                          ("spacenets_fine.0.", True)):
        for name, i, o in space_shapes(use_time):
            lin(pre + name, i, o)
    m_ins = [84] + [HEAD] * 5
    m_outs = [HEAD] * 5 + [3]
    for name, i, o in zip(MOTIONNET_KEYS, m_ins, m_outs):
        lin("time_deform_nets.0." + name, i, o)
    return sd


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


class ClockSampler:
    """SM clock samples (MHz) from nvidia-smi while the timed loop runs."""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            try:
                self.samples.append(float(smi("clocks.sm")[0]))
            except Exception:
                pass
            self._stop.wait(0.1)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        return statistics.median(self.samples) if self.samples else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2p", type=int, default=21, help="points per call = 2^log2p (at least 2^20)")
    ap.add_argument("--modes", nargs="+", default=["exact", "exact_cf"], choices=["exact", "exact_cf", "mixed", "fast"])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    a = ap.parse_args()
    if a.log2p < 20:
        ap.error("--log2p must be at least 20: smaller calls leave SMs idle for part of the launch")
    if not torch.cuda.is_available():
        raise SystemExit("bench_spacenet.py needs a CUDA device")
    dev = torch.device("cuda")
    card, power_limit, max_sm = smi("name,power.limit,clocks.max.sm")
    print("# %s, power limit %s W, max SM clock %s MHz" % (card, power_limit, max_sm))
    gen = torch.Generator().manual_seed(0)
    r = NativeRenderer(2, [False, True], precision="exact")
    r.load_state_dict(random_state_dict(gen))
    P = 1 << a.log2p
    pos = (torch.rand((P, 3), generator=gen) * 2 - 1).to(dev)
    dirs = torch.nn.functional.normalize(torch.randn((P, 3), generator=gen), dim=1).to(dev)
    tm = torch.full((P,), 17.0).to(dev)
    print("%-6s %-9s %9s %10s %10s %10s %10s %9s" % ("net", "mode", "P", "call ms", "kernel ms", "alg TF/s", "exec TF/s",
                                                     "SM MHz"))
    rows = []
    for net, layer, times in (("bkgd", 0, None), ("perf", 1, tm)):
        for mode in a.modes:
            r.set_precision(mode)

            def call():
                return r.spacenet(layer, False, pos, dirs, times)

            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with ClockSampler() as clk:
                ev0.record()
                for _ in range(a.iters):
                    call()
                ev1.record()
                torch.cuda.synchronize()
            call_ms = ev0.elapsed_time(ev1) / a.iters
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    call()
                torch.cuda.synchronize()
            ka = [e for e in prof.key_averages() if "mlp_tc_kernel" in e.key]
            n_launch = sum(e.count for e in ka)
            if n_launch != a.iters:
                raise RuntimeError("expected %d mlp_tc_kernel launches in the trace, found %d" % (a.iters, n_launch))
            kernel_ms = sum(e.device_time_total for e in ka) / n_launch / 1e3
            alg = 2.0 * algorithmic_macs(times is not None) * P / (kernel_ms * 1e-3) / 1e12
            exe = 2.0 * executed_macs(mode) * P / (kernel_ms * 1e-3) / 1e12
            mhz = clk.median()
            print("%-6s %-9s %9d %10.3f %10.3f %10.1f %10.1f %9s" % (net, mode, P, call_ms, kernel_ms, alg, exe,
                                                                    "%.0f" % mhz if mhz else "?"))
            rows.append({"net": net, "mode": mode, "points": P, "call_ms": call_ms, "kernel_ms": kernel_ms,
                         "alg_tflops": alg, "exec_tflops": exe, "sm_mhz_median": mhz})
    res = {"card": card, "power_limit_w": power_limit, "max_sm_mhz": max_sm, "rows": rows}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    r.close()


if __name__ == "__main__":
    main()
