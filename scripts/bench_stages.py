#!/usr/bin/env python
"""Stage-level roofline numbers (HBM-bound kernels): CUDA-event timings over inputs larger than L2, algorithmic bytes
from SURVEY 8(d).  Prints one JSON line."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "st-nerf_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch
from stnerf_b200 import ops
from stnerf_b200 import synthetic as O

dev = torch.device("cuda", 0)
peaks = {}
try:
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
except Exception:
    pass
hbm = peaks.get("hbm_gbs", 6650.0)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


res = {}
# a10 VolumeRenderer: 20 B/sample in, 4 B/sample out (weights) + 20 B/ray
for S in (192, 576):
    N = 1 << 20 if S == 192 else 1 << 18
    t = torch.sort(torch.rand(N, S, device=dev) * 6, 1)[0].contiguous()
    rgb = torch.randn(N, S, 3, device=dev)
    sig = torch.randn(N, S, device=dev) * 5
    ms = timeit(lambda: ops.composite(t, rgb, sig, want_weights=True))
    b = N * (S * 24 + 20)
    res["composite_simple_S%d" % S] = {"ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / hbm, "bytes": b}
    ms = timeit(lambda: ops.composite(t, rgb, sig, want_weights=False))
    b = N * (S * 20 + 20)
    res["composite_simple_now_S%d" % S] = {"ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / hbm, "bytes": b}
    del t, rgb, sig
# a3/a4 sampler (one box): reads 24 B/ray (+4*n1 jitter), writes 4*n1 (t) + 12*n1 (xyz) + 9 B
N, n1 = 1 << 21, 64
K, T = O.synthetic_camera(0, 16, 1080, 1920)
rays = ops.generate_rays(K, T, 1080, 1920)[:N].contiguous()
jit = torch.rand(N, n1, device=dev)
ms = timeit(lambda: ops.intersect_sample(rays, (-0.4, -0.4, 0.0), (0.4, 0.4, 1.8), n1, jit, want_xyz=False))
b = N * (24 + 4 * n1 + 4 * n1 + 9)
res["intersect_sample_n64"] = {"ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / hbm, "bytes": b}
# a1 ray generation: 24 B/ray written (+ frame ids)
ms = timeit(lambda: ops.generate_rays(K, T, 1080, 1920, frame_ids=[0, 10, 11]))
b = 1080 * 1920 * 36
res["raygen_1080p"] = {"ms": ms, "GBps": b / ms / 1e6, "frac_hbm": b / ms / 1e6 / hbm, "bytes": b}
print(json.dumps({"hbm_peak_GBps": hbm, "stages": res}))
