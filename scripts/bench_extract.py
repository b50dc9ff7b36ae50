"""Times geometry extraction on the device: a performer's field on a grid (stnerf_layer_grid) and marching cubes on it.

    python scripts/bench_extract.py [--res 256] [--reps 5] [--json out.json]

Synthetic weights of one performer with a time input (the shipped configuration) on the synthetic scene boxes; frame 10.5
(fractional: the MotionNet encoding is lerped).  Reports per precision the grid's points/s and algorithmic TFLOP/s -- 2 x the
multiply-adds of every Linear of MotionNet + SpaceNet per point (DESIGN 6) -- and, on that grid, marching cubes' cells/s
(count + fill, which includes its one device->host copy of the counts).  Times are CUDA events around the calls after a warm-up
call, median of --reps.  Prints the card's name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "st-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from stnerf_b200 import extract as X  # noqa: E402
from stnerf_b200 import native as N  # noqa: E402
from stnerf_b200.config import make_cfg  # noqa: E402
from stnerf_b200.model import fresh_state_dict  # noqa: E402

SPACE_MACS = 63 * 256 + 3 * 256 * 256 + 319 * 256 + 2 * 256 * 256 + 256 + (256 + 27 + 21) * 128 + 128 * 3
MOTION_MACS = 84 * 128 + 4 * 128 * 128 + 128 * 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def boxes():
    lo, hi = np.array([-0.4, -0.4, 0.0]), np.array([0.4, 0.4, 1.8])
    corners = lambda a, b: torch.tensor([[a[0], a[1], a[2]], [b[0], a[1], a[2]], [b[0], b[1], a[2]], [a[0], b[1], a[2]],
                                         [a[0], a[1], b[2]], [b[0], a[1], b[2]], [b[0], b[1], b[2]], [a[0], b[1], b[2]]],
                                        dtype=torch.float32)
    bkgd = corners((-6, -6, -1), (6, 6, 4))
    frames = corners(lo, hi)[None, None].expand(101, 1, 8, 3).clone()
    return bkgd, frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_extract needs a CUDA device (H100); there is no CPU fallback")
    import modeling
    torch.manual_seed(0)
    sd = fresh_state_dict(1, True)
    bkgd, frames = boxes()
    frame, R = 10.5, args.res
    out = {"card": card(), "res": R, "frame": frame}
    print("card: %s" % out["card"])
    sigma = None
    for prec in ("exact", "fp32"):
        model = modeling.build_layered_model(make_cfg(1, 64, 128, True, prec), 0)
        model.load_state_dict(sd)
        model.set_bkgd_bbox(bkgd)
        model.set_bboxes(frames)
        model.cuda()
        nat, scene = X._scene_at(model, frame)
        lo, hi = X.layer_box(model, 1, frame)
        origin, step, dims = X._grid(lo, hi, R)
        buf = torch.empty(dims, dtype=torch.float32, device="cuda")
        ms = timed(lambda: nat.layer_grid(1, True, frame, origin, step, dims, out=buf), args.reps)
        pts = float(R ** 3)
        row = {"ms": ms, "points_per_s": pts / ms * 1e3, "alg_tflops": 2.0 * (SPACE_MACS + MOTION_MACS) * pts / ms * 1e-9}
        out["grid_" + prec] = row
        print("layer_grid %-6s %d^3: %8.2f ms  %7.3f Gpoints/s  %6.1f TFLOP/s (algorithmic)" %
              (prec, R, ms, row["points_per_s"] * 1e-9, row["alg_tflops"]))
        sigma = buf.clone()
        geo = (origin, step)
    level = float(sigma.float().quantile(0.75)) if sigma.numel() <= 1 << 24 else float(sigma.reshape(-1)[::7].quantile(0.75))
    ms = timed(lambda: N.marching_cubes(sigma, geo[0], geo[1], level), args.reps)
    v, f = N.marching_cubes(sigma, geo[0], geo[1], level)
    cells = float((R - 1) ** 3)
    out["mc"] = {"ms": ms, "cells_per_s": cells / ms * 1e3, "level": level, "verts": int(v.shape[0]), "faces": int(f.shape[0])}
    print("marching cubes %d^3: %8.2f ms  %7.3f Gcells/s  (%d verts, %d faces at level %.4g)" %
          (R, ms, out["mc"]["cells_per_s"] * 1e-9, v.shape[0], f.shape[0], level))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
