"""Cost of the rotation edit on the bench.py workload: rays/s with no layer, one performer and every performer rotated, and
the device time of the rotate kernel.

    python scripts/bench_rotation.py [--steps 8] [--warmup 2] [--rounds 3] [--json out.json]

The workload, scene, cameras and weights are bench.py's (taekwondo 2-layer, 1080p, 64 + 128 samples, stnerf_render_views with
the coarse images, one view per step).  The variants alternate round by round so that their spread can be compared; each
number is CUDA events around `steps` views after `warmup` views.  The rotate kernel's time comes from a separate torch.profiler
run (CUDA activities) of the all-rotated variant: the summed durations of rotate_rays_kernel over the profiled views.  The extra
device memory is the rotated rays' scratch, computed from the shapes.  Prints the card's name and power limit with the numbers."""
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

import bench  # noqa: E402
from stnerf_b200.config import make_cfg  # noqa: E402
from stnerf_b200.dist import ShardedViewRenderer  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="exact")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rotation needs a CUDA device")
    import modeling
    wl = bench.WORKLOADS["taekwondo2"]
    H, W, N1, N2, LAYERS, VIEWS = wl["H"], wl["W"], wl["n1"], wl["n2"], wl["layers"], wl["views"]
    dev = torch.device("cuda", 0)
    sd, data = bench.load_weights(wl)
    bkgd, frames, cams = bench.scene_setup(wl)
    model = modeling.build_layered_model(make_cfg(LAYERS, N1, N2, wl["space_time"], args.precision))
    model.load_state_dict(sd)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    nat = model._ensure_native(dev)
    model.near = wl["near"]
    model.retiming = True
    scene = model._resolve_scene(torch.tensor(wl["frame_ids"]), wl["thr"][0], wl["thr"][1])
    svr = ShardedViewRenderer(nat, H, W, N1, N2, 0, 1)
    quarter = [0.0, 0.0, np.pi / 2]                                      # a quarter turn about z, about each box's centre
    variants = {"none": None, "one": [None, quarter] + [None] * (LAYERS - 1), "all": [None] + [quarter] * LAYERS}

    def step(i):
        v = nat.make_view(cams[i % VIEWS][0], cams[i % VIEWS][1], wl["frame_ids"], scene, i + 1)
        return svr.render([v], with_coarse=True)

    def run(name, steps, warmup):
        model.rotation = variants[name]
        model._upload_rotation(nat)
        for i in range(warmup):
            step(i)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(steps):
            step(warmup + i)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    rates = {k: [] for k in variants}
    for _ in range(args.rounds):
        for name in variants:
            ms = run(name, args.steps, args.warmup)
            rates[name].append(H * W * args.steps / (ms * 1e-3))
    # the rotate kernel's device time, in a run of its own
    model.rotation = variants["all"]
    model._upload_rotation(nat)
    step(0)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    n_prof = 2
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(n_prof):
            step(i)
        torch.cuda.synchronize()
    rot_us, rot_n = 0.0, 0
    for e in prof.events():
        if "rotate_rays_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
            rot_us += e.device_time
            rot_n += 1
    chunk = int(getattr(model, "chunk_rays", 0)) or 65536
    stride = 6 + LAYERS + 1
    res = {
        "card": card(), "workload": wl["name"], "data": data, "precision": args.precision,
        "rays_per_s": {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v)), "runs": v} for k, v in rates.items()},
        "rotate_kernel": {"views": n_prof, "launches": rot_n, "device_ms_per_view": rot_us / 1e3 / n_prof,
                          "bytes_moved_per_view": 2 * H * W * stride * 4 * LAYERS},
        "extra_device_bytes_per_chunk_per_rotated_layer": chunk * stride * 4, "chunk_rays": chunk,
    }
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
