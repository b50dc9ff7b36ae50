#!/usr/bin/env python
"""The training-data pipeline (stnerf_b200.train_data) at user scale.

    python scripts/bench_train_data.py [--cams 16] [--frames 4] [--width 1920] [--height 1080] [--performers 2]
                                       [--bkgd-rate 0.05] [--batch 2000] [--batches 1000] [--steps 40]

Writes a seeded capture in the reference's layout to a temporary directory (images with smooth content and noise, each
performer a labelled ellipse, box point clouds), builds the ray pool and reports, as one JSON line:
  * pool build time, split into host decode, host randperm and device selection (selection includes the uploads);
  * rays in the pool and bytes per ray;
  * time per batch of the loader (CUDA events over `--batches` batches of one epoch order; host-bound at this size), and
    the batch kernel's own device time from a torch.profiler run of the same batches;
  * the same batches built the reference's way: a restatement of Ray_Dataset.__getitem__ (ray_dataset.py:72-83, a walk over
    the (layer, frame) datasets per item) over host tensors holding each item's 7+3+1+1+24+2 floats, plus default collate;
  * a tf32x3 fine-stage training step (2 performers, 90 + 30 samples, the trainer's MSE loss) fed by the loader, against the
    same steps on the same batches built beforehand (the best of three alternated rounds each);
  * the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "st-nerf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from stnerf_b200 import train_data as TD  # noqa: E402
from stnerf_b200.synthetic import corners_from_minmax, synthetic_camera, synthetic_state_dict  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def write_ply(path, pts):
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                 "property float z\nend_header\n" % len(pts)).encode())
        f.write(np.asarray(pts, dtype="<f4").tobytes())


def write_capture(root, a):
    from PIL import Image
    rng = np.random.RandomState(0)
    H, W = a.height, a.width
    os.makedirs(os.path.join(root, "pose"))
    os.makedirs(os.path.join(root, "background"))
    Ks, Ts = [], []
    for v in range(a.cams):
        K, T = synthetic_camera(v, a.cams, H, W)
        Ks.append(K.double().reshape(-1).numpy()); Ts.append(T.double()[:3].reshape(-1).numpy())
    np.savetxt(os.path.join(root, "pose", "K.txt"), np.stack(Ks), fmt="%.10g")
    np.savetxt(os.path.join(root, "pose", "RT_c2w.txt"), np.stack(Ts), fmt="%.10g")
    write_ply(os.path.join(root, "background", "0.ply"), corners_from_minmax((-6, -6, -1), (6, 6, 4)).numpy())
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([(xx * 255 // max(W - 1, 1)), (yy * 255 // max(H - 1, 1)), ((xx + yy) % 256)], -1).astype(np.int16)
    for f in range(1, a.frames + 1):
        for d in ("images", "labels", "pointclouds"):
            os.makedirs(os.path.join(root, "frame%d" % f, d))
        for i in range(a.performers):
            cx = 0.0 if a.performers == 1 else -2.0 + 4.0 * i / (a.performers - 1)
            write_ply(os.path.join(root, "frame%d" % f, "pointclouds", "%d.ply" % (i + 1)),
                      corners_from_minmax((cx - 0.4, -0.4, 0.0), (cx + 0.4, 0.4, 1.8)).numpy())
        for v in range(a.cams):
            img = np.clip(base + rng.randint(-8, 9, size=base.shape), 0, 255).astype(np.uint8)
            lab = np.zeros((H, W), np.uint8)
            for i in range(a.performers):                          # an ellipse per performer, ~3% of the image each
                cx, cy = W * (i + 1) / (a.performers + 1) + 10 * f, H * 0.55
                lab[((xx - cx) / (0.07 * W)) ** 2 + ((yy - cy) / (0.3 * H)) ** 2 <= 1] = i + 1
            Image.fromarray(img).save(os.path.join(root, "frame%d" % f, "images", "%03d.png" % v), compress_level=1)
            np.save(os.path.join(root, "frame%d" % f, "labels", "%03d.npy" % v), lab)


def make_cfg(root, a):
    import types
    D = types.SimpleNamespace(TRAIN=root, FRAME_NUM=a.frames, LAYER_NUM=a.performers, FRAME_OFFSET=0,
                              BKGD_SAMPLE_RATE=a.bkgd_rate, FIXED_LAYER=[], USE_LABEL=True, CAMERA_STEPSIZE=1, FILE_OFFSET=0,
                              CAMERA_NUM=0, VIEW_MASK=None, SCALE=1.0, FIXED_NEAR=0.5, FIXED_FAR=20.0, SHIFT=0, MAXRATION=0.0,
                              ROTATION=0.0)
    M = types.SimpleNamespace(POSE_REFINEMENT=False, USE_DEFORM_VIEW=False, USE_DEFORM_TIME=True, USE_SPACE_TIME=True)
    I = types.SimpleNamespace(SIZE_TRAIN=[a.width, a.height], SIZE_LAYER=[a.width, a.height])
    return types.SimpleNamespace(DATASETS=D, MODEL=M, INPUT=I, SOLVER=types.SimpleNamespace(IMS_PER_BATCH=a.batch))


def reference_way(ds, a, n_batches):
    """Ray_Dataset.__getitem__ + default collate over host tensors, restated: per (layer, frame) segment the stored
    items (rays 7, rgbs 3, labels 1, bbox labels 1, box 8x3, near/far 2), an index walk over the segments per item."""
    from torch.utils.data import default_collate
    segs, o = [], 0
    host = [t.cpu() for t in ds.items(torch.arange(len(ds), device=ds.device))]
    for l, slot, n in ds.segments:
        segs.append([h[o:o + n] for h in host])
        o += n

    def getitem(index):
        temp = 0
        for s in segs:
            n = s[0].shape[0]
            if temp + n > index:
                i = index - temp
                return s[0][i, :], s[1][i, :], s[2][i, :], s[3][i, :], s[4][i], s[5][i, :]
            temp += n

    perm = torch.randperm(len(ds))
    t0 = time.perf_counter()
    for b in range(n_batches):
        idx = perm[b * a.batch:(b + 1) * a.batch].tolist()
        default_collate([getitem(i) for i in idx])
    return (time.perf_counter() - t0) / n_batches * 1e3


def train_step_ms(ds, a):
    import modeling
    from stnerf_b200.config import make_cfg as model_cfg
    from stnerf_b200.synthetic import synthetic_boxes
    cfg = model_cfg(a.performers, 90, 30, True, "fp32")
    cfg.MODEL.B200_TRAINABLE = True
    cfg.MODEL.B200_TRAIN_PRECISION = "tf32x3"
    model = modeling.build_layered_model(cfg, 0)
    model.load_state_dict(synthetic_state_dict(a.performers, True, seed=0))
    bkgd, frames = synthetic_boxes(a.performers, a.frames + 2)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model = model.cuda()
    opt = torch.optim.Adam(model.parameters(), lr=4e-4)

    def step(batch):
        rays, rgbs, labels, bbl, bboxes, nf = batch
        opt.zero_grad()
        s2, s1, _, _, _ = model(rays, bbl, bboxes, False, near_far=nf)
        loss = torch.nn.functional.mse_loss(s1[0], rgbs) + torch.nn.functional.mse_loss(s2[0], rgbs)
        loss.backward()
        opt.step()

    # the same batches twice: built by the loader inside the timed loop, or built beforehand and only read
    n_steps = 3 + a.steps

    def loader_batches():
        while True:
            for b in TD.RayLoader(ds, a.batch, seed=9):
                yield b

    src = loader_batches()
    prebuilt = [[t.clone() for t in next(src)] for _ in range(n_steps)]
    res = {}
    for rep in range(3):                                     # alternate the two, three times
        for name in ("loader", "prebuilt"):
            src = loader_batches()
            batches = (next(src) for _ in range(n_steps)) if name == "loader" else iter(prebuilt)
            for _ in range(3):
                step(next(batches))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                step(next(batches))
            torch.cuda.synchronize()
            res.setdefault(name, []).append((time.perf_counter() - t0) / a.steps * 1e3)
    return {k: min(v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--performers", type=int, default=2)
    ap.add_argument("--bkgd-rate", type=float, default=0.05)
    ap.add_argument("--batch", type=int, default=2000)
    ap.add_argument("--batches", type=int, default=1000)
    ap.add_argument("--ref-batches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=40)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_data.py measures on a CUDA device; none is visible")
    out = dict(card=torch.cuda.get_device_name(), power_limit_w=power_limit(), cams=a.cams, frames=a.frames,
               width=a.width, height=a.height, performers=a.performers, bkgd_rate=a.bkgd_rate, batch=a.batch)
    with tempfile.TemporaryDirectory(prefix="stnerf_train_data_") as root:
        t0 = time.perf_counter()
        write_capture(root, a)
        out["capture_write_s"] = round(time.perf_counter() - t0, 2)
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loader, ds = TD.make_ray_data_loader(make_cfg(root, a), seed=0)
        torch.cuda.synchronize()
        out["pool_build_s"] = round(time.perf_counter() - t0, 3)
        out.update({"pool_" + k: round(v, 3) for k, v in ds.timing.items()})
        out["pool_rays"] = len(ds)
        out["bytes_per_ray"] = ds.pool_bytes / max(len(ds), 1)
        perm = loader.epoch_order()
        n_b = min(a.batches, len(loader) - 1)
        for b in range(10):
            ds.items(perm[b * a.batch:(b + 1) * a.batch])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for b in range(n_b):
            ds.items(perm[b * a.batch:(b + 1) * a.batch])
        e1.record()
        torch.cuda.synchronize()
        out["batches_timed"] = n_b
        out["batch_loader_us"] = round(e0.elapsed_time(e1) / n_b * 1e3, 2)
        # the kernel alone: the window above is bound by the host's per-batch Python; a profiler run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for b in range(n_b):
                ds.items(perm[b * a.batch:(b + 1) * a.batch])
            torch.cuda.synchronize()
        ks = [e for e in prof.key_averages() if "batch_kernel" in e.key]
        dev_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ks)
        out["batch_kernel_us"] = round(dev_us / n_b, 2)
        out["batch_kernel_launches"] = int(sum(e.count for e in ks))
        out["batch_reference_way_ms"] = round(reference_way(ds, a, a.ref_batches), 2)
        steps = train_step_ms(ds, a)
        out["train_step_loader_ms"] = round(steps["loader"], 2)
        out["train_step_prebuilt_ms"] = round(steps["prebuilt"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
