#!/usr/bin/env python
"""The edit sessions of the reference's demo/taekwondo_demo.py (origin / shift / scale) on the native H100 path.

The dataset (images, point clouds, camera files) is not shipped with the reference, so the scene geometry and the 16
ground-truth cameras are the synthetic rig of SURVEY 8(d); everything else follows the demo line by line:

    demo/taekwondo_demo.py:39-52   retime_by_key_frames(1, ...), retime_by_key_frames(2, ...), set_smooth_path_poses(101),
                                    render_path(density_threshold=0)
    :55-62  shift=[[0,0,0],[0,2,0],[0,-2,0]]          :65-72  scale=[1,0.75,1.5]

    python examples/taekwondo_demo_b200.py --size 480x270 --steps 21 --out /tmp/tkd        # frames as PNG (needs PIL)
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "st-nerf_b200"))      # ahead of a reference checkout: native modeling/utils/layers/engine

import torch                                                  # noqa: E402

import modeling                                               # noqa: E402  (the reference's import name)
from stnerf_b200 import CameraPath, PoseRenderer, checkpoint_io, synthetic as O   # noqa: E402
from stnerf_b200.config import make_cfg                       # noqa: E402  cfg stub with the fields the model reads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="480x270")
    ap.add_argument("--steps", type=int, default=21)
    ap.add_argument("--out", default="")
    ap.add_argument("--precision", default="exact")
    a = ap.parse_args()
    W, H = [int(v) for v in a.size.split("x")]
    key_frames_layer_1, key_frames_layer_2, key_frames = [21, 49, 74, 87], [13, 42, 80, 90], [20, 50, 74, 85]
    density_threshold = 0

    cams = [O.synthetic_camera(v, 16, H, W) for v in range(16)]
    gt_poses = torch.stack([T for _, T in cams]).numpy()
    gt_Ks = [K.numpy() for K, _ in cams]
    bkgd, frames = O.synthetic_boxes(2)
    ckpt = checkpoint_io.find_checkpoint("taekwondo")

    for session, kw in (("origin", {}), ("shift", dict(shift=[[0, 0, 0], [0, 2, 0], [0, -2, 0]])),
                        ("scale", dict(scale=[1, 0.75, 1.5]))):
        model = modeling.build_layered_model(make_cfg(2, 64, 128, True, a.precision), 0, kw.get("scale"), kw.get("shift"))
        if ckpt is not None:
            checkpoint_io.load_checkpoint(model, ckpt)         # back-fills keys the file lacks (renderer :109-117)
        model.set_bkgd_bbox(bkgd); model.set_bboxes(frames); model.cuda()
        path = CameraPath(gt_poses, gt_Ks, layer_num=2, frame_num=101)
        path.set_smooth_path_poses(a.steps, around=False)
        path.retime_by_key_frames(1, key_frames_layer_1, key_frames)
        path.retime_by_key_frames(2, key_frames_layer_2, key_frames)
        pr = PoseRenderer(model, H, W, far=20.0)
        t0 = time.time()
        n = 0
        for idx, (color, depth, color_layer, depth_layer) in enumerate(
                pr.render_path(path.poses, path.Ks, path.layer_frame_pairs, density_threshold, 0, path.per_frame_state())):
            n += 1
            if a.out:
                from PIL import Image
                d = os.path.join(a.out, session)
                os.makedirs(d, exist_ok=True)
                Image.fromarray((color.clamp(0, 1) * 255).byte().numpy()).save(os.path.join(d, "%03d.png" % idx))
        dt = time.time() - t0
        print("%-6s %d frames of %dx%d in %.2fs  (%.0f rays/s incl. D2H)" % (session, n, W, H, dt, n * W * H / dt))


if __name__ == "__main__":
    main()
