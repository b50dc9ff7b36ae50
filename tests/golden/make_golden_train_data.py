#!/usr/bin/env python
"""Golden items of the reference's training data pipeline on the three captures of train_data_captures.py.  Runs the
UNMODIFIED reference on the CPU (its `data` and `utils` packages) with harness-side shims only:

  * an `open3d` module whose `io.read_point_cloud(path).points` is stnerf_b200.scene_data.read_ply_points(path);
  * torchvision's `rotate(..., resample=)` (random_transforms.py:106) mapped to today's `interpolation=`;
  * a namespace cfg with `clean_ray` (train_data_captures.make_cfg) and a temporary dataset directory, whose box and
    near/far caches are removed before the view dataset is built.

    python tests/golden/make_golden_train_data.py <reference root>

For each capture it stores the inputs (train_data_captures.capture_arrays), every `Ray_Dataset` item under
torch.manual_seed(0), the `Ray_Dataset_View.__getitem__` 8-tuple under np.random.seed(3), and the two
`ray_sampling_label_*` functions on one transformed image of the capture.  Writes tests/golden/train_data.npz."""
import contextlib
import io
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
VIEW_SEED, POOL_SEED = 3, 0


def _shims(ref_root):
    sys.path.insert(0, os.path.join(ROOT, "st-nerf_b200"))
    from stnerf_b200.scene_data import read_ply_points          # host-only module: no facade package is imported
    o3d = types.ModuleType("open3d")
    o3d.io = types.SimpleNamespace(read_point_cloud=lambda p: types.SimpleNamespace(points=read_ply_points(p)))
    sys.modules["open3d"] = o3d
    import torchvision.transforms.functional as TF
    rotate = TF.rotate

    def rotate_resample(img, *a, resample=None, **k):
        if resample is not None:
            k["interpolation"] = TF.InterpolationMode.BICUBIC if resample == 3 else resample
        return rotate(img, *a, **k)

    TF.rotate = rotate_resample
    sys.path.insert(0, ref_root)
    sys.path.insert(1, HERE)
    sys.path.insert(2, ROOT)


@contextlib.contextmanager
def recording(calls, draws):
    """Record what Ray_Frame_Layer_Dataset passes to the two sampling functions and every torch.randperm it draws."""
    import data.datasets.ray_dataset as RD
    f_bbox, f_label, randperm = RD.ray_sampling_label_bbox, RD.ray_sampling_label_label, torch.randperm

    def by_bbox(image, label, K, T, bbox=None, bboxes=None):
        r = f_bbox(image, label, K, T, bbox, bboxes)
        m = r[3][..., 0].numpy() > 0
        rows, cols = np.nonzero(m.any(1))[0], np.nonzero(m.any(0))[0]
        calls.append((K.numpy().copy(), T.numpy().copy(), (rows[0], rows[-1] + 1, cols[0], cols[-1] + 1)))
        return r

    def by_label(image, label, K, T, label0):
        calls.append((K.numpy().copy(), T.numpy().copy(), (-1, -1, -1, -1)))
        return f_label(image, label, K, T, label0)

    def rp(n, *a, **k):
        p = randperm(n, *a, **k)
        draws.append(p.numpy().copy())
        return p

    RD.ray_sampling_label_bbox, RD.ray_sampling_label_label, torch.randperm = by_bbox, by_label, rp
    try:
        yield
    finally:
        RD.ray_sampling_label_bbox, RD.ray_sampling_label_label, torch.randperm = f_bbox, f_label, randperm


def main(ref_root):
    _shims(ref_root)
    import train_data_captures as TC
    with contextlib.redirect_stdout(io.StringIO()):
        import data
        from utils import ray_sampling_label_bbox, ray_sampling_label_label
    out = {}
    for name in TC.NAMES:
        arrays = TC.capture_arrays(name)
        for k, v in arrays.items():
            out["%s.in.%s" % (name, k)] = v
        with tempfile.TemporaryDirectory() as d:
            TC.write_capture(d, name, arrays)
            cfg = TC.make_cfg(name, d)
            torch.manual_seed(POOL_SEED)
            calls, draws = [], []
            with contextlib.redirect_stdout(io.StringIO()), recording(calls, draws):
                _, ds = data.make_ray_data_loader(cfg, is_train=True)
            # per selection call, in the reference's order: K, T after the transform, and the kept rectangle (minh, maxh,
            # minw, maxw) of a box selection (-1s for a label selection); the background randperm draws
            out["%s.call_K" % name] = np.stack([c[0] for c in calls])
            out["%s.call_T" % name] = np.stack([c[1] for c in calls])
            out["%s.call_rect" % name] = np.array([c[2] for c in calls], dtype=np.int64)
            out["%s.draw_n" % name] = np.array([len(p) for p in draws], dtype=np.int64)
            out["%s.draw_perm" % name] = np.concatenate([p for p in draws]) if draws else np.zeros(0, np.int64)
            n = len(ds)
            items = [ds[i] for i in range(n)]
            for j, key in enumerate(("rays", "rgbs", "labels", "bbox_labels", "bboxes", "near_far")):
                # a performer without a point cloud has layer_bbox = zeros(8,3) (ray_dataset.py:370), whose [0] is a (3,) row
                # of zeros that default collate cannot stack with (8,3) boxes: stored as the zero box it stands for
                vals = [it[j].expand(8, 3) if key == "bboxes" and it[j].shape == (3,) else it[j] for it in items]
                out["%s.%s" % (name, key)] = torch.stack(vals).numpy()
            out["%s.bboxes_table" % name] = ds.bboxes.numpy()
            out["%s.segments" % name] = np.array([len(fl) for row in ds.datasets for fl in row])
            out["%s.camera_num" % name] = np.array(ds.camera_num)
            # view, from a fresh directory state: the reference's box / near-far caches hold numpy pickles that torch.load
            # refuses by default today
            for cache in ("bbox_tmp", "near_far_tmp"):
                shutil.rmtree(os.path.join(d, cache), ignore_errors=True)
            # (the reference cannot build a view of a capture with a box-less performer: it assigns None as a box, :187)
            if not TC.SPECS[name]["no_cloud"]:
                np.random.seed(VIEW_SEED)
                with contextlib.redirect_stdout(io.StringIO()):
                    _, vds = data.make_ray_data_loader_view(cfg)
                    tup = vds[0]
                for j, key in enumerate(("rays", "rgbs", "labels", "image", "label", "ray_mask", "layered_bboxes",
                                         "near_far")):
                    out["%s.view.%s" % (name, key)] = tup[j].numpy()
            # the two sampling functions on frame slot 0, first unmasked camera of the performer geometry
            fl = ds.datasets[1][0].frame_dataset
            cam = next(i for i in range(fl.cam_num) if fl.get_data(i)[7])
            image, label, K, T, _, bbox, _, _ = fl.get_data(cam)
            out["%s.fn.image" % name], out["%s.fn.label" % name] = image.numpy(), label.numpy()
            out["%s.fn.K" % name], out["%s.fn.T" % name] = K.numpy(), T.numpy()
            out["%s.fn.bbox" % name] = (bbox if bbox is not None else torch.zeros(1, 8, 3)).numpy()
            with contextlib.redirect_stdout(io.StringIO()):
                r = ray_sampling_label_bbox(image, label, K, T, bbox)
                for j, key in enumerate(("rays", "labels", "rgbs", "ray_mask")):
                    out["%s.fn.bbox_%s" % (name, key)] = r[j].numpy()
                r = ray_sampling_label_label(image, label, K, T, 1)
                for j, key in enumerate(("rays", "labels", "rgbs", "ray_mask")):
                    out["%s.fn.label_%s" % (name, key)] = r[j].numpy()
    np.savez_compressed(os.path.join(HERE, "train_data.npz"), **out)
    for name in TC.NAMES:
        print(name, out["%s.rays" % name].shape, out["%s.segments" % name])


if __name__ == "__main__":
    main(sys.argv[1])
