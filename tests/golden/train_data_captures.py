"""Three small captured scenes in the reference's dataset layout, for the training-data pipeline's golden and tests.

    tkd     taekwondo-like: USE_LABEL, background rate 0.5, two performers, a VIEW_MASK that hides camera 2, a time column
    walk    walking-like: box rectangles (one box partly off-screen, one with corners behind camera 1+FILE_OFFSET), background
            rate 0, FIXED_LAYER [3], CAMERA_NUM 3 with FILE_OFFSET 1, FRAME_OFFSET 2, image names `%d.png`, `%03d_label.npy`
    resize  SIZE_TRAIN (20x15) != SIZE_LAYER (16x10) below the 40x30 images (the layer crop runs past the image edge), a
            camera without a label map, label values >= 256 (np.uint8 wraps them), a performer without a point cloud, fixed
            near/far, labels named `%d.npy`

`capture_arrays(name)` builds every input from a seed; `write_capture(root, arrays)` writes them as files, so the tests
rebuild the very scene the golden was made from out of the arrays stored in train_data.npz."""
import os
import types

import numpy as np

import cases as C
from oracle import stnerf_oracle as O

NAMES = ("tkd", "walk", "resize")

SPECS = {
    "tkd": dict(layer_num=2, frame_num=2, frame_offset=0, cams=4, poses=4, size=(30, 20), size_train=(30, 20),
                size_layer=(30, 20), use_label=True, rate=0.5, fixed_layer=[], camera_num=0, file_offset=0,
                view_mask=[1, 1, 0, 1], near_far=(-1.0, -1.0), time=True, scale=1.0, img_fmt="%03d.png",
                lbl_fmt="%03d.npy", no_label=(), no_cloud=(), batch=64),
    "walk": dict(layer_num=3, frame_num=2, frame_offset=2, cams=3, poses=5, size=(32, 24), size_train=(32, 24),
                 size_layer=(32, 24), use_label=False, rate=0.0, fixed_layer=[3], camera_num=3, file_offset=1,
                 view_mask=None, near_far=(-1.0, -1.0), time=False, scale=1.0, img_fmt="%d.png", lbl_fmt="%03d_label.npy",
                 no_label=(), no_cloud=(), batch=100),
    "resize": dict(layer_num=2, frame_num=2, frame_offset=0, cams=3, poses=3, size=(40, 30), size_train=(20, 15),
                   size_layer=(16, 10), use_label=True, rate=0.3, fixed_layer=[], camera_num=0, file_offset=0,
                   view_mask=None, near_far=(0.5, 20.0), time=True, scale=1.0, img_fmt="%03d.png", lbl_fmt="%d.npy",
                   no_label=((1, 1),), no_cloud=(2,), batch=50),
}


def _points(name, layer, frame):
    rng = np.random.RandomState(1000 * NAMES.index(name) + 10 * layer + frame)
    if layer == 0:
        p = rng.uniform([-6, -6, -1], [6, 6, 4], size=(200, 3))
    elif name == "walk" and layer == 2:
        p = rng.uniform([0.5, 3.5, 0.2], [2.6, 6.0, 1.6], size=(60, 3))        # spans camera 1's position (1.55, 4.76, 1)
    elif name == "walk" and layer == 1:
        p = rng.uniform([-0.5, 1.5, 0.0], [0.5, 3.9, 1.8], size=(60, 3))       # partly off-screen in some views
    else:
        c = np.array([-1.0 + layer * 0.8 + 0.1 * frame, 0.2 * frame, 0.9])
        p = c + rng.normal(size=(80, 3)) * np.array([0.3, 0.3, 0.5])
    return p.astype(np.float32).astype(np.float64)


def capture_arrays(name):
    sp = SPECS[name]
    rng = np.random.RandomState(77 + NAMES.index(name))
    W, H = sp["size"]
    out = {}
    Ks, Ts = [], []
    for v in range(sp["poses"]):
        K, T = O.synthetic_camera(v, sp["poses"], H, W)
        Ks.append(np.asarray(K, dtype=np.float64).reshape(-1))
        Ts.append(np.asarray(T, dtype=np.float64)[:3].reshape(-1))
    out["K"], out["RT"] = np.stack(Ks), np.stack(Ts)
    out["cloud.0"] = _points(name, 0, 0)
    frames = range(1 + sp["frame_offset"], sp["frame_offset"] + sp["frame_num"] + 1)
    for f in frames:
        for l in range(1, sp["layer_num"] + 1):
            if l not in sp["no_cloud"]:
                out["cloud.%d.%d" % (l, f)] = _points(name, l, f)
        for c in range(sp["poses"]):
            out["image.%d.%d" % (f, c)] = rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8)
            if (f - sp["frame_offset"], c) in sp["no_label"]:
                continue
            lab = rng.randint(0, sp["layer_num"] + 2, size=(H, W)).astype(np.int64)
            if name == "resize":
                lab = lab + 256 * rng.randint(0, 2, size=(H, W))                 # 256 + k wraps to k
            out["label.%d.%d" % (f, c)] = lab
    return out


def write_capture(root, name, arrays):
    from PIL import Image
    sp = SPECS[name]
    os.makedirs(os.path.join(root, "pose"), exist_ok=True)
    os.makedirs(os.path.join(root, "background"), exist_ok=True)
    np.savetxt(os.path.join(root, "pose", "K.txt"), arrays["K"], fmt="%.10g")
    np.savetxt(os.path.join(root, "pose", "RT_c2w.txt"), arrays["RT"], fmt="%.10g")
    C.write_ply(os.path.join(root, "background", "0.ply"), arrays["cloud.0"], "le_f4")
    for k, v in arrays.items():
        parts = k.split(".")
        if parts[0] == "cloud" and len(parts) == 3:
            d = os.path.join(root, "frame" + parts[2], "pointclouds")
            os.makedirs(d, exist_ok=True)
            C.write_ply(os.path.join(d, "%s.ply" % parts[1]), v, "le_f4")
        elif parts[0] == "image":
            d = os.path.join(root, "frame" + parts[1], "images")
            os.makedirs(d, exist_ok=True)
            Image.fromarray(v).save(os.path.join(d, sp["img_fmt"] % int(parts[2])))
        elif parts[0] == "label":
            d = os.path.join(root, "frame" + parts[1], "labels")
            os.makedirs(d, exist_ok=True)
            np.save(os.path.join(d, sp["lbl_fmt"] % int(parts[2])), v)
    if sp["view_mask"] is not None:
        with open(os.path.join(root, "view_mask.txt"), "w") as f:
            f.write("".join("%d\n" % m for m in sp["view_mask"]))
    return root


def make_cfg(name, root):
    """The cfg fields the reference's data package and stnerf_b200.train_data read (configs/config_*.yml layout)."""
    sp = SPECS[name]
    D = types.SimpleNamespace(
        TRAIN=root, FRAME_NUM=sp["frame_num"], LAYER_NUM=sp["layer_num"], FRAME_OFFSET=sp["frame_offset"],
        BKGD_SAMPLE_RATE=sp["rate"], FIXED_LAYER=list(sp["fixed_layer"]), USE_LABEL=sp["use_label"], CAMERA_STEPSIZE=1,
        FILE_OFFSET=sp["file_offset"], CAMERA_NUM=sp["camera_num"],
        VIEW_MASK=os.path.join(root, "view_mask.txt") if sp["view_mask"] is not None else None, SCALE=sp["scale"],
        FIXED_NEAR=sp["near_far"][0], FIXED_FAR=sp["near_far"][1], SHIFT=0, MAXRATION=0.0, ROTATION=0.0,
        TMP_RAYS="rays_tmp")
    M = types.SimpleNamespace(POSE_REFINEMENT=False, USE_DEFORM_VIEW=False, USE_DEFORM_TIME=sp["time"],
                              USE_SPACE_TIME=sp["time"], REMOVE_OUTLIERS=False)
    I = types.SimpleNamespace(SIZE_TRAIN=list(sp["size_train"]), SIZE_LAYER=list(sp["size_layer"]),
                              SIZE_TEST=list(sp["size"]))
    return types.SimpleNamespace(DATASETS=D, MODEL=M, INPUT=I, SOLVER=types.SimpleNamespace(IMS_PER_BATCH=sp["batch"]),
                                 DATALOADER=types.SimpleNamespace(NUM_WORKERS=0), clean_ray=True)
