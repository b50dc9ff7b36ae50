"""Host side of the training-data pipeline (stnerf_b200.train_data) against the unmodified reference's pipeline on the three
captures of tests/golden/train_data_captures.py (golden: tests/golden/train_data.npz, make_golden_train_data.py): camera
tables after the transform, box rectangles, background subsample draws, decoded images, file-name fallbacks, loud failures."""
import os

import numpy as np
import pytest
import torch

import train_data_captures as TC
from stnerf_b200 import train_data as TD


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(os.path.dirname(TC.__file__), "train_data.npz"))


def capture_inputs(golden, name):
    pre = name + ".in."
    return {k[len(pre):]: golden[k] for k in golden.files if k.startswith(pre)}


@pytest.fixture(scope="module")
def captures(golden, tmp_path_factory):
    out = {}
    for name in TC.NAMES:
        root = str(tmp_path_factory.mktemp(name))
        TC.write_capture(root, name, capture_inputs(golden, name))
        out[name] = root
    return out


def test_inputs_rebuild_from_seed(golden):
    """The stored inputs are what capture_arrays makes, so the fixture can be regenerated."""
    for name in TC.NAMES:
        got = TC.capture_arrays(name)
        want = capture_inputs(golden, name)
        assert sorted(got) == sorted(want)
        for k in got:
            assert np.array_equal(got[k], want[k]), (name, k)


def reference_calls(cfg, cap):
    """(layer, frame slot, camera) of every selection call Ray_Dataset makes, in its order."""
    D = cfg.DATASETS
    rates = [D.BKGD_SAMPLE_RATE] + [0.0 if l in D.FIXED_LAYER else 1.0 for l in range(1, cap.layer_num + 1)]
    cams = [cap.camera_id(i) for i in range(0, cap.camera_num, D.CAMERA_STEPSIZE)]
    cams = [c for c in cams if cap.mask[c] != 0]
    return [(l, s, c) for l in range(cap.layer_num + 1) if rates[l] != 0 for s in range(cap.frame_num) for c in cams]


def size_of(cfg, layer):
    return TD._hw(cfg.INPUT.SIZE_TRAIN if layer == 0 else cfg.INPUT.SIZE_LAYER)


@pytest.mark.parametrize("name", TC.NAMES)
def test_camera_tables_and_rectangles(golden, captures, name):
    cfg = TC.make_cfg(name, captures[name])
    cap = TD._Capture(cfg)
    calls = reference_calls(cfg, cap)
    assert len(calls) == golden[name + ".call_K"].shape[0]
    for i, (l, s, c) in enumerate(calls):
        H, W = size_of(cfg, l)
        height = TC.SPECS[name]["size"][1]
        K, T = TD.transform_camera(cap.Ks[c], cap.Ts[c], height, (H, W))
        assert np.array_equal(K.numpy(), golden[name + ".call_K"][i]), (l, s, c)
        assert np.array_equal(T.numpy(), golden[name + ".call_T"][i]), (l, s, c)
        want = tuple(golden[name + ".call_rect"][i])
        if want[0] >= 0:
            b = cap.fl[l][s].bbox
            got = (0, H, 0, W) if b is None else TD.box_rectangle(b, K, T, H, W)
            assert got == want, (l, s, c)
    if name == "walk":            # boxes that cover part of the image, not only clipped-to-full ones
        assert any(tuple(r) != (0, 24, 0, 32) for r in golden[name + ".call_rect"])


@pytest.mark.parametrize("name", TC.NAMES)
def test_background_subsample_draws(golden, name):
    rate = TC.SPECS[name]["rate"]
    ns, perms = golden[name + ".draw_n"], golden[name + ".draw_perm"]
    torch.manual_seed(0)
    o = 0
    for n in ns:
        keep = TD.subsample_order(int(n), rate)
        assert np.array_equal(keep.numpy(), perms[o:o + int(n * rate)])
        o += int(n)
    assert TD.subsample_order(10, 1.0) is None


def test_subsample_takes_the_product_in_double():
    torch.manual_seed(5)
    n, rate = 100, 0.57                                # 100 * 0.57 = 56.99999999999999 in double
    assert TD.subsample_order(n, rate).numel() == 56


@pytest.mark.parametrize("name", TC.NAMES)
def test_decoded_image_matches_reference_transform(golden, captures, name):
    """The Pillow crop + bicubic resize gives the reference's to_tensor image and label map, byte for byte."""
    cfg = TC.make_cfg(name, captures[name])
    cap = TD._Capture(cfg)
    first = cap.fl[1][0]
    cam = next(c for c in range(first.cam_num) if cap.mask[cap.camera_id(c)] != 0)
    cam = cap.camera_id(cam)
    H, W = size_of(cfg, 1)
    lbl_dir = os.path.join(os.path.dirname(first.image_path), "labels")
    rgb, lbl, _ = TD.decode(TD.image_path(first.image_path, cam), TD.label_path(lbl_dir, cam), (H, W))
    img = torch.from_numpy(np.ascontiguousarray(rgb)).permute(2, 0, 1).float().div(255)
    assert np.array_equal(img.numpy(), golden[name + ".fn.image"])
    assert np.array_equal(torch.from_numpy(lbl).float()[None].div(255).mul(255.0).numpy(), golden[name + ".fn.label"])


def test_missing_label_map_under_a_padding_crop():
    """A missing label map is the layer id everywhere; where the crop runs past the image edge Pillow pads it with 0 and the
    resize blends the two, as the reference's transform of np.ones * layer_id does."""
    from PIL import Image
    assert TD.constant_label(2, (40, 30), (15, 20)) is None                       # crop 40 wide: no padding
    got = TD.constant_label(2, (40, 30), (10, 16))                                # crop 48 wide: 8 padded columns
    want = np.array(Image.fromarray(np.full((30, 40), 2, np.uint8)).crop((0, 0, 48, 30)).resize((16, 10), Image.BICUBIC))
    assert np.array_equal(got, want) and (want != 2).any() and (want[:, :8] == 2).all()


def test_label_bytes_round_trip():
    """to_tensor(uint8 L image) * 255 is every byte exactly, so a uint8 label map carries the reference's float labels."""
    from PIL import Image
    import torchvision.transforms.functional as F
    b = np.arange(256, dtype=np.uint8).reshape(16, 16)
    assert np.array_equal((F.to_tensor(Image.fromarray(b)) * 255.0).numpy()[0], b.astype(np.float32))


def test_label_values_wrap_like_np_uint8(tmp_path):
    from PIL import Image
    lab = np.array([[0, 1, 255, 256], [257, 258, 511, 512]], dtype=np.int64)
    np.save(str(tmp_path / "000.npy"), lab)
    Image.fromarray(np.zeros((2, 4, 3), np.uint8)).save(str(tmp_path / "000.png"))
    _, got, _ = TD.decode(str(tmp_path / "000.png"), str(tmp_path / "000.npy"), (2, 4))
    assert np.array_equal(got, np.uint8(lab))


def test_file_name_fallbacks(tmp_path):
    d = str(tmp_path)
    assert TD.image_path(d, 7) is None and TD.label_path(d, 7) is None
    open(os.path.join(d, "7.png"), "w").close()
    assert TD.image_path(d, 7).endswith("/7.png")
    open(os.path.join(d, "007.png"), "w").close()
    assert TD.image_path(d, 7).endswith("/007.png")
    for nm in ("7.npy", "007_label.npy", "007.npy"):
        open(os.path.join(d, nm), "w").close()
        assert TD.label_path(d, 7).endswith("/" + nm)
    assert TD.read_view_mask(None) is None and TD.read_view_mask(os.path.join(d, "nope.txt")) is None


def test_crop_width_follows_the_target_aspect():
    assert TD.crop_width(1080, (1080, 1920)) == 1920
    assert TD.crop_width(30, (10, 16)) == 48          # wider than a 40-pixel image: Pillow pads the crop with zeros


@pytest.mark.parametrize("field,value,exc", [
    ("DATASETS.SHIFT", 2, NotImplementedError), ("DATASETS.MAXRATION", 0.1, NotImplementedError),
    ("DATASETS.ROTATION", 5.0, NotImplementedError), ("MODEL.POSE_REFINEMENT", True, NotImplementedError),
    ("MODEL.USE_DEFORM_VIEW", True, NotImplementedError)])
def test_unsupported_config_fails_loudly(captures, field, value, exc):
    cfg = TC.make_cfg("tkd", captures["tkd"])
    sec, key = field.split(".")
    setattr(getattr(cfg, sec), key, value)
    with pytest.raises(exc):
        TD.TrainRayDataset(cfg)
    with pytest.raises(exc):
        TD.ViewDataset(cfg)


def test_missing_image_fails_loudly(golden, tmp_path):
    root = TC.write_capture(str(tmp_path), "tkd", capture_inputs(golden, "tkd"))
    os.remove(os.path.join(root, "frame2", "images", "001.png"))
    with pytest.raises(ValueError, match="missing image"):
        TD.TrainRayDataset(TC.make_cfg("tkd", root))


def test_non_rgb_image_fails_loudly(golden, tmp_path):
    from PIL import Image
    root = TC.write_capture(str(tmp_path), "tkd", capture_inputs(golden, "tkd"))
    p = os.path.join(root, "frame1", "images", "000.png")
    Image.open(p).convert("RGBA").save(p)
    with pytest.raises(ValueError, match="8-bit RGB"):
        TD.TrainRayDataset(TC.make_cfg("tkd", root))


def test_every_camera_masked_fails_loudly(golden, tmp_path):
    root = TC.write_capture(str(tmp_path), "tkd", capture_inputs(golden, "tkd"))
    with open(os.path.join(root, "view_mask.txt"), "w") as f:
        f.write("0\n0\n0\n0\n")
    with pytest.raises(ValueError, match="view mask"):
        TD.TrainRayDataset(TC.make_cfg("tkd", root))
