"""Training data from a captured scene (SURVEY 8f row 4): the reference's training ray set, built on the GPU and batched there.

    make_ray_data_loader       <- data/build.py:13-27 + Ray_Dataset / Ray_Frame_Layer_Dataset  data/datasets/ray_dataset.py:13-83,339-460
    make_ray_data_loader_view  <- data/build.py:29-42 + Ray_Dataset_View                       ray_dataset.py:85-201
    select_pixels              <- utils/ray_sampling.py:75-240 (the pixel choice of ray_sampling_label_bbox / _label)

Host side: cameras, boxes and near/far come from `scene_data.FrameLayerData`; each (frame, camera) image is decoded once per
image geometry with Pillow (the deterministic branch of data/transforms/random_transforms.py:56-163: crop, bicubic resize,
K * s with K[2,2] = 1) and uploaded once as uint8 RGB plus a uint8 label map.  Device side: a selection kernel per (image,
layer) appends 16-byte pool entries (pixel, camera, frame slot, layer, RGB, label) in the reference's order, the background is
subsampled with the reference's `torch.randperm` draws, and one kernel turns B pool indices into the trainer's batch.
"""
from __future__ import annotations

import concurrent.futures
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import ops
from .scene_data import FrameLayerData

ENTRY_BYTES = 16


# ---------------------------------------------------------------------------------------------------------------------
# host: images, labels, cameras
# ---------------------------------------------------------------------------------------------------------------------
def image_path(image_dir: str, camera_id: int) -> Optional[str]:
    """frame_dataset.py:264-266: `%03d.png`, then `%d.png`."""
    for nm in ("%03d.png" % camera_id, "%d.png" % camera_id):
        p = os.path.join(image_dir, nm)
        if os.path.exists(p):
            return p
    return None


def label_path(label_dir: str, camera_id: int) -> Optional[str]:
    """frame_dataset.py:273-277: `%03d.npy`, then `%03d_label.npy`, then `%d.npy`."""
    for nm in ("%03d.npy" % camera_id, "%03d_label.npy" % camera_id, "%d.npy" % camera_id):
        p = os.path.join(label_dir, nm)
        if os.path.exists(p):
            return p
    return None


def read_view_mask(path) -> Optional[np.ndarray]:
    """data/datasets/utils.py:80-90 (one int per line); None when unset or absent, as frame_dataset.py:137-141."""
    if path is None or not os.path.exists(path):
        return None
    with open(path) as f:
        return np.array([int(line) for line in f.readlines()])


def crop_width(height: int, size_hw: Sequence[int]) -> int:
    """random_transforms.py:108 with ration = 1.0: the crop keeps the full height and a width of the target's aspect."""
    return int(height * size_hw[1] / 1.0 / size_hw[0])


def transform_image(img, size_hw: Sequence[int]):
    """random_transforms.py:106-110 with SHIFT = MAXRATION = ROTATION = 0 (rotate and affine are the identity): crop to
    (0, 0, crop_width, height), then a bicubic resize to size_hw = (H, W) -- the Pillow calls torchvision makes."""
    from PIL import Image
    width, height = img.size
    img = img.crop((0, 0, crop_width(height, size_hw), height))
    return img.resize((int(size_hw[1]), int(size_hw[0])), Image.BICUBIC)


def transform_camera(K: torch.Tensor, T: torch.Tensor, height: int, size_hw: Sequence[int]):
    """random_transforms.py:70-73, :149-156 with zero rotation and translation: (K * s with K[2,2] = 1, T)."""
    K = K.clone()
    Tc = T.clone()
    Tc[0:3, 0:3] = torch.matmul(Tc[0:3, 0:3], torch.eye(3))
    K[0, 2] = K[0, 2] + 0.0
    K[1, 2] = K[1, 2] + 0.0
    s = size_hw[0] * 1.0 / height
    K = K * s
    K[2, 2] = 1
    return K, Tc


def decode(img_file: str, lbl_file: Optional[str], size_hw: Sequence[int]):
    """One (frame, camera) image at one geometry -> (rgb uint8 (H,W,3), label uint8 (H,W) or None, original (width, height))."""
    from PIL import Image
    with Image.open(img_file) as im:
        if im.mode != "RGB":
            raise ValueError("%s: %s image; training images must be 8-bit RGB" % (img_file, im.mode))
        im.load()
        size = im.size
        rgb = np.array(transform_image(im, size_hw))
        lbl = None
        if lbl_file is not None:
            lab = Image.fromarray(np.uint8(np.load(lbl_file)))      # random_transforms.py:134 (values >= 256 wrap)
            lbl = np.array(transform_image(lab, size_hw))
    return rgb, lbl, size


def constant_label(value: int, size_wh: Sequence[int], size_hw: Sequence[int]) -> Optional[np.ndarray]:
    """The transformed full map of `value` that stands in for a missing label map (frame_dataset.py:278-284), or None when it
    is the constant itself: bicubic resizing keeps a constant map constant, but a crop wider than the image pads it with 0."""
    if crop_width(size_wh[1], size_hw) <= size_wh[0]:
        return None
    from PIL import Image
    return np.array(transform_image(Image.fromarray(np.full((size_wh[1], size_wh[0]), value, np.uint8)), size_hw))


def box_rectangle(bbox: torch.Tensor, K: torch.Tensor, T: torch.Tensor, H: int, W: int) -> Tuple[int, int, int, int]:
    """ray_sampling.py:79-119 in the same torch CPU ops: the pixel rectangle (minh, maxh, minw, maxw) of a box's projection."""
    b = torch.transpose(bbox.reshape(8, 3), 0, 1)
    b = torch.cat([b, torch.ones(1, b.shape[1])], 0)
    pts = torch.mm(torch.inverse(T), b)[:3, :]
    px = torch.mm(K, pts)
    px = (px / px[2, :])[:2, :]
    hw = torch.zeros_like(px)
    hw[1, :] = px[0, :]
    hw[0, :] = px[1, :]
    lo, hi = torch.min(hw, dim=1)[0], torch.max(hw, dim=1)[0]
    for v in (lo, hi):
        v[v < 0.0] = 0
        if v[0] >= H - 1:
            v[0] = H - 1
        if v[1] >= W - 1:
            v[1] = W - 1
    return int(lo[0]), int(hi[0]) + 1, int(lo[1]), int(hi[1]) + 1


# ---------------------------------------------------------------------------------------------------------------------
# device: selection
# ---------------------------------------------------------------------------------------------------------------------
def _select(label, label_is_float: int, const_label: int, H: int, W: int, mode: int, layer: int, rect, rgb=None,
            camera: int = 0, frame_slot: int = 0, want_pool: bool = True):
    """Run the selection kernel on one image; returns pool entries (n,4) int32 or pixel indices (n,) int32 on the device."""
    dev = (label if label is not None else rgb).device
    lib = L.lib()
    scratch = torch.empty(int(lib.stnerf_td_select_scratch_ints(H, W)), dtype=torch.int32, device=dev)
    rect_h = None if rect is None else torch.tensor(list(rect), dtype=torch.int32)
    with torch.cuda.device(dev):
        L.check(lib.stnerf_td_select_count(L.ptr(label), label_is_float, int(const_label), H, W, mode, layer, L.ptr(rect_h),
                                           L.ptr(scratch), L.stream_ptr()), "stnerf_td_select_count")
        n = int(scratch[-1].item())
        out = torch.empty((n, 4) if want_pool else (n,), dtype=torch.int32, device=dev)
        if n:
            L.check(lib.stnerf_td_select_write(L.ptr(label), label_is_float, int(const_label), L.ptr(rgb), H, W, mode, layer,
                                               L.ptr(rect_h), int(camera), int(frame_slot), L.ptr(scratch),
                                               L.ptr(out) if want_pool else None, None if want_pool else L.ptr(out),
                                               L.stream_ptr()), "stnerf_td_select_write")
    return out


def select_pixels(label: torch.Tensor, layer: int = 0, rect=None) -> torch.Tensor:
    """Row-major indices of the pixels of an (H,W) CUDA label map (float or uint8) that ray_sampling_label_label keeps
    (label == layer, rect None) or ray_sampling_label_bbox keeps (rect = (minh, maxh, minw, maxw))."""
    H, W = label.shape[-2:]
    lab = label.reshape(H, W).contiguous()
    is_float = 1 if lab.dtype.is_floating_point else 0
    if is_float:
        lab = lab.to(torch.float32)
    elif lab.dtype != torch.uint8:
        raise ValueError("label maps are float or uint8, got %s" % lab.dtype)
    mode = L.TD_BY_LABEL if rect is None else L.TD_BY_RECT
    return _select(lab, is_float, 0, H, W, mode, int(layer), rect, want_pool=False)


def subsample_order(n: int, rate: float) -> Optional[torch.Tensor]:
    """ray_dataset.py:429-439: None at rate 1 (no draw), else the first int(n * rate) entries of one torch.randperm(n) from
    the default CPU generator, in permuted order."""
    if rate == 1:
        return None
    perm = torch.randperm(n)
    return perm[:int(n * rate)]


# ---------------------------------------------------------------------------------------------------------------------
# the training ray pool
# ---------------------------------------------------------------------------------------------------------------------
def _check_cfg(cfg):
    D, M = cfg.DATASETS, cfg.MODEL
    for k in ("SHIFT", "MAXRATION", "ROTATION"):
        if getattr(D, k, 0) != 0:
            raise NotImplementedError("DATASETS.%s != 0 (random augmentation) is not supported; every shipped config uses 0" % k)
    if getattr(M, "POSE_REFINEMENT", False):
        raise NotImplementedError("MODEL.POSE_REFINEMENT is not supported (no shipped config sets it)")
    if getattr(M, "USE_DEFORM_VIEW", False):
        raise NotImplementedError("MODEL.USE_DEFORM_VIEW is not supported (no shipped config sets it)")


def _hw(size_wh) -> Tuple[int, int]:
    return int(size_wh[1]), int(size_wh[0])


class _Capture:
    """Cameras, boxes and near/far of every (layer, frame), and the camera ids the training set walks."""

    def __init__(self, cfg):
        D = cfg.DATASETS
        self.path = D.TRAIN
        self.layer_num, self.frame_num, self.frame_offset = int(D.LAYER_NUM), int(D.FRAME_NUM), int(D.FRAME_OFFSET)
        self.camera_num_cfg = int(getattr(D, "CAMERA_NUM", 0))
        self.file_offset = int(getattr(D, "FILE_OFFSET", 0))
        self.frames = list(range(1 + self.frame_offset, self.frame_offset + self.frame_num + 1))
        self.fl: List[List[FrameLayerData]] = []
        for layer_id in range(self.layer_num + 1):
            self.fl.append([FrameLayerData(self.path, f, layer_id, float(D.SCALE), float(D.FIXED_NEAR), float(D.FIXED_FAR),
                                           self.camera_num_cfg) for f in self.frames])
        first = self.fl[0][0]
        self.Ts, self.Ks = first.Ts, first.Ks
        self.n_poses = int(self.Ts.shape[0])
        self.camera_num = first.cam_num
        self.mask = read_view_mask(getattr(D, "VIEW_MASK", None))
        if self.mask is None:
            self.mask = np.ones(self.n_poses)
        self.bboxes = torch.zeros(self.frame_num + self.frame_offset, self.layer_num, 8, 3)
        for layer_id in range(1, self.layer_num + 1):
            for j, f in enumerate(self.frames):
                self.bboxes[f - 1, layer_id - 1] = self.box(layer_id, j)
        self.bkgd_bbox = first.bbox

    def box(self, layer_id: int, slot: int) -> torch.Tensor:
        """Ray_Frame_Layer_Dataset.layer_bbox (ray_dataset.py:367-370): the box, or zeros without a point cloud."""
        b = self.fl[layer_id][slot].bbox
        return torch.zeros(8, 3) if b is None else b.reshape(8, 3)

    def camera_id(self, i: int) -> int:
        """frame_dataset.py:254-255: CAMERA_NUM != 0 offsets the camera before the mask, file and pose lookups."""
        return i + self.file_offset if self.camera_num_cfg != 0 else i

    def near_far(self, layer_id: int, slot: int, cam: int) -> torch.Tensor:
        d = self.fl[layer_id][slot]
        return torch.tensor([d.near[cam], d.far[cam]]).unsqueeze(0)


class TrainRayDataset:
    """The training ray set of `Ray_Dataset` as a device pool.  `items(idx)` is the collated batch of those indices."""

    def __init__(self, cfg, device="cuda", workers: Optional[int] = None):
        import time
        _check_cfg(cfg)
        D, M = cfg.DATASETS, cfg.MODEL
        self.device = torch.device(device)
        self.cap = cap = _Capture(cfg)
        self.layer_num, self.frame_num, self.frame_offset = cap.layer_num, cap.frame_num, cap.frame_offset
        self.bboxes, self.bkgd_bbox, self.camera_num = cap.bboxes, cap.bkgd_bbox, cap.camera_num
        self.time_col = 1 if (getattr(M, "USE_DEFORM_TIME", False) or getattr(M, "USE_SPACE_TIME", False)) else 0
        fixed = set(int(x) for x in getattr(D, "FIXED_LAYER", []))
        use_label = bool(getattr(D, "USE_LABEL", False))
        step = int(getattr(D, "CAMERA_STEPSIZE", 1))
        bkgd_rate = float(D.BKGD_SAMPLE_RATE)
        # per layer: sample rate, selection mode and image geometry (transforms/build.py:37-39: SIZE_TRAIN for the background)
        self.rate = [bkgd_rate] + [0.0 if l in fixed else 1.0 for l in range(1, cap.layer_num + 1)]
        self.by_label = [True] + [use_label] * cap.layer_num
        sizes = [_hw(cfg.INPUT.SIZE_TRAIN), _hw(cfg.INPUT.SIZE_LAYER)]
        self.geometries = sorted(set(sizes[0 if l == 0 else 1] for l in range(cap.layer_num + 1)))
        self.geom_of_layer = [self.geometries.index(sizes[0 if l == 0 else 1]) for l in range(cap.layer_num + 1)]
        cams = [cap.camera_id(i) for i in range(0, cap.camera_num, step)]
        self.cameras = [c for c in cams if cap.mask[c] != 0]
        self.timing = {"decode_s": 0.0, "select_s": 0.0, "randperm_s": 0.0}
        for l in range(cap.layer_num + 1):
            if self.rate[l] != 0.0 and not self.cameras:
                raise ValueError("layer %d: every camera is hidden by the view mask" % l)

        # camera tables after the transform, per (geometry, pose); images are decoded from their own height
        self.K_tab = torch.zeros(len(self.geometries), cap.n_poses, 3, 3)
        self.T_tab = torch.zeros(len(self.geometries), cap.n_poses, 4, 4)
        cam_tab = torch.zeros(len(self.geometries), cap.n_poses, 24)
        seg: Dict[Tuple[int, int], List[torch.Tensor]] = {}
        live = [l for l in range(cap.layer_num + 1) if self.rate[l] != 0.0]
        geoms_needed = sorted(set(self.geom_of_layer[l] for l in live))
        heights = {}
        frame_files = []          # every file is looked up before any work starts
        for frame_id in cap.frames:
            img_dir = os.path.join(cap.path, "frame%d" % frame_id, "images")
            lbl_dir = os.path.join(cap.path, "frame%d" % frame_id, "labels")
            files = []
            for c in (self.cameras if live else []):
                p = image_path(img_dir, c)
                if p is None:
                    raise ValueError("missing image for camera %d under %s" % (c, img_dir))
                files.append((c, p, label_path(lbl_dir, c)))
            frame_files.append(files)
        pool_ex = concurrent.futures.ThreadPoolExecutor(max_workers=workers or min(16, os.cpu_count() or 1))
        try:
            for slot, files in enumerate(frame_files):
                t0 = time.perf_counter()
                jobs = {(c, g): pool_ex.submit(decode, p, lp, self.geometries[g]) for c, p, lp in files for g in geoms_needed}
                decoded = {k: f.result() for k, f in jobs.items()}
                self.timing["decode_s"] += time.perf_counter() - t0
                t0 = time.perf_counter()
                for c, _, _ in files:
                    for g in geoms_needed:
                        rgb, lbl, size = decoded[(c, g)]
                        height = size[1]
                        H, W = self.geometries[g]
                        if heights.setdefault((g, c), size) != size:
                            raise ValueError("camera %d changes image size between frames" % c)
                        K, T = transform_camera(cap.Ks[c], cap.Ts[c], height, (H, W))
                        self.K_tab[g, c], self.T_tab[g, c] = K, T
                        cam_tab[g, c, 0:9] = torch.inverse(K).reshape(9)
                        cam_tab[g, c, 9:18] = T[:3, :3].reshape(9)
                        cam_tab[g, c, 18:21] = T[:3, 3]
                        cam_tab[g, c, 21] = float(W)
                        rgb_d = torch.from_numpy(rgb).to(self.device)
                        lbl_d = None if lbl is None else torch.from_numpy(lbl).to(self.device)
                        for l in live:
                            if self.geom_of_layer[l] != g:
                                continue
                            lbl_l = lbl_d
                            if lbl is None:
                                const = constant_label(l, size, (H, W))
                                if const is not None:
                                    lbl_l = torch.from_numpy(const).to(self.device)
                            if self.by_label[l]:
                                mode, rect = L.TD_BY_LABEL, None
                            else:       # no point cloud: get_data's bbox is None and the whole image is kept (:120-124)
                                b = cap.fl[l][slot].bbox
                                mode = L.TD_BY_RECT
                                rect = (0, H, 0, W) if b is None else box_rectangle(b, K, T, H, W)
                            seg.setdefault((l, slot), []).append(
                                _select(lbl_l, 0, l, H, W, mode, l, rect, rgb=rgb_d, camera=c, frame_slot=slot))
                self.timing["select_s"] += time.perf_counter() - t0
        finally:
            pool_ex.shutdown()

        # segments in the reference's order; the background keeps the first int(n * rate) of one randperm per frame
        # (ray_dataset.py:429-439), drawn from the default CPU generator in construction order
        parts = []
        self.segments = []
        self.subsample_idx = {}
        for l in range(cap.layer_num + 1):
            for slot in range(cap.frame_num):
                if self.rate[l] == 0.0:
                    self.segments.append((l, slot, 0))
                    continue
                s = torch.cat(seg[(l, slot)], 0)
                t0 = time.perf_counter()
                keep = subsample_order(s.shape[0], self.rate[l])
                self.timing["randperm_s"] += time.perf_counter() - t0
                if keep is not None:
                    self.subsample_idx[(l, slot)] = keep
                    s = s[keep.to(self.device)]
                parts.append(s)
                self.segments.append((l, slot, int(s.shape[0])))
        self.pool = torch.cat(parts, 0).contiguous() if parts else torch.zeros((0, 4), dtype=torch.int32, device=self.device)
        self.cams = cam_tab.to(self.device).contiguous()
        boxes = torch.zeros(cap.layer_num + 1, cap.frame_num, 24)
        nf = torch.zeros(cap.layer_num + 1, cap.frame_num, cap.n_poses, 2)
        for l in range(cap.layer_num + 1):
            for slot in range(cap.frame_num):
                if l == 0:
                    b = cap.fl[0][slot].bbox
                    boxes[l, slot] = torch.zeros(24) if b is None else b.reshape(24)
                else:
                    boxes[l, slot] = cap.box(l, slot).reshape(24)
                d = cap.fl[l][slot]
                nf[l, slot, :, 0] = d.near
                nf[l, slot, :, 1] = d.far
        self.boxes, self.near_far_tab = boxes.to(self.device), nf.to(self.device)
        self._geom = (torch.tensor(self.geom_of_layer, dtype=torch.int32))

    def __len__(self):
        return int(self.pool.shape[0])

    @property
    def pool_bytes(self) -> int:
        return self.pool.numel() * self.pool.element_size()

    def items(self, idx: torch.Tensor, out: Optional[torch.Tensor] = None):
        """The collated batch of pool indices `idx` (device int32 / int64): (rays (B,6[+1]), rgbs (B,3), labels (B,1),
        bbox_labels (B,1), bboxes (B,8,3), near_far (B,2)), views of one fresh buffer."""
        idx = idx.to(self.device)
        if idx.dtype not in (torch.int32, torch.int64):
            idx = idx.long()
        idx = idx.contiguous()
        B = int(idx.shape[0])
        w = 6 + self.time_col
        cols = (w, 3, 1, 1, 24, 2)
        buf = torch.empty((sum(cols) * B,), dtype=torch.float32, device=self.device)
        views, o = [], 0
        for c in cols:
            views.append(buf[o:o + B * c].view(B, c))
            o += B * c
        rays, rgbs, labels, bbl, bboxes, nf = views
        with torch.cuda.device(self.device):
            L.check(L.lib().stnerf_td_batch(L.ptr(self.pool), L.ptr(idx), 1 if idx.dtype == torch.int64 else 0, B,
                                            L.ptr(self.cams), L.ptr(self._geom), self.layer_num + 1, self.cap.n_poses,
                                            L.ptr(self.boxes), L.ptr(self.near_far_tab), self.frame_num,
                                            float(self.frame_offset + 1), self.time_col, L.ptr(rays), L.ptr(rgbs),
                                            L.ptr(labels), L.ptr(bbl), L.ptr(bboxes), L.ptr(nf), L.stream_ptr()),
                    "stnerf_td_batch")
        return rays, rgbs, labels, bbl, bboxes.view(B, 8, 3), nf

    def keys(self, idx) -> Dict[str, np.ndarray]:
        """Host view of pool entries: layer, frame id, camera, pixel row / col, rgb, label."""
        e = self.pool[torch.as_tensor(idx, device=self.device).long()].cpu().numpy().view(np.uint32)
        g = np.asarray(self.geom_of_layer)[e[:, 3]]
        W = np.array([self.geometries[k][1] for k in range(len(self.geometries))])[g]
        z = e[:, 2]
        return dict(layer=e[:, 3].astype(np.int64), frame=(e[:, 1] >> 16).astype(np.int64) + self.frame_offset + 1,
                    camera=(e[:, 1] & 0xffff).astype(np.int64), row=(e[:, 0] // W).astype(np.int64),
                    col=(e[:, 0] % W).astype(np.int64),
                    rgb=np.stack([z & 255, (z >> 8) & 255, (z >> 16) & 255], 1).astype(np.uint8),
                    label=(z >> 24).astype(np.uint8))

    def apply_to(self, model):
        """render/layered_neural_renderer.py:107-108: the background box and the (frame, layer) box table."""
        model.set_bkgd_bbox(self.bkgd_bbox)
        model.set_bboxes(self.bboxes)
        return model


class RayLoader:
    """`DataLoader(dataset, batch_size=B, shuffle=True)` over the device pool: one device `torch.randperm` per epoch from a
    seeded generator, consecutive slices of it, a last partial batch."""

    def __init__(self, dataset: TrainRayDataset, batch_size: int, seed: Optional[int] = None):
        self.dataset, self.batch_size = dataset, int(batch_size)
        if self.batch_size < 1:
            raise ValueError("batch size must be >= 1")
        self.generator = torch.Generator(device=dataset.device)
        self.generator.manual_seed(torch.initial_seed() if seed is None else int(seed))

    def __len__(self):
        return math.ceil(len(self.dataset) / self.batch_size)

    def epoch_order(self) -> torch.Tensor:
        n = len(self.dataset)
        dt = torch.int32 if n < 2 ** 31 else torch.int64
        return torch.randperm(n, generator=self.generator, device=self.dataset.device, dtype=dt)

    def __iter__(self):
        perm = self.epoch_order()
        for i in range(0, perm.shape[0], self.batch_size):
            yield self.dataset.items(perm[i:i + self.batch_size])


def make_ray_data_loader(cfg, is_train: bool = True, device="cuda", seed: Optional[int] = None):
    """data/build.py:13-27 -> (loader, dataset); batch size SOLVER.IMS_PER_BATCH."""
    if not is_train:
        raise NotImplementedError("make_ray_data_loader builds the training set; use make_ray_data_loader_view for views")
    ds = TrainRayDataset(cfg, device=device)
    return RayLoader(ds, cfg.SOLVER.IMS_PER_BATCH, seed), ds


# ---------------------------------------------------------------------------------------------------------------------
# validation views
# ---------------------------------------------------------------------------------------------------------------------
def sample_label_bbox(image, label, K, T, bbox=None, bboxes=None):
    """utils/ray_sampling.py:75-192 with the rays generated and the pixels chosen on the device; returns on image's device."""
    _, H, W = image.shape
    dev = torch.device("cuda") if not image.is_cuda else image.device
    rect = None if bbox is None else box_rectangle(torch.as_tensor(bbox).reshape(8, 3).cpu(), K.cpu(), T.cpu(), H, W)
    lab = label.to(dev, torch.float32).reshape(H, W)
    if rect is None:
        idx = torch.arange(H * W, device=dev)
    else:
        idx = select_pixels(lab, 0, rect).long()
    rays = ops.generate_rays(K.cpu(), T.cpu(), H, W, device=dev)[idx]
    ray_mask = torch.zeros(H * W, device=dev, dtype=label.dtype)
    ray_mask[idx] = 1.0
    labels = lab.reshape(-1)[idx].reshape(-1, 1).to(label.dtype)
    rgbs = image.to(dev).reshape(3, -1)[:, idx].permute(1, 0)
    out = [rays, labels, rgbs, ray_mask.reshape(H, W, 1)]
    if bboxes is not None:
        lb = torch.zeros(rays.shape[0], 8, 3, device=dev)
        for i, b in enumerate(bboxes):
            lb[(labels == i).squeeze(-1)] = torch.as_tensor(b, dtype=torch.float32).to(dev)
        out.append(lb)
    return tuple(t.to(image.device) for t in out)


def sample_label_label(image, label, K, T, label0):
    """utils/ray_sampling.py:194-240 with the rays generated and the pixels chosen on the device; returns on image's device."""
    _, H, W = image.shape
    dev = torch.device("cuda") if not image.is_cuda else image.device
    lab = label.to(dev).reshape(H, W)
    idx = select_pixels(lab if lab.dtype == torch.uint8 else lab.to(torch.float32), int(label0)).long()
    rays = ops.generate_rays(K.cpu(), T.cpu(), H, W, device=dev)[idx]
    ray_mask = torch.zeros(H * W, device=dev, dtype=label.dtype)
    ray_mask[idx] = 1.0
    labels = lab.reshape(-1)[idx].reshape(-1, 1)
    rgbs = image.to(dev).reshape(3, -1)[:, idx].permute(1, 0)
    return tuple(t.to(image.device) for t in (rays, labels, rgbs, ray_mask.reshape(H, W, 1)))


class ViewDataset:
    """Ray_Dataset_View (ray_dataset.py:85-201) at SIZE_TEST: `__getitem__` draws a frame and an unmasked view with np.random
    and returns the 8-tuple the evaluator unpacks (engine/layered_trainer.py:20), its rays generated on the device."""

    def __init__(self, cfg, device="cuda"):
        _check_cfg(cfg)
        M = cfg.MODEL
        self.device = torch.device(device)
        self.cap = _Capture(cfg)
        self.layer_num, self.frame_num, self.frame_offset = self.cap.layer_num, self.cap.frame_num, self.cap.frame_offset
        self.camera_num = self.cap.camera_num
        self.size_hw = _hw(cfg.INPUT.SIZE_TEST)
        self.time_col = bool(getattr(M, "USE_DEFORM_TIME", False) or getattr(M, "USE_SPACE_TIME", False))

    def __len__(self):
        return 1

    def _image(self, cam: int, slot: int):
        d = self.cap.fl[0][slot]
        p = image_path(d.image_path, cam)
        if p is None:
            raise ValueError("missing image for camera %d under %s" % (cam, d.image_path))
        lp = label_path(os.path.join(os.path.dirname(d.image_path), "labels"), cam)
        rgb, lbl, size = decode(p, lp, self.size_hw)
        if lbl is None:                                             # layer 0's full label map (frame_dataset.py:283)
            lbl = constant_label(0, size, self.size_hw)
            if lbl is None:
                lbl = np.zeros(self.size_hw, dtype=np.uint8)
        return rgb, lbl, size[1]

    def get_fixed_image(self, index_view: int, index_frame: int):
        """The 8-tuple of view `index_view` at frame slot `index_frame` (what ray_dataset.py:117-154 means to return)."""
        cam = self.cap.camera_id(int(index_view))
        rgb, lbl, height = self._image(cam, index_frame)
        K, T = transform_camera(self.cap.Ks[cam], self.cap.Ts[cam], height, self.size_hw)
        # to_tensor on the host: a CUDA division by a scalar multiplies by its reciprocal and rounds differently
        image = torch.from_numpy(rgb).permute(2, 0, 1).float().div(255).to(self.device)
        label = (torch.from_numpy(lbl).float()[None].div(255) * 255.0).to(self.device)
        bboxes = [self.cap.fl[l][index_frame].bbox for l in range(self.layer_num + 1)]
        bboxes = [torch.zeros(8, 3) if b is None else b for b in bboxes]
        rays, labels, rgbs, ray_mask, layered = sample_label_bbox(image, label, K, T, bboxes=bboxes)
        if self.time_col:
            fid = torch.full((rays.shape[0], 1), float(index_frame + self.frame_offset + 1), device=rays.device)
            rays = torch.cat([rays, fid], dim=-1)
        # the loop variable of ray_dataset.py:174-184 leaks: near_far is the LAST layer's
        nf = self.cap.near_far(self.layer_num, index_frame, cam).to(self.device)
        return rays, rgbs, labels, image, label, ray_mask, layered, nf.repeat(rays.shape[0], 1)

    def __getitem__(self, index):
        index_frame = np.random.randint(0, self.frame_num)
        index_view = np.random.randint(0, self.camera_num)
        while self.cap.mask[self.cap.camera_id(index_view)] == 0:
            index_view = np.random.randint(0, self.camera_num)
        return self.get_fixed_image(index_view, index_frame)


def make_ray_data_loader_view(cfg, is_train: bool = False, device="cuda"):
    """data/build.py:29-42 -> (loader, dataset); the loader yields the dataset's one item per epoch with a batch axis."""
    ds = ViewDataset(cfg, device=device)

    class _Loader:
        def __len__(self):
            return 1

        def __iter__(self):
            yield tuple(t.unsqueeze(0) for t in ds[0])

    return _Loader(), ds
