"""`LayeredNeuralRenderer` over the native path: the object the reference's demos drive (render/layered_neural_renderer.py).

Same constructor and public methods, assembled from the pieces of this package instead of the reference's dataset / yacs /
imageio stack:

    __init__(cfg, scale, shift, rotation, s_shift, s_scale, s_alpha)   :19-94     load_dataset_model          :96-121
    render_pose                                                          :364-392   render_path                 :401-488
    set_smooth_path_poses / load_path_poses / retime_by_key_frames /     (CameraPath: camera_path.py)
    set_frame_duration / set_pose_duration / invert_poses
    set_path_gt_poses :171-186   set_path_fixed_gt_poses :188-228   hide_layer / show_layer :653-664
    set_save_dir :643   set_fps :646   save_video :624-641   save_poses :620   zoom_in :731-738   set_near :740-741
    get_center_frame_layer :649

`cfg` is any attribute bag with the fields the reference reads: `OUTPUT_DIR` (newest `layered_rfnr_checkpoint_<n>.pt` is
loaded from it, through the packed-weight cache), `DATASETS.{TRAIN, LAYER_NUM, FRAME_NUM, FRAME_OFFSET, SCALE, FIXED_NEAR,
FIXED_FAR, CAMERA_NUM}`, `INPUT.SIZE_TEST`, `MODEL.*`.  Differences, all on the IO side: frames are written with Pillow
(`color/<n>.jpg`, `depth/<n>.png`, floats clipped to [0,1] and scaled to 8 bits as imageio does); `save_video` needs imageio
and otherwise leaves the frame folders; the rays of a pose are generated on the device and a frame is one native call, with
the device->host copy of frame i overlapping the rendering of frame i+1 (PoseRenderer).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from stnerf_b200.camera_path import CameraPath
from stnerf_b200.checkpoint_io import get_iteration_path, load_checkpoint_cached
from stnerf_b200.pose_renderer import PoseRenderer
from stnerf_b200.scene_data import RenderDataset


def _to_u8(img: torch.Tensor) -> np.ndarray:
    a = img.detach().cpu().numpy()
    return (np.clip(a, 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8)


def _imwrite(path: str, img: torch.Tensor):
    from PIL import Image
    a = _to_u8(img)
    if a.ndim == 3 and a.shape[2] == 1:
        a = a[..., 0]
    Image.fromarray(a).save(path, quality=95) if path.endswith(".jpg") else Image.fromarray(a).save(path)


class LayeredNeuralRenderer(CameraPath):
    def __init__(self, cfg, scale=None, shift=None, rotation=None, s_shift=None, s_scale=None, s_alpha=None):
        self.alpha = None
        self.cfg, self.scale, self.shift, self.rotation = cfg, scale, shift, rotation
        if s_shift is not None:
            self.shift = s_shift[0]
        if s_scale is not None:
            self.scale = s_scale[0]
        if s_alpha is not None:
            self.alpha = s_alpha[0]
        self.dataset_dir = cfg.OUTPUT_DIR
        self.output_dir = os.path.join(cfg.OUTPUT_DIR, "rendered")
        self.dataset, self.model = self.load_dataset_model()
        D = cfg.DATASETS
        super().__init__(self.dataset.poses.numpy(), [k.numpy() for k in self.dataset.Ks], D.LAYER_NUM, D.FRAME_NUM,
                         getattr(D, "FRAME_OFFSET", 0), s_shift, s_scale, s_alpha)
        self.far = 20.0
        self.frame_num, self.fps = D.FRAME_NUM, 25
        self.height, self.width = cfg.INPUT.SIZE_TEST[1], cfg.INPUT.SIZE_TEST[0]
        self.images, self.depths = [], []
        self.image_num = self.save_count = 0
        self.trace_layer = -1
        self.dir_name = ""
        self._pose_renderer = PoseRenderer(self.model, self.dataset.height, self.dataset.width, self.far)

    # ---- :96-121 ------------------------------------------------------------------------------------------------------
    def load_dataset_model(self):
        import modeling
        cfg, D = self.cfg, self.cfg.DATASETS
        para_file = get_iteration_path(self.dataset_dir)
        if para_file is None:
            raise FileNotFoundError("no layered_rfnr_checkpoint_<iter>.pt under %s" % self.dataset_dir)
        dataset = RenderDataset(D.TRAIN, D.LAYER_NUM, D.FRAME_NUM, getattr(D, "FRAME_OFFSET", 0), cfg.INPUT.SIZE_TEST,
                                getattr(D, "SCALE", 1.0), getattr(D, "FIXED_NEAR", -1.0), getattr(D, "FIXED_FAR", -1.0),
                                getattr(D, "CAMERA_NUM", 0), getattr(D, "ORIGINAL_SIZE", None),
                                use_time=cfg.MODEL.USE_DEFORM_TIME or cfg.MODEL.USE_SPACE_TIME)
        model = modeling.build_layered_model(cfg, dataset.camera_num, scale=self.scale, shift=self.shift)
        dataset.apply_to(model)
        load_checkpoint_cached(model, para_file)
        if self.alpha is not None:
            model.alpha = self.alpha
        if torch.cuda.is_available():          # (a host without a device can still script paths; rendering raises StnerfError)
            model.cuda()
        return dataset, model

    def set_rotation(self, rotation):
        """Rotate layers: one entry per layer incl. the background, each None, a 3x3 matrix, a rotation vector (axis * angle,
        radians) or (R, centre) (stnerf_b200.rotation).  The constructor's `rotation` is stored and unused, as in the
        reference; this is the call that turns performers."""
        self.model.rotation = rotation

    # ---- layer display: renderer and model stay in step (:653-664) ----------------------------------------------------------
    def hide_layer(self, layer_id):
        self.model.hide_layer(layer_id)
        self.display_layers[layer_id] = 0

    def show_layer(self, layer_id):
        self.model.show_layer(layer_id)
        self.display_layers[layer_id] = 1

    # ---- the remaining path constructors (:171-228) ----------------------------------------------------------------------------
    def set_path_gt_poses(self):
        poses = [self.dataset.poses[i] for i in range(self.dataset.poses.shape[0])]
        self.poses = self.poses + poses
        self.Ks = self.Ks + list(self.gt_Ks)
        self._append_layer_frame_pairs(len(poses))

    def set_path_fixed_gt_poses(self, id, num=None):
        if self.s_shift is not None:
            s0, s1 = np.array(self.s_shift[0]), np.array(self.s_shift[1])
            shift_step = (s1 - s0) / (num - 1)
            self.s_shift_frame = []
        if self.s_scale is not None:
            c0, c1 = np.array(self.s_scale[0]), np.array(self.s_scale[1])
            scale_step = (c1 - c0) / (num - 1)
            self.s_scale_frame = []
        poses, Ks = [], []
        for i in range(num):
            poses.append(self.dataset.poses[id])
            Ks.append(self.dataset.Ks[id])
            if self.s_shift is not None:
                self.s_shift_frame.append((s0 + i * shift_step).tolist())
            if self.s_scale is not None:
                self.s_scale_frame.append((c0 + i * scale_step).tolist())
        self.poses = self.poses + poses
        self.Ks = self.Ks + Ks
        self._append_layer_frame_pairs(len(poses))

    # ---- :364-392 -------------------------------------------------------------------------------------------------------------
    def render_pose(self, pose, K, layer_frame_pair, density_threshold=0, bkgd_density_threshold=0):
        return self._pose_renderer.render_pose(pose, K, layer_frame_pair, density_threshold, bkgd_density_threshold)

    # ---- :401-488 -------------------------------------------------------------------------------------------------------------
    def _video_dir(self, leaf):
        parts = [self.output_dir] + ([self.dir_name] if self.dir_name else []) + ["video_%d" % self.save_count, str(leaf)]
        d = os.path.join(*parts)
        if not os.path.exists(d):
            os.makedirs(os.path.join(d, "color"))
            os.makedirs(os.path.join(d, "depth"))
        return d

    def render_path(self, inverse_y_axis=False, density_threshold=0, bkgd_density_threshold=0, auto_save=True):
        save_dir = self._video_dir("mixed")
        with open(os.path.join(save_dir, "poses"), "w") as f:
            for pose in self.poses:
                f.write(str(pose) + "\n")
        with open(os.path.join(save_dir, "Ks"), "w") as f:
            for K in self.Ks:
                f.write(str(K) + "\n")
        self.images, self.depths = [], []
        self.images_layer = [[] for _ in range(self.layer_num + 1)]
        self.depths_layer = [[] for _ in range(self.layer_num + 1)]
        self.image_num = 0
        frames = self._pose_renderer.render_path(self.poses, self.Ks, self.layer_frame_pairs, density_threshold,
                                                 bkgd_density_threshold, self.per_frame_state())
        for color, depth, color_layer, depth_layer in frames:
            if inverse_y_axis:
                color, depth = torch.flip(color, [0]), torch.flip(depth, [0])
                color_layer = [torch.flip(i, [0]) for i in color_layer]
                depth_layer = [torch.flip(i, [0]) for i in depth_layer]
            if auto_save:
                d = self._video_dir("mixed")
                _imwrite(os.path.join(d, "color", "%d.jpg" % self.image_num), color)
                _imwrite(os.path.join(d, "depth", "%d.png" % self.image_num), depth)
                self.images.append(color)
                self.depths.append(depth)
                for layer_id in range(self.layer_num + 1):
                    if self.is_shown_layer(layer_id):
                        d = self._video_dir(layer_id)
                        _imwrite(os.path.join(d, "color", "%d.jpg" % self.image_num), color_layer[layer_id])
                        _imwrite(os.path.join(d, "depth", "%d.png" % self.image_num), depth_layer[layer_id])
                        self.images_layer[layer_id].append(color)       # the reference appends the MIXED image here (:484-485)
                        self.depths_layer[layer_id].append(depth)
            self.image_num += 1

    # ---- :550-618 (flat folder layout + the layer-2-over-background composite "02") --------------------------------------------
    def render_path_walking(self, inverse_y_axis=False, density_threshold=0, bkgd_density_threshold=0, auto_save=True):
        self.images, self.depths = [], []
        self.images_layer = [[] for _ in range(self.layer_num + 1)]
        self.depths_layer = [[] for _ in range(self.layer_num + 1)]
        self.image_num = 0

        def folder(leaf, depth=True):
            d = os.path.join(self.output_dir, str(leaf))
            if not os.path.exists(d):
                os.makedirs(os.path.join(d, "color"))
                if depth:
                    os.makedirs(os.path.join(d, "depth"))
            return d

        frames = self._pose_renderer.render_path(self.poses, self.Ks, self.layer_frame_pairs, density_threshold, bkgd_density_threshold)
        for color, depth, color_layer, depth_layer in frames:
            if inverse_y_axis:
                color, depth = torch.flip(color, [0]), torch.flip(depth, [0])
                color_layer = [torch.flip(i, [0]) for i in color_layer]
                depth_layer = [torch.flip(i, [0]) for i in depth_layer]
            if auto_save:
                d = folder("mixed")
                _imwrite(os.path.join(d, "color", "%d.jpg" % self.image_num), color)
                _imwrite(os.path.join(d, "depth", "%d.png" % self.image_num), depth)
                self.images.append(color)
                self.depths.append(depth)
                for layer_id in range(self.layer_num + 1):
                    d = folder(layer_id)
                    _imwrite(os.path.join(d, "color", "%d.jpg" % self.image_num), color_layer[layer_id])
                    _imwrite(os.path.join(d, "depth", "%d.png" % self.image_num), depth_layer[layer_id])
                    self.images_layer[layer_id].append(color)
                    self.depths_layer[layer_id].append(depth)
                color_hide = color_layer[0].clone()                     # layer 2 pasted over the background where it is nearer (:601-605)
                index = depth_layer[2] < depth_layer[0]
                index = torch.cat([index, index, index], dim=2)
                index = torch.logical_and(index, color_layer[2] != 0)
                color_hide[index] = color_layer[2][index]
                _imwrite(os.path.join(folder("02", depth=False), "color", "%d.jpg" % self.image_num), color_hide)
            self.image_num += 1

    # ---- small helpers -----------------------------------------------------------------------------------------------------------
    def save_poses(self, path):
        np.save(path, self.poses)

    def save_video(self):
        if len(self.images) == 0:
            print("Warning: Cannot generate video for all rendered images, data is empty.")
            return
        video_dir = os.path.join(*([self.output_dir] + ([self.dir_name] if self.dir_name else []) + ["video"]))
        os.makedirs(video_dir, exist_ok=True)
        try:
            import imageio
        except ImportError:
            print("imageio is not installed: no .mp4 written; the frames are under %s" % os.path.dirname(video_dir))
            self.save_count += 1
            return
        imageio.mimwrite(video_dir + "/color_%d.mp4" % self.save_count, [_to_u8(i) for i in self.images], fps=self.fps, quality=8)
        imageio.mimwrite(video_dir + "/depth_%d.mp4" % self.save_count, [_to_u8(i) for i in self.depths], fps=self.fps, quality=8)
        self.save_count += 1

    def set_save_dir(self, dir_name): self.dir_name = dir_name
    def set_fps(self, fps): self.fps = fps
    def set_trace_layer(self, layer_id): self.trace_layer = layer_id
    def set_near(self, near): self.model.near = near

    def get_center_frame_layer(self, frame_id, layer_id):
        return self.dataset.datasets[layer_id][frame_id].center

    def zoom_in(self, layer_id, frame_id, scale):
        center = np.asarray(self.dataset.datasets[layer_id][frame_id].center, dtype=np.float32)
        for idx in range(self.gt_poses.shape[0]):              # in place: later smooth paths start from the moved cameras
            self.gt_poses[idx, :3, 3] = center + 1 / scale * (self.gt_poses[idx, :3, 3] - center)
