"""`LayeredRFRender`-compatible model object over the native renderer.

Mirrors the call surface of the reference class (modeling/layered_rfrender.py:19-141): constructor fields,
`set_bboxes` / `set_bkgd_bbox` / `hide_layer` / `show_layer`, the mutable `shift` / `scale` / `alpha` / `near`
attributes the renderer writes between frames (render/layered_neural_renderer.py:435-440), `state_dict` key
names (SURVEY App. B) and the 5-tuple returned by `forward`.  The arithmetic lives in libstnerf_b200.so.

Host-side work done here is only the per-call prologue of forward (layered_rfrender.py:151-242): ray-layout
parse, frame-lerped boxes taken from ray 0, the scale/shift edits of the boxes and the edit flags.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import List, Optional

import torch

from . import _lib as L
from . import rotation as ROT
from .native import NativeRenderer, split_planes

_SPACE_SHAPES = [("stage1.0", 256, 63), ("stage1.2", 256, 256), ("stage1.4", 256, 256), ("stage1.6", 256, 256),
                 ("stage2.0", 256, 319), ("stage2.2", 256, 256), ("stage2.4", 256, 256), ("density_net.0", 1, 256),
                 ("rgb_net.1", 128, None), ("rgb_net.3", 3, 128)]
_MOTION_SHAPES = [("motion_net.0", 128, 84), ("motion_net.2", 128, 128), ("motion_net.4", 128, 128),
                  ("motion_net.6", 128, 128), ("motion_net.8", 128, 128), ("motion_net.10", 3, 128)]


def _linear_init(out_f: int, in_f: int):
    """nn.Linear's default init (kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(in), 1/sqrt(in)) for both tensors)."""
    b = 1.0 / math.sqrt(in_f)
    return torch.empty(out_f, in_f).uniform_(-b, b), torch.empty(out_f).uniform_(-b, b)


def fresh_state_dict(layer_num: int, use_space_time: bool, bkgd_use_space_time: bool = False) -> "OrderedDict":
    """Randomly initialised weights with the reference's key order (modeling/layered_rfrender.py:59-90)."""
    sd = OrderedDict()

    def space(prefix, use_time):
        for name, o, i in _SPACE_SHAPES:
            i = i if i is not None else 256 + 27 + (21 if use_time else 0)
            sd[prefix + name + ".weight"], sd[prefix + name + ".bias"] = _linear_init(o, i)

    def clone(src, dst):
        for k in [k for k in sd if k.startswith(src)]:
            sd[dst + k[len(src):]] = sd[k].clone()

    space("bkgd_spacenet.", bkgd_use_space_time)
    clone("bkgd_spacenet.", "bkgd_spacenet_fine.")                       # deepcopy (:63)
    for i in range(layer_num):
        if i == 0:
            space("spacenets.0.", use_space_time)
        else:
            clone("spacenets.0.", "spacenets.%d." % i)                   # (:69)
    for i in range(layer_num):
        clone("spacenets.%d." % i, "spacenets_fine.%d." % i)             # (:73)
    for i in range(layer_num):
        for name, o, k in _MOTION_SHAPES:
            sd["time_deform_nets.%d.%s.weight" % (i, name)], sd["time_deform_nets.%d.%s.bias" % (i, name)] = \
                _linear_init(o, k)
    # registration order of the reference module (ModuleLists first, :59-93) == key order of the shipped checkpoints
    order = ["spacenets.", "spacenets_fine.", "bkgd_spacenet.", "bkgd_spacenet_fine.", "time_deform_nets."]
    return OrderedDict((k, sd[k]) for pre in order for k in sd if k.startswith(pre))


class LayeredRFRender(torch.nn.Module):
    """Drop-in for modeling.layered_rfrender.LayeredRFRender at render time (BBOX sampling, retiming rays)."""

    def __init__(self, cfg, camera_num=0, scale=None, shift=None, precision: Optional[str] = None, rotation=None):
        super().__init__()
        M = cfg.MODEL
        if M.SAMPLE_METHOD != "BBOX":
            raise NotImplementedError("SAMPLE_METHOD=%r: only 'BBOX' is usable in the reference (SURVEY A.9)" % M.SAMPLE_METHOD)
        for flag in ("POSE_REFINEMENT", "USE_DEFORM_VIEW", "BKGD_USE_DEFORM_TIME", "SAME_SPACENET"):
            if getattr(M, flag, False):
                raise NotImplementedError("cfg.MODEL.%s=True is not part of the native hot path (disabled in every shipped config)" % flag)
        if getattr(M, "DEEP_RGB", False) and M.USE_SPACE_TIME:
            raise NotImplementedError("DEEP_RGB head is not used by any shipped checkpoint")
        if not M.USE_DEFORM_TIME or not M.USE_DIR or not M.TKERNEL_INC_RAW:
            raise NotImplementedError("the native path implements USE_DEFORM_TIME=USE_DIR=TKERNEL_INC_RAW=True (both shipped configs)")
        self.layer_num = int(cfg.DATASETS.LAYER_NUM)
        self.camera_num = camera_num
        self.coarse_ray_sample = int(M.COARSE_RAY_SAMPLING)
        self.fine_ray_sample = int(M.FINE_RAY_SAMPLING)
        self.sample_method = M.SAMPLE_METHOD
        self.boarder_weight = float(M.BOARDER_WEIGHT)
        self.use_space_time = bool(M.USE_SPACE_TIME)
        self.bkgd_use_space_time = bool(M.BKGD_USE_SPACE_TIME)
        self.use_deform_time = True
        self.scale, self.shift = scale, shift
        self.rotation = rotation          # per layer: None, 3x3 matrix, rotation vector or (R, centre) (stnerf_b200.rotation)
        self.near, self.alpha = 0, 1
        self.precision = precision or getattr(M, "B200_PRECISION", "exact")
        self.chunk_rays = int(getattr(M, "B200_CHUNK_RAYS", 0))
        self.display_layers = {i: 1 for i in range(self.layer_num + 1)}
        self._sd = fresh_state_dict(self.layer_num, self.use_space_time, self.bkgd_use_space_time)
        self._native: Optional[NativeRenderer] = None
        self._uploaded = False
        self._inject = None
        self.seed = 0
        self.bboxes = None
        self.bkgd_bbox = None
        self.retiming = True

    # ---- nn.Module-ish surface used by render/layered_neural_renderer.py:105-121 ------------------------------
    def state_dict(self, *a, **k):
        if getattr(self, "_packed", None) is not None and getattr(self, "_sd_source", None) is not None:
            src, self._sd_source = self._sd_source, None
            for k_, v in src().items():                                   # lazily materialise the tensors behind a packed image
                if k_ in self._sd:
                    self._sd[k_] = v.detach().to("cpu", torch.float32).clone()
        return OrderedDict((k_, v) for k_, v in self._sd.items())

    def load_state_dict(self, sd, strict=True):
        missing = [k for k in self._sd if k not in sd]
        unexpected = [k for k in sd if k not in self._sd]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict: missing %s unexpected %s" % (missing[:4], unexpected[:4]))
        for k in self._sd:
            if k in sd:
                if tuple(sd[k].shape) != tuple(self._sd[k].shape):
                    raise RuntimeError("size mismatch for %s: %s vs %s" % (k, tuple(sd[k].shape), tuple(self._sd[k].shape)))
                self._sd[k] = sd[k].detach().to("cpu", torch.float32).clone()
        self._uploaded = False
        self._packed = None
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def load_packed(self, image: bytes, state_dict_source=None):
        """Take the networks from a packed-weight image (NativeRenderer.export_weights) instead of a state_dict.
        `state_dict_source`: optional zero-argument callable returning the matching state_dict, used only if someone asks
        this model for `state_dict()` later (the render path never does)."""
        self._packed = bytes(image)
        self._sd_source = state_dict_source
        self._uploaded = False

    def export_packed(self, device=None) -> bytes:
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        with torch.cuda.device(dev):
            return self._ensure_native(dev).export_weights()

    def cuda(self, device=None):
        self._device = torch.device("cuda", torch.cuda.current_device() if device is None else device) \
            if not isinstance(device, torch.device) else device
        return self

    def hide_layer(self, layer_id): self.display_layers[layer_id] = 0
    def show_layer(self, layer_id): self.display_layers[layer_id] = 1
    def is_shown_layer(self, layer_id): return self.display_layers[layer_id] == 1
    def set_bkgd_bbox(self, bbox): self.bkgd_bbox = bbox
    def set_bboxes(self, bboxes): self.bboxes = bboxes
    def set_bkgd_near_far(self, near_far): self.bkgd_near_torchfar = near_far       # same typo'd attribute (:120-121)
    def set_max_min(self, maxs, mins): self.maxs, self.mins = maxs, mins
    def set_precision(self, precision):
        self.precision = precision
        if self._native is not None:
            self._native.set_precision(precision)

    def inject_uniforms(self, jitter, u):
        """Parity hook: use these uniforms for the next forward instead of the in-kernel Philox stream.
        jitter (l,N,n1) replaces torch.rand of layers/RaySamplePoint.py:98, u (l,N,n2) that of utils/sample_pdf.py:31."""
        self._inject = (jitter, u)

    # ---- host prologue (layered_rfrender.py:190-242) -------------------------------------------------------------
    def bbox_interpolation(self, float_frame_id, layer_id):
        start = self.bboxes[math.floor(float_frame_id), layer_id]
        end = self.bboxes[math.ceil(float_frame_id), layer_id]
        return torch.lerp(start, end, float_frame_id - math.floor(float_frame_id))

    def _edit_boxes(self, boxes, table, bk):
        """Scale / shift edits of one set of boxes (l,8,3) about the pivot of the FIRST table row (layered_rfrender.py:216-242).
        Returns the min corners (l,3), max corners (l,3) and the pivot."""
        l = self.layer_num + 1
        first = torch.cat([bk, table[0]], 0)                              # (:216-220)
        centre = first.mean(1)
        centre[:, 2] = first[:, 1, 2]                                     # (:226)
        pivot = torch.zeros(3)
        if self.scale is not None:
            if l < 3:
                raise IndexError("scale edits need at least two performer layers (layered_rfrender.py:232)")
            pivot = (centre[2] + centre[1]) / 2
            for i in range(len(self.scale)):
                boxes[i] = (boxes[i] - pivot) * self.scale[i] + pivot     # (:230-232)
        if self.shift is not None:
            for i in range(len(self.shift)):
                if self.shift[i] is None:
                    continue
                boxes[i] = boxes[i] + torch.tensor(self.shift[i], dtype=torch.float32)   # (:237-242)
        # the kernels take min / max corners; the reference indexes corners 0,6 (and 1..5,7 for the same planes)
        lo, hi = boxes[:, 0, :], boxes[:, 6, :]
        ref = torch.stack([torch.stack([lo[:, 0], lo[:, 1], lo[:, 2]], -1), torch.stack([hi[:, 0], lo[:, 1], lo[:, 2]], -1),
                           torch.stack([hi[:, 0], hi[:, 1], lo[:, 2]], -1), torch.stack([lo[:, 0], hi[:, 1], lo[:, 2]], -1),
                           torch.stack([lo[:, 0], lo[:, 1], hi[:, 2]], -1), torch.stack([hi[:, 0], lo[:, 1], hi[:, 2]], -1),
                           torch.stack([hi[:, 0], hi[:, 1], hi[:, 2]], -1), torch.stack([lo[:, 0], hi[:, 1], hi[:, 2]], -1)], 1)
        if not torch.equal(ref, boxes):
            raise ValueError("bounding boxes must be axis-aligned with the corner order of data/datasets/frame_dataset.py:187-188")
        return lo, hi, pivot

    def _box_table(self) -> torch.Tensor:
        """(F, l, 2, 3): min / max corners of every layer at every frame after the edits -- what a ray of frame f gets from
        `self.bboxes.index_select(0, frame_id - 1)` (layered_rfrender.py:193) followed by :207-242 (row f-1)."""
        table = self.bboxes.detach().to("cpu", torch.float32)
        bk = self.bkgd_bbox.detach().to("cpu", torch.float32).reshape(1, 8, 3)
        rows = []
        for f in range(table.shape[0]):
            lo, hi, _ = self._edit_boxes(torch.cat([bk, table[f]], 0).clone(), table, bk)
            rows.append(torch.stack([lo, hi], 1))
        return torch.stack(rows, 0)

    def _resolve_scene(self, frame_ids_row0, density_threshold, bkgd_density_threshold) -> L.Scene:
        l = self.layer_num + 1
        if self.bboxes is None or self.bkgd_bbox is None:
            raise RuntimeError("set_bboxes / set_bkgd_bbox must be called before rendering")
        table = self.bboxes.detach().to("cpu", torch.float32)
        bk = self.bkgd_bbox.detach().to("cpu", torch.float32).reshape(1, 8, 3)
        self.bboxes = table                                               # what .cuda() would have kept on the model
        boxes = [bk[0].clone()]
        for i in range(self.layer_num):
            if self.retiming:
                f = torch.tensor(float(frame_ids_row0[i + 1]), dtype=torch.float32) - 1       # (:200)
                boxes.append(self.bbox_interpolation(f, i))
            else:                                                         # index_select(int64(frame_id) - 1) (:193)
                boxes.append(table[int(float(frame_ids_row0[i + 1])) - 1, i])
        boxes = torch.stack(boxes, 0)                                     # (l,8,3)
        lo, hi, pivot = self._edit_boxes(boxes, table, bk)
        sc = L.Scene()
        for i in range(l):
            for a in range(3):
                sc.bmin[i][a], sc.bmax[i][a] = float(lo[i, a]), float(hi[i, a])
            sc.shown[i] = 1 if self.display_layers.get(i, 1) == 1 else 0
            sh_given = self.shift is not None
            if sh_given and len(self.shift) < l:
                raise IndexError("shift must have one entry per layer incl. background (layered_rfrender.py:468)")
            entry = self.shift[i] if sh_given else None
            sc.shift_on[i] = 1 if entry is not None else 0
            if entry is not None:
                sv = torch.tensor(entry, dtype=torch.float32)
                for a in range(3):
                    sc.shift[i][a] = float(sv[a])
            sc_given = self.scale is not None
            if sc_given and len(self.scale) < l:
                raise IndexError("scale must have one entry per layer incl. background (layered_rfrender.py:475)")
            sc.scale_coarse_on[i] = 1 if sc_given else 0                                  # (:300-303)
            sc.scale_fine_on[i] = 1 if (sc_given and not (sh_given and entry is None)) else 0   # `continue` at :468-469
            sc.scale[i] = float(torch.tensor(float(self.scale[i]), dtype=torch.float32)) if sc_given else 1.0
        for a in range(3):
            sc.pivot[a] = float(pivot[a])
        sc.near_plane = float(self.near)
        sc.alpha_layer2 = float(self.alpha)
        sc.density_threshold = float(density_threshold)
        sc.bkgd_density_threshold = float(bkgd_density_threshold)
        sc.boarder_weight = self.boarder_weight
        sc.apply_thresholds = 1 if self.retiming else 0
        sc.shared_frame_id = 0 if self.retiming else 1
        return sc

    def _rotation_entries(self):
        """Every layer's parsed rotation (stnerf_b200.rotation.resolve): None or (R float32 (3,3), centre or None)."""
        return ROT.resolve(self.rotation, self.layer_num + 1)

    def _upload_rotation(self, nat) -> bytes:
        """Set the model's rotation on the context (centres left to the library are each call's box centres).  Returns a key
        that changes exactly when what was uploaded does."""
        entries = self._rotation_entries()
        if all(e is None for e in entries):
            nat.set_rotation(None)
            return b""
        arrays = ROT.abi_arrays(entries)
        nat.set_rotation(*arrays)
        return b"".join(a.tobytes() for a in arrays)

    def _ensure_native(self, device):
        if self._native is None:
            with torch.cuda.device(device):
                st = [self.bkgd_use_space_time] + [self.use_space_time] * self.layer_num
                self._native = NativeRenderer(self.layer_num + 1, st, self.precision, self.chunk_rays)
        if not self._uploaded:
            with torch.cuda.device(device):
                if getattr(self, "_packed", None) is not None:
                    self._native.import_weights(self._packed)
                else:
                    self._native.load_state_dict(self._sd)
            self._uploaded = True
        return self._native

    # ---- forward (layered_rfrender.py:141) ---------------------------------------------------------------------
    def _prologue(self, rays, density_threshold, bkgd_density_threshold):
        """Ray-layout parse, scene constants and box table of one forward (layered_rfrender.py:151-242) on the context.
        Returns the context and the rays as detached fp32."""
        l = self.layer_num + 1
        width = rays.size(-1)
        if width == 7 + self.layer_num:
            self.retiming = True                                         # (:159-160)
        elif width == 7:
            # evaluator rays [o,d,frame_id] (engine/layered_trainer.py:36,383): boxes by frame id (:193), no thresholds.
            # One image per call shares its frame id; mixed-frame training batches are outside the render hot path.
            self.retiming = False                                        # (:157-158)
            per_ray_frames = not bool((rays[:, 6] == rays[0, 6]).all())  # a mixed-frame batch: boxes per ray (:193)
        else:
            raise ValueError("undefined ray format in LayeredRFRender, ray dimension is %d" % width)   # (:162-163)
        if not rays.is_cuda:
            raise L.StnerfError("rays must be CUDA tensors: the native path has no CPU fallback")
        if rays.size(0) < 2:
            raise ValueError("need more than one ray per call (layered_rfrender.py:309)")
        rays = rays.detach().to(torch.float32)
        nat = self._ensure_native(rays.device)
        frame_ids = rays[0, 6:].cpu()                                    # boxes come from ray 0 only (:195-200)
        if not self.retiming:
            frame_ids = frame_ids[:1].expand(l)                          # index_select(frame_id - 1) for every layer (:193)
        nat.set_scene(self._resolve_scene(frame_ids, density_threshold, bkgd_density_threshold))
        self._upload_rotation(nat)                                       # after the scene: default centres are its boxes'
        if width == 7 and per_ray_frames:
            ids = rays[:, 6]
            if float(ids.min()) < 1 or float(ids.max()) >= self.bboxes.shape[0] + 1:
                raise IndexError("frame id out of range for index_select(0, frame_id - 1) (layered_rfrender.py:193)")
            key = (id(self.bboxes), repr(self.scale), repr(self.shift), repr(self.rotation))
            if getattr(self, "_table_key", None) != key:
                nat.set_box_table(self._box_table())
                self._table_key = key
        elif getattr(self, "_table_key", None) is not None:
            nat.set_box_table(None)
            self._table_key = None
        return nat, rays

    def forward(self, rays, labels=None, bboxes=None, only_coarse=False, near_far=None, near_far_points=[],
                density_threshold=0.0001, bkgd_density_threshold=0):
        l = self.layer_num + 1
        nat, rays = self._prologue(rays, density_threshold, bkgd_density_threshold)
        jitter, u = self._inject if self._inject is not None else (None, None)
        self._inject = None
        self.seed += 1
        out, mask = nat.render(rays, self.coarse_ray_sample, self.fine_ray_sample, only_coarse=bool(only_coarse),
                               jitter=jitter, u=u, seed=self.seed)
        fine_mixed, coarse_mixed, fine_layer, coarse_layer = split_planes(out, l)
        if only_coarse:
            fine_mixed, fine_layer = coarse_mixed, coarse_layer          # (:721-722)
        ray_mask = [mask[i].bool() for i in range(l)]
        return fine_mixed, coarse_mixed, fine_layer, coarse_layer, ray_mask


def build_layered_model(cfg, camera_num=0, scale=None, shift=None, rotation=None):
    """modeling/__init__.py:5-7.  cfg.MODEL.B200_TRAINABLE (default False) selects the trainable model
    (stnerf_b200.train.TrainableLayeredRFRender): network parameters, a differentiable forward whose networks train in
    cfg.MODEL.B200_TRAIN_PRECISION ("fp32", the default, or "tf32x3")."""
    if bool(getattr(cfg.MODEL, "B200_TRAINABLE", False)):
        from .train import TrainableLayeredRFRender
        return TrainableLayeredRFRender(cfg, camera_num=camera_num, scale=scale, shift=shift,
                                        train_precision=getattr(cfg.MODEL, "B200_TRAIN_PRECISION", "fp32"), rotation=rotation)
    return LayeredRFRender(cfg, camera_num=camera_num, scale=scale, shift=shift, rotation=rotation)
