"""Fast path of `LayeredNeuralRenderer.render_pose` / `render_path` (SURVEY 8f row 1).

The reference builds the H*W rays of a pose on the CPU (`data/datasets/ray_dataset.py:260-283` ->
`utils/render_helpers.py:42-126`), uploads 75 MB per 1080p frame (`render/layered_neural_renderer.py:372-375`), renders
chunk by chunk and copies every image back synchronously (`:451-454`).  Here a BATCH of poses goes down in one native call
(`stnerf_render_views`): rays are generated on the device, only the fine images are produced (the coarse pass just
resamples), and on the path renderer the device->host copy of frame i overlaps the rendering of frame i+1
(`stnerf_render_views_host`).  With a process group initialised, each rank renders its interleaved rows straight into its
slot of an all-gather buffer and one in-place all-gather assembles the batch (stnerf_b200.dist).

Returned values follow `render_pose` (`render/layered_neural_renderer.py:364-392`): `color (H,W,3)`, `depth (H,W,1)`
(negative depths zeroed, divided by `far`), `color_layer` and `depth_layer` lists over the l layers -- including the
reference's quirk that the per-layer depths are zeroed where the *mixed* depth is negative (`:386-388`), which is tested
AFTER the mixed depth was clamped and scaled and therefore never fires.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from .dist import ShardedViewRenderer


class PoseRenderer:
    def __init__(self, model, height: int, width: int, far: float = 20.0, rank: int = 0, world: int = 1, batch: int = 4):
        self.model, self.H, self.W, self.far = model, int(height), int(width), float(far)
        self.rank, self.world, self.batch = rank, world, max(1, int(batch))
        self.l = model.layer_num + 1
        self._svr: Optional[ShardedViewRenderer] = None
        self._pinned = None
        self._rot_key = None          # the rotation the views made since the last native call were made with

    def _renderer(self) -> ShardedViewRenderer:
        dev = torch.device("cuda", torch.cuda.current_device())
        nat = self.model._ensure_native(dev)
        if self._svr is None:
            self._svr = ShardedViewRenderer(nat, self.H, self.W, self.model.coarse_ray_sample,
                                            self.model.fine_ray_sample, self.rank, self.world)
        return self._svr

    def frame_ids(self, layer_frame_pair: Sequence[Tuple[int, float]]) -> List[float]:
        """`frame_ids[:, layer_id] = frame_id` (data/datasets/ray_dataset.py:276-279)."""
        ids = [0.0] * self.l
        for layer_id, frame_id in layer_frame_pair:
            ids[int(layer_id)] = float(frame_id)
        return ids

    def make_view(self, pose, K, layer_frame_pair, density_threshold=0, bkgd_density_threshold=0):
        """The `stnerf_view` of one pose: camera, frame ids and the prologue of forward() for THIS frame -- boxes of the
        frame ids, the model's current shift/scale/alpha edits, thresholds (layered_rfrender.py:190-242).  render_pose goes
        through layered_batchify_ray with N >= chunk size, so the thresholds are forwarded (utils/batchify_rays.py:53-79)."""
        svr = self._renderer()
        ids = self.frame_ids(layer_frame_pair)
        self.model.retiming = True
        scene = self.model._resolve_scene(torch.tensor(ids), density_threshold, bkgd_density_threshold)
        # the rotation lives on the context, not in the view: one native call renders every view with the same one (centres
        # left to the library follow each view's boxes)
        key = self.model._upload_rotation(svr.nat)
        if self._rot_key is not None and key != self._rot_key:
            raise ValueError("model.rotation changed between the views of one batch: a per-frame rotation needs batch=1")
        self._rot_key = key
        self.model.seed += 1
        return svr.nat.make_view(K, pose, ids, scene, self.model.seed)

    @torch.no_grad()
    def render_images(self, pose, K, layer_frame_pair, density_threshold=0, bkgd_density_threshold=0) -> torch.Tensor:
        """(l+1, H, W, 5) device tensor: image 0 = mixed, 1+i = layer i; channels rgb(3), raw depth, acc."""
        return self.render_images_batch([pose], [K], [layer_frame_pair], density_threshold, bkgd_density_threshold)[0]

    @torch.no_grad()
    def render_images_batch(self, poses, Ks, layer_frame_pairs, density_threshold=0, bkgd_density_threshold=0,
                            per_frame_state=None, first_index: int = 0) -> torch.Tensor:
        """Several poses in ONE native call: (B, l+1, H, W, 5) on the device."""
        svr = self._renderer()
        views = []
        self._rot_key = None
        for j in range(len(poses)):
            if per_frame_state is not None:
                per_frame_state(first_index + j, self.model)
            views.append(self.make_view(poses[j], Ks[j], layer_frame_pairs[j], density_threshold, bkgd_density_threshold))
        return svr.assembled(svr.render(views))

    def render_pose(self, pose, K, layer_frame_pair, density_threshold=0, bkgd_density_threshold=0):
        """Same return value as LayeredNeuralRenderer.render_pose (render/layered_neural_renderer.py:364-392)."""
        img = self.render_images(pose, K, layer_frame_pair, density_threshold, bkgd_density_threshold)
        return self._post(img)

    def _post(self, img: torch.Tensor):
        color = img[0, ..., :3]
        depth = img[0, ..., 3:4].clone()
        depth[depth < 0] = 0                                         # :382
        depth = depth / self.far                                     # :383
        color_layer = [img[1 + i, ..., :3] for i in range(self.l)]   # :384
        depth_layer = []
        for i in range(self.l):
            d1 = img[1 + i, ..., 3:4].clone()
            d1[depth < 0] = 0        # quirk kept: tests the (already clamped, scaled) mixed depth -> never true (:387)
            depth_layer.append(d1 / self.far)
        return color, depth, color_layer, depth_layer

    def render_path(self, poses, Ks, layer_frame_pairs, density_threshold=0, bkgd_density_threshold=0,
                    per_frame_state=None):
        """Generator over the frames of a camera path (`render_path`, :401-488, without the file IO).  Yields CPU tensors
        `(color, depth, color_layer, depth_layer)`.  Frames go down `batch` poses per native call; on one GPU the
        device->host copy of a frame overlaps the rendering of the next one inside the call (stnerf_render_views_host).
        `per_frame_state(idx, model)` may set model.shift / scale / alpha per frame (:435-440)."""
        n = len(poses)
        for i0 in range(0, n, self.batch):
            i1 = min(n, i0 + self.batch)
            b = i1 - i0
            if self.world == 1:
                svr = self._renderer()
                views = []
                self._rot_key = None
                for j in range(i0, i1):
                    if per_frame_state is not None:
                        per_frame_state(j, self.model)
                    views.append(self.make_view(poses[j], Ks[j], layer_frame_pairs[j], density_threshold, bkgd_density_threshold))
                if self._pinned is None or self._pinned.shape[0] < b:
                    self._pinned = torch.empty((self.batch, self.l + 1, self.H * self.W, 5), dtype=torch.float32).pin_memory()
                host = svr.nat.render_views_host(views, self.H, self.W, svr.n1, svr.n2, out_host=self._pinned[:b])
                host = host.view(b, self.l + 1, self.H, self.W, 5)
            else:
                dev = self.render_images_batch(poses[i0:i1], Ks[i0:i1], layer_frame_pairs[i0:i1], density_threshold,
                                               bkgd_density_threshold, per_frame_state, i0)
                host = dev.cpu()
            for j in range(b):
                yield self._finish(host[j])

    def _finish(self, host: torch.Tensor):
        color = host[0, ..., :3].clone()
        depth = host[0, ..., 3:4].clone()
        depth[depth < 0] = 0
        depth = depth / self.far
        color_layer = [host[1 + i, ..., :3].clone() for i in range(self.l)]
        depth_layer = [host[1 + i, ..., 3:4].clone() / self.far for i in range(self.l)]
        return color, depth, color_layer, depth_layer
