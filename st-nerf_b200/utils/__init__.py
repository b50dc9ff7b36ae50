"""Reference import name `utils` (utils/__init__.py:7-13): boundary helpers + per-stage operators."""
import torch

from stnerf_b200 import _fallthrough, ops

# `utils.<name>` for anything not replaced here (metrics, render_helpers, ...) resolves to the reference tree when one is on
# sys.path (stnerf_b200/_fallthrough.py); the submodules the demos import by name (`logger`, `vis_density`, `high_dim_dics`,
# `batchify_rays`) ship here so the import block of demo/taekwondo_demo.py:16-23 works with or without it.
_fallthrough.extend("utils", __path__)

from .batchify_rays import batchify_ray, layered_batchify_ray, layered_batchify_ray_big  # noqa: E402
from .vis_density import vis_density  # noqa: E402
from .high_dim_dics import add_two_dim_dict, add_three_dim_dict  # noqa: E402

try:      # camera helpers of the reference (`lookat`, `getSphericalPosition`: utils/render_helpers.py:5-40), when it is there
    from .render_helpers import lookat, getSphericalPosition  # noqa: E402,F401
except ImportError:
    pass


class Trigonometric_kernel:
    """utils/dimension_kernel.py:54-73."""

    def __init__(self, L=10, input_dim=3, include_input=True):
        if not include_input:
            raise NotImplementedError("include_input=False is not used by any shipped config (TKERNEL_INC_RAW: True)")
        self.L, self.input_dim = L, input_dim
        self.out_ch = input_dim * (1 + 2 * L)

    def __call__(self, x):
        return ops.positional_encoding(x, self.L)

    def calc_dim(self, dims=0):
        return self.out_ch


def sample_pdf(z_vals, weights, N_samples, det=False, pytest=False):
    """utils/sample_pdf.py:18-63.  `weights` is the inner slice w[...,1:-1] exactly as the reference call site passes
    it (layered_rfrender.py:460); uniforms are drawn with torch.rand on the device like the reference (:31)."""
    n = z_vals.shape[0]
    if det:
        u = torch.linspace(0., 1., steps=N_samples, device=z_vals.device).expand(n, N_samples).contiguous()
    else:
        u = torch.rand((n, N_samples), device=z_vals.device)
    w_full = torch.nn.functional.pad(weights, (1, 1))
    return ops.sample_pdf(z_vals, w_full, u)


def generate_rays(K, T, bbox, h, w):
    """utils/render_helpers.py:42-126 with bbox=None (the only form the render path uses, ray_dataset.py:263)."""
    if bbox is not None:
        raise NotImplementedError("bbox-cropped ray generation belongs to the training data pipeline (out of scope)")
    rays = ops.generate_rays(K, T, h, w)
    return rays, torch.ones(h, w, 1)


def ray_sampling(Ks, Ts, image_size, masks=None, mask_threshold=0.5, images=None, outlier_map=None):
    """utils/ray_sampling.py:22-72 (render-time form: no images / outlier map)."""
    if images is not None or outlier_map is not None:
        raise NotImplementedError("image / outlier-map sampling belongs to the training data pipeline (out of scope)")
    h, w = int(image_size[0]), int(image_size[1])
    out = []
    for m in range(Ks.shape[0]):
        rays = ops.generate_rays(Ks[m], Ts[m], h, w)
        if masks is not None:
            rays = rays[(masks[m] > mask_threshold).reshape(-1).to(rays.device)]
        out.append(rays)
    return torch.cat(out, 0), None


def ray_sampling_label_bbox(image, label, K, T, bbox=None, bboxes=None):
    """utils/ray_sampling.py:75-192: rays / labels / rgbs of the pixels in the box's projected rectangle (all pixels without
    a box), the (H,W,1) ray mask, and with `bboxes` each ray's box by its label.  Pixels are chosen and rays generated on the
    GPU; the results are returned on the input's device."""
    from stnerf_b200 import train_data
    return train_data.sample_label_bbox(image, label, K, T, bbox=bbox, bboxes=bboxes)


def ray_sampling_label_label(image, label, K, T, label0):
    """utils/ray_sampling.py:194-240: rays / labels / rgbs of the pixels whose label is label0, and the (H,W,1) ray mask."""
    from stnerf_b200 import train_data
    return train_data.sample_label_label(image, label, K, T, label0)


__all__ = ["Trigonometric_kernel", "sample_pdf", "generate_rays", "ray_sampling", "batchify_ray",
           "layered_batchify_ray", "layered_batchify_ray_big", "ray_sampling_label_bbox", "ray_sampling_label_label",
           "vis_density", "add_two_dim_dict", "add_three_dim_dict"]
