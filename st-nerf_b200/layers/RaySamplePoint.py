"""layers/RaySamplePoint.py of the reference on the native kernels (the module `demo/*.py` imports `RaySamplePoint` from)."""
import torch

from stnerf_b200 import ops


def intersection(rays, bbox):
    """layers/RaySamplePoint.py:8-62.  rays (N,>=6), bbox (N,8,3) -> (N,2) = [t_far, t_near] (topk(2) of the face hits,
    -1000 where a face is missed).  The box is read from row 0 (every reference caller repeats one box per call,
    modeling/layered_rfrender.py:195-208)."""
    corners = bbox[0].detach().cpu()
    n = rays.shape[0]
    jitter = torch.zeros((n, 1), device=rays.device)
    _, _, _, tt = ops.intersect_sample(rays, corners[0], corners[6], 1, jitter, is_bkgd=False, want_xyz=False)
    return tt


class RaySamplePoint(torch.nn.Module):
    """layers/RaySamplePoint.py:64-107.  forward(rays (N,>=6), bbox (N,L,8,3)) -> lists of t (N,C,1), xyz (N,C,3), mask (N).
    Boxes are read from row 0 (all rows are identical in every reference caller, layered_rfrender.py:195-208)."""

    def __init__(self, coarse_num=64):
        super().__init__()
        self.coarse_num = coarse_num

    def forward(self, rays, bbox, pdf=None, method='coarse'):
        n, l = rays.shape[0], bbox.shape[1]
        ts, pts, masks = [], [], []
        for i in range(l):
            corners = bbox[0, i].detach().cpu()
            jitter = torch.rand((n, self.coarse_num), device=rays.device)          # :98
            t, xyz, mask, _ = ops.intersect_sample(rays, corners[0], corners[6], self.coarse_num, jitter, is_bkgd=(i == 0))
            ts.append(t.unsqueeze(-1)); pts.append(xyz); masks.append(mask)
        return ts, pts, masks


class RaySamplePoint_Near_Far(torch.nn.Module):
    """Unusable in the reference's layered model (SURVEY A.9: reads an attribute that is never set)."""

    def __init__(self, sample_num=75):
        super().__init__()
        self.sample_num = sample_num

    def forward(self, *a, **k):
        raise NotImplementedError("NEAR_FAR sampling is a dead branch of the reference (modeling/layered_rfrender.py:254)")


class RayDistributedSamplePoint(torch.nn.Module):
    """layers/RaySamplePoint.py:110-152: superseded in the reference by utils.sample_pdf (never constructed by the layered model)."""

    def __init__(self, fine_num=10):
        super().__init__()
        self.fine_num = fine_num

    def forward(self, *a, **k):
        raise NotImplementedError("RayDistributedSamplePoint is not used by the layered renderer; use utils.sample_pdf")
