"""layers/render_layer.py of the reference on the native compositing kernels (stnerf_b200.volume): differentiable in rgb and
sigma, like the reference."""
import torch

from stnerf_b200 import volume


def gen_weight(sigma, delta, act_fn=torch.nn.functional.relu):
    """layers/render_layer.py:8-16.  sigma (N,S,1), delta (N,S) -> weights (N,S).  Computed through the compositing kernel with
    depths rebuilt from the deltas (t_0 = 0, last delta taken as the border weight), so the deltas get no gradient."""
    if act_fn is not torch.nn.functional.relu:
        raise NotImplementedError("only the default relu activation is used by the reference")
    if torch.is_grad_enabled() and delta.requires_grad:
        raise NotImplementedError("gen_weight has no gradient with respect to delta (the reference's deltas are detached)")
    n, s = sigma.shape[0], sigma.shape[1]
    d = delta.reshape(n, s)
    t = torch.cumsum(torch.cat([torch.zeros_like(d[:, :1]), d[:, :-1]], 1), 1)
    if not bool((d[:, -1] == d[0, -1]).all()):
        raise NotImplementedError("per-ray border deltas are not produced by any reference caller")
    rgb = torch.zeros((n, s, 3), device=sigma.device)
    _, _, _, w = volume.composite(t, rgb, sigma.reshape(n, s), float(d[0, -1]))
    return w


class VolumeRenderer(torch.nn.Module):
    """layers/render_layer.py:19-58.  forward(depth (N,L,1), rgb (N,L,3), sigma (N,L,1)) -> color, depth, acc, weights (N,L,1)."""

    def __init__(self, use_mask=False, boarder_weight=1e10):
        super().__init__()
        if use_mask:
            raise NotImplementedError("use_mask=True is never used by the layered renderer")
        self.boarder_weight = boarder_weight

    def forward(self, depth, rgb, sigma, noise=0):
        if noise > 0.:
            sigma = sigma + torch.randn_like(sigma) * noise                         # :42-43
        n, s = depth.shape[0], depth.shape[1]
        c, d, a, w = volume.composite(depth.reshape(n, s), rgb, sigma.reshape(n, s), self.boarder_weight)
        return c, d, a, w.unsqueeze(-1)
