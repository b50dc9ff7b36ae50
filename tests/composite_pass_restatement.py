"""A plain restatement of one compositing pass of LayeredRFRender.forward, for the tests of composite_pass_kernel.

Written from the reference's formulas -- layers/render_layer.py:8-58 (gen_weight / VolumeRenderer.forward),
utils/sample_pdf.py:18-63, modeling/layered_rfrender.py:412-422 (coarse density masks), :425-463 (coarse merge + resampling),
:538-606 (fine masks + merge) -- with whole-array torch ops: cumprod, cumsum, searchsorted(right=True), a stable argsort of the
concatenation.  Nothing here follows the kernels' structure (no warps, no ranks, no bitmasks).  Every function computes in the
dtype of its inputs: float64 is the truth the kernels are held to, float32 on the CPU is the yardstick that says how far a
correct fp32 evaluation of the same formulas lands from it.  tests/test_composite_pass_restatement.py pins it to the
reference's own outputs (tests/golden/functions.npz).

A scene is a dict: near, alpha2, thr_layer, thr_bkgd, boarder (floats), apply_thr (bool), shown (list of bool per layer; entry 0
is ignored like the reference ignores it).
"""
from __future__ import annotations

import torch


def weights(t, sigma, boarder):
    """gen_weight of the deltas of `t` (render_layer.py:8-17, 37-40).  t, sigma (..., S) -> w (..., S)."""
    pad = torch.full_like(t[..., :1], boarder)
    delta = torch.cat([t[..., 1:] - t[..., :-1], pad], -1)
    alpha = 1.0 - torch.exp(-torch.relu(sigma) * delta)
    f = 1.0 - alpha + 1e-10
    T = torch.cumprod(torch.cat([torch.ones_like(f[..., :1]), f], -1), -1)[..., :-1]
    return alpha * T


def composite(t, logits, sigma, boarder):
    """VolumeRenderer.forward (render_layer.py:25-58).  t, sigma (..., S), logits (..., S, 3) -> pixel (..., 5) = rgb, depth,
    acc; w (..., S)."""
    w = weights(t, sigma, boarder)
    color = (torch.sigmoid(logits) * w[..., None]).sum(-2)
    depth = (w * t).sum(-1, keepdim=True)
    acc = w.sum(-1, keepdim=True)
    return torch.cat([color, depth, acc], -1), w


def mask_density(scene, layer, fine, t, sigma):
    """The density a pass composites for `layer` (layered_rfrender.py:401,414-422 coarse; :538-547, 556, 564-576 fine)."""
    if layer > 0 and not scene["shown"][layer]:
        return torch.zeros_like(sigma)
    zero = torch.zeros_like(sigma)
    thr = scene["thr_bkgd"] if (layer == 0 and fine) else scene["thr_layer"]
    if not fine:
        sigma = torch.where(t < (scene["near"] if layer == 0 else 0.0), zero, sigma)
        if layer > 0 and scene["apply_thr"]:
            sigma = torch.where(sigma < thr, zero, sigma)
        return sigma
    if scene["apply_thr"]:
        sigma = torch.where(sigma < thr, zero, sigma)
    if layer == 2:
        sigma = sigma * scene["alpha2"]
    return sigma


def sample_pdf(t, w, u):
    """utils/sample_pdf.py:18-63.  t, w (..., n1) (w = the FULL weights; the [1:-1] slice is taken here like the caller does,
    layered_rfrender.py:460), u (..., n2) -> z (..., n2) and the intermediate values a test conditions its tolerance on."""
    bins = 0.5 * (t[..., 1:] + t[..., :-1])
    wi = w[..., 1:-1] + 1e-5
    pdf = wi / wi.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[..., :1]), torch.cumsum(pdf, -1)], -1)
    inds = torch.searchsorted(cdf, u.contiguous(), right=True)
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    cb, ca = cdf.gather(-1, below), cdf.gather(-1, above)
    bb, ba = bins.gather(-1, below), bins.gather(-1, above)
    den_raw = ca - cb
    den = torch.where(den_raw < 1e-5, torch.ones_like(den_raw), den_raw)
    z = bb + (u - cb) / den * (ba - bb)
    return z, {"cdf": cdf, "bins": bins, "cb": cb, "ca": ca, "bb": bb, "ba": ba, "den_raw": den_raw, "den": den,
               "below": below}


def merged_pixel(scene, fine, ts, logits, sigmas, reverse_ties=False):
    """The merged image (layered_rfrender.py:425-448 / :587-606): sort the concatenation of the lists by depth -- ties in
    concatenation order, as a stable sort leaves them -- gather colours and densities, composite.  ts[h], sigmas[h] (n, S),
    logits[h] (n, S, 3), already masked per layer.  reverse_ties: the opposite tie order (for tests that show a case
    discriminates)."""
    t = torch.cat(ts, -1)
    if reverse_ties:
        idx = torch.argsort(t.flip(-1), dim=-1, stable=True)
        idx = t.shape[-1] - 1 - idx
    else:
        idx = torch.argsort(t, dim=-1, stable=True)
    t = t.gather(-1, idx)
    sg = torch.cat(sigmas, -1).gather(-1, idx)
    lg = torch.cat(logits, -2).gather(-2, idx[..., None].expand(idx.shape + (3,)))
    if fine:
        sg = torch.where(t < scene["near"], torch.zeros_like(sg), sg)                      # :605
    return composite(t, lg, sg, scene["boarder"])[0]


def run_pass(scene, fine, t, raw, mask, u=None, reverse_ties=False):
    """One pass over l layers.  t (l,n,S), raw (l,n,S,4), mask (l,n) bool (row 0 ignored: the background is always hit),
    u (l,n,n2) or None.  A missed layer takes no part in the merge (the reference parks its samples at t = -1000 with zero
    density, where they change nothing) and gets a zero image.  -> images (l+1, n, 5); with u also z (l,n,n2) in draw order,
    t_fine (l,n,S+n2) and `pdf`, the per-layer intermediates of sample_pdf."""
    l, n, S = t.shape
    hit = mask.clone().bool()
    hit[0] = True
    shown = [True] + [bool(scene["shown"][i]) for i in range(1, l)]
    images = torch.zeros((l + 1, n, 5), dtype=t.dtype)
    sig = [mask_density(scene, i, fine, t[i], raw[i, ..., 3]) for i in range(l)]
    lg = [raw[i, ..., :3] if shown[i] else torch.zeros_like(raw[i, ..., :3]) for i in range(l)]
    out = {"images": images}
    ws = []
    for i in range(l):
        pix, w = composite(t[i], lg[i], sig[i], scene["boarder"])
        images[1 + i] = torch.where(hit[i][:, None], pix, torch.zeros_like(pix))
        ws.append(w)
    # the merge, one group of rays per set of hit layers
    code = sum(hit[i].long() << i for i in range(l))
    for c in torch.unique(code).tolist():
        rows = torch.nonzero(code == c)[:, 0]
        ls = [i for i in range(l) if (c >> i) & 1]
        images[0, rows] = merged_pixel(scene, fine, [t[i][rows] for i in ls], [lg[i][rows] for i in ls],
                                       [sig[i][rows] for i in ls], reverse_ties)
    if u is not None:
        zs, pdfs = zip(*[sample_pdf(t[i], ws[i], u[i]) for i in range(l)])
        out["z"] = torch.stack(zs)
        out["pdf"] = pdfs
        out["t_fine"] = torch.sort(torch.cat([t, out["z"]], -1), -1)[0]                    # :462
    return out
