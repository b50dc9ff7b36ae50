"""CPU oracle for the st-nerf layered ray-march hot path.

TEST INFRASTRUCTURE ONLY.  This module is a CPU restatement (torch fp32 tensors
used as the array library, because the reference's arithmetic *is* ATen fp32) of
the reference algorithm.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it.  The
product path (``st-nerf_b200/``) never does: it fails loudly when the CUDA
library is missing.

Parity status: PINNED.  ``tests/golden/make_golden.py`` runs the unmodified
reference (``/root/reference``, imported in the build container with a no-op
``.cuda()`` shim and injected uniforms) and stores its outputs under
``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks every function
here against those vectors.

Every function cites the reference file:line it restates (paths relative to the
reference root).  The structure is deliberately different from the reference
(per-layer min/max boxes instead of (N,l,8,3) tensors, a single flat weights
dict, explicit uniforms) -- it restates the arithmetic, not the code.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

F32 = torch.float32
_EPS64 = 2.220446049250313e-16  # np.finfo(float).eps, layers/RaySamplePoint.py:17-22


# --------------------------------------------------------------------------- a6
def positional_encoding(x: torch.Tensor, n_freq: int) -> torch.Tensor:
    """utils/dimension_kernel.py:24-33,36-51.  [x, sin(2^0 x), cos(2^0 x), ...]."""
    out = [x]
    for k in range(n_freq):
        f = float(2.0 ** k)          # exact power of two (log_sampling linspace)
        out.append(torch.sin(x * f))
        out.append(torch.cos(x * f))
    return torch.cat(out, -1)


# --------------------------------------------------------------------------- a14
def split_state_dict(sd: Dict[str, torch.Tensor], layer_num: int) -> dict:
    """Group a reference ``state_dict`` (SURVEY App. B key names) by network."""
    def sub(prefix):
        return {k[len(prefix):]: v.detach().to(F32).contiguous()
                for k, v in sd.items() if k.startswith(prefix)}
    nets = {
        "bkgd": sub("bkgd_spacenet."),
        "bkgd_fine": sub("bkgd_spacenet_fine."),
        "space": [sub("spacenets.%d." % i) for i in range(layer_num)],
        "space_fine": [sub("spacenets_fine.%d." % i) for i in range(layer_num)],
        "motion": [sub("time_deform_nets.%d." % i) for i in range(layer_num)],
    }
    return nets


# --------------------------------------------------------------------------- a8
def spacenet_forward(w: Dict[str, torch.Tensor], pos: torch.Tensor, dirs: torch.Tensor,
                     times: Optional[torch.Tensor]):
    """modeling/spacenet.py:101-160.

    pos (P,3); dirs (P,3); times (P,1) or None.  Returns raw rgb (P,3), sigma (P,1).
    Whether the net consumes ``times`` is decided by its rgb_net.1 width (283 vs 304).
    """
    pe = positional_encoding(pos, 10)                                   # :127
    x = pe
    for i in (0, 2, 4, 6):                                              # stage1 :45-54
        x = F.relu(F.linear(x, w["stage1.%d.weight" % i], w["stage1.%d.bias" % i]))
    x = torch.cat([x, pe], 1)                                           # :137
    for i in (0, 2, 4):                                                 # stage2 :56-63
        x = F.relu(F.linear(x, w["stage2.%d.weight" % i], w["stage2.%d.bias" % i]))
    sigma = F.linear(x, w["density_net.0.weight"], w["density_net.0.bias"])   # :139
    feats = [x, positional_encoding(dirs, 4)]                           # :128-129,143
    use_time = w["rgb_net.1.weight"].shape[1] == 256 + 27 + 21
    if use_time:
        feats.append(positional_encoding(times, 10))                    # :130-131,149
    h = F.relu(torch.cat(feats, 1))                                     # rgb_net[0] ReLU :82
    h = F.relu(F.linear(h, w["rgb_net.1.weight"], w["rgb_net.1.bias"]))
    rgb = F.linear(h, w["rgb_net.3.weight"], w["rgb_net.3.bias"])
    return rgb, sigma


# --------------------------------------------------------------------------- a7
def motionnet_forward(w: Dict[str, torch.Tensor], xyzt: torch.Tensor) -> torch.Tensor:
    """modeling/motion_net.py:34-71.  xyzt (P,4) -> flow (P,3)."""
    xyz, t = xyzt[:, :3], xyzt[:, 3:]
    lower = torch.floor(t)
    if not bool(torch.all(lower == t)):                                 # :53 batch-global test
        wgt = t - lower
        lo = positional_encoding(torch.cat([xyz, lower], -1), 10)
        hi = positional_encoding(torch.cat([xyz, lower + 1], -1), 10)
        x = (1 - wgt) * lo + wgt * hi                                   # :63
    else:
        x = positional_encoding(xyzt, 10)
    for i in (0, 2, 4, 6, 8):
        x = F.relu(F.linear(x, w["motion_net.%d.weight" % i], w["motion_net.%d.bias" % i]))
    return F.linear(x, w["motion_net.10.weight"], w["motion_net.10.bias"])


# --------------------------------------------------------------------------- a3
def ray_box_candidates(o: torch.Tensor, d: torch.Tensor, bmin: torch.Tensor, bmax: torch.Tensor) -> torch.Tensor:
    """layers/RaySamplePoint.py:8-58.  (N,6) face candidates in the order left, right, front, back, bottom, up: the face's t
    where its hit point lies in the face (inclusive), else -1e3."""
    n = o.shape[0]
    eps = torch.tensor(_EPS64, dtype=F32)
    cand = torch.full((n, 6), -1000.0, dtype=F32)
    col = 0
    for axis in range(3):
        a1, a2 = [a for a in range(3) if a != axis]
        for face in (bmin[..., axis], bmax[..., axis]):               # bmin / bmax: (3,) one box, or (N,3) a box per ray
            t = (face - o[:, axis]) / (d[:, axis] + eps)                # :17-22
            p = t[:, None] * d + o                                      # :27-32 (mul then add)
            ok = (p[:, a1] >= bmin[..., a1]) & (p[:, a1] <= bmax[..., a1]) & \
                 (p[:, a2] >= bmin[..., a2]) & (p[:, a2] <= bmax[..., a2])        # :34-51 inclusive
            cand[:, col] = torch.where(ok, t, cand[:, col])
            col += 1
    return cand


def ray_box_intersect(o: torch.Tensor, d: torch.Tensor, bmin: torch.Tensor, bmax: torch.Tensor, cols: int = 6):
    """layers/RaySamplePoint.py:8-62.  Returns (t_far, t_near) = the top-2 of the face candidates and the -1e3 sentinels of
    tlist = -1e3 * ones_like(rays) (:53), which has one slot per ray column: ``cols`` is the rays' width, 6 for bare
    [o, d] rays; rays that carry frame-id columns pass their full width."""
    cand = ray_box_candidates(o, d, bmin, bmax)
    tlist = torch.cat([cand, torch.full((o.shape[0], cols - 6), -1000.0, dtype=F32)], 1)
    top = tlist.topk(k=2, dim=-1)[0]                                    # :60
    return top[:, 0], top[:, 1]


# --------------------------------------------------------------------------- a4
def stratified_samples(o, d, bmin, bmax, n1: int, jitter: torch.Tensor, is_bkgd: bool, cols: int = 6):
    """layers/RaySamplePoint.py:85-105.  jitter (N,n1) in [0,1), rays ``cols`` columns wide (see ``ray_box_intersect``).
    Returns t (N,n1), xyz (N,n1,3), mask (N)."""
    t_far, t_near = ray_box_intersect(o, d, bmin, bmax, cols)
    start = t_near.clone()
    if is_bkgd:
        start[start <= 0] = 0                                           # :93-95
    width = ((t_far - start) / n1)[:, None]                             # :100
    k = torch.arange(0, n1, dtype=F32)[None, :]
    t = (k + jitter) * width + start[:, None]                           # :102
    xyz = t[..., None] * d[:, None, :] + o[:, None, :]                  # :103
    mask = (width.abs() > 1e-5)[:, 0]                                   # :105
    return t, xyz, mask


# --------------------------------------------------------------------------- a10
def composite(t: torch.Tensor, rgb: torch.Tensor, sigma: torch.Tensor, boarder: float = 1e10):
    """layers/render_layer.py:8-17,25-58.  t (N,S), rgb (N,S,3) raw, sigma (N,S) raw."""
    n = t.shape[0]
    delta = torch.cat([t[:, 1:] - t[:, :-1], torch.full((n, 1), boarder, dtype=F32)], -1)
    alpha = 1.0 - torch.exp(-F.relu(sigma) * delta)
    trans = torch.cumprod(torch.cat([torch.ones((n, 1), dtype=F32), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * trans
    color = torch.sum(torch.sigmoid(rgb) * w[..., None], dim=1)
    depth = torch.sum(w * t, dim=1, keepdim=True)
    acc = torch.sum(w, dim=1, keepdim=True)
    return color, depth, acc, w


# --------------------------------------------------------------------------- a11
def sample_pdf(t: torch.Tensor, w_inner: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    """utils/sample_pdf.py:18-63 with injected uniforms.  t (N,n1), w_inner = w[:,1:-1] (N,n1-2), u (N,n2)."""
    bins = 0.5 * (t[:, 1:] + t[:, :-1])
    wp = w_inner + 1e-5
    pdf = wp / torch.sum(wp, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)            # (N, n1-1)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)                    # :49 (== n1-2)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    tt = (u - cdf_b) / denom
    return bin_b + tt * (bin_a - bin_b)


# --------------------------------------------------------------------------- a1
def generate_rays(K: torch.Tensor, T: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """utils/render_helpers.py:96-123 (bbox=None) == utils/ray_sampling.py:22-72 without masks.  -> (h*w, 6)."""
    ii, jj = torch.meshgrid(torch.arange(h, dtype=F32), torch.arange(w, dtype=F32), indexing="ij")
    pix = torch.stack([jj, ii, torch.ones_like(ii)], -1)[..., None]    # (h,w,3,1): (col,row,1)
    dirs = torch.matmul(torch.inverse(K.to(F32)), pix)
    dirs = dirs / torch.norm(dirs, dim=2, keepdim=True)
    dirs = torch.matmul(T.to(F32)[:3, :3], dirs)[..., 0]
    pos = T.to(F32)[:3, 3].expand(h, w, 3)
    return torch.cat([pos, dirs], -1).reshape(-1, 6)


# --------------------------------------------------------------------------- a2
def resolve_scene(bboxes: torch.Tensor, bkgd_bbox: torch.Tensor, frame_ids: Sequence[float],
                  scale: Optional[Sequence[float]], shift: Optional[Sequence]) -> dict:
    """modeling/layered_rfrender.py:190-242 in the retiming branch.

    bboxes (F,L,8,3) per-frame performer boxes, bkgd_bbox (1,8,3), frame_ids = ray 0's
    columns 6.. (index 0 = bkgd).  Returns per-layer min/max corners *after* the scale /
    shift edits plus the scale pivot.
    """
    L = bboxes.shape[1]
    boxes = [bkgd_bbox.reshape(8, 3).to(F32).clone()]
    for i in range(L):
        f = float(frame_ids[i + 1]) - 1.0
        f = torch.tensor(f, dtype=F32)
        lo, hi = bboxes[math.floor(f), i], bboxes[math.ceil(f), i]
        boxes.append(torch.lerp(lo.to(F32), hi.to(F32), f - math.floor(f)))          # :123-127
    boxes = torch.stack(boxes, 0)                                                     # (l,8,3)
    first = torch.cat([bkgd_bbox.reshape(1, 8, 3).to(F32), bboxes[0].to(F32)], 0)    # :216-220
    centre = first.mean(1)                                                            # :221
    centre[:, 2] = first[:, 1, 2]                                                     # :226
    pivot = None
    if scale is not None:
        pivot = (centre[2] + centre[1]) / 2                                           # :232
        for i in range(len(scale)):
            boxes[i] = (boxes[i] - pivot) * scale[i] + pivot
    if shift is not None:
        for i in range(len(shift)):
            if shift[i] is None:
                continue
            boxes[i] = boxes[i] + torch.tensor(shift[i], dtype=F32)                   # :237-242
    return {"bmin": boxes[:, 0, :].clone(), "bmax": boxes[:, 6, :].clone(), "pivot": pivot}


def box_table(bboxes: torch.Tensor, bkgd_bbox: torch.Tensor, scale: Optional[Sequence[float]], shift: Optional[Sequence]) -> torch.Tensor:
    """(F, l, 2, 3) min / max corners of every layer's box at every frame after the scale / shift edits: what
    `bboxes = self.bboxes.index_select(0, frame_id - 1)` (:193) followed by :207-242 gives a ray of frame `f` (row f-1)."""
    Fn = bboxes.shape[0]
    rows = []
    for f in range(Fn):
        sc = resolve_scene(bboxes, bkgd_bbox, [0.0] + [float(f + 1)] * bboxes.shape[1], scale, shift)
        rows.append(torch.stack([sc["bmin"], sc["bmax"]], 1))
    return torch.stack(rows, 0)


def _inverse_edit(xyz, i, scale, shift, pivot, fine: bool):
    """modeling/layered_rfrender.py:293-303 (coarse) / :467-475 (fine, where a None shift entry also skips the scale)."""
    if shift is not None:
        if fine:
            if shift[i] is None:
                return xyz
            xyz = xyz - torch.tensor(shift[i], dtype=F32)
        elif i < len(shift) and shift[i] is not None:
            xyz = xyz - torch.tensor(shift[i], dtype=F32)
    if scale is not None and (fine or i < len(scale)):
        xyz = (xyz - pivot) / scale[i] + pivot
    return xyz


# --------------------------------------------------------------------------- a2..a13
def render(nets: dict, scene: dict, rays: torch.Tensor, n1: int, n2: int,
           jitter: torch.Tensor, u: Optional[torch.Tensor], only_coarse: bool = False,
           density_threshold: float = 1e-4, bkgd_density_threshold: float = 0.0, shared_frame: bool = False) -> dict:
    """modeling/layered_rfrender.py:141-734, retiming (render-time) branch, BBOX sampling.

    rays (N, 6+l) fp32; jitter (l,N,n1); u (l,N,n2).
    scene: bmin/bmax (l,3) (already edited, see ``resolve_scene``), pivot, scale, shift,
           shown (list of l bools), near, alpha, boarder.
           Optional ``box_table`` (F,l,2,3) with ``shared_frame``: rays of a mixed-frame batch, each taking the boxes of ITS
           frame id, `self.bboxes.index_select(0, frame_id - 1)` (:193; see ``box_table``).
    """
    rays = rays.to(F32)
    o, d = rays[:, :3], rays[:, 3:6]
    l = scene["bmin"].shape[0]
    fid = rays[:, 6:]
    if shared_frame:
        # 7-column evaluator rays [o,d,frame_id] (:157-158,171): every layer reads the same column, boxes come from
        # index_select(frame_id - 1) (:193) and the density thresholds are skipped (`if self.retiming`, :416,538,564)
        fid = rays[:, 6:7].expand(-1, l)
        density_threshold = bkgd_density_threshold = float("-inf")
    N = rays.shape[0]
    scale, shift, pivot = scene.get("scale"), scene.get("shift"), scene.get("pivot")
    shown = scene.get("shown", [True] * l)
    near = float(scene.get("near", 0.0))
    alpha2 = float(scene.get("alpha", 1.0))
    boarder = float(scene.get("boarder", 1e10))

    def run_layer(i, xyz, fine):
        """Deform (a7) + radiance (a8) on the hit rays of layer i.  xyz (N,S,3) already inverse-edited."""
        S = xyz.shape[1]
        rgb = torch.zeros(N, S, 3, dtype=F32)
        sig = torch.zeros(N, S, dtype=F32)
        if i == 0:
            net = nets["bkgd_fine"] if fine else nets["bkgd"]
            r, s = spacenet_forward(net, xyz.reshape(-1, 3), d[:, None, :].expand(N, S, 3).reshape(-1, 3),
                                    fid[:, 0:1][:, None, :].expand(N, S, 1).reshape(-1, 1))
            return r.reshape(N, S, 3), s.reshape(N, S)
        idx = masks[i]
        M = int(idx.sum())
        if M == 0:
            return rgb, sig
        p = xyz[idx]
        tcol = fid[idx, i][:, None, None].expand(M, S, 1)
        flow = motionnet_forward(nets["motion"][i - 1], torch.cat([p, tcol], -1).reshape(-1, 4))     # :340-356
        p = p + flow.reshape(M, S, 3)
        if not shown[i]:
            return rgb, sig
        net = (nets["space_fine"] if fine else nets["space"])[i - 1]
        r, s = spacenet_forward(net, p.reshape(-1, 3), d[idx][:, None, :].expand(M, S, 3).reshape(-1, 3),
                                tcol.reshape(-1, 1))
        rgb[idx] = r.reshape(M, S, 3)
        sig[idx] = s.reshape(M, S)
        return rgb, sig

    # ---- coarse pass --------------------------------------------------------------
    ts, masks, rgbs, sigs = [], [], [], []
    xyzs = []
    table = scene.get("box_table") if shared_frame else None
    row = (rays[:, 6].to(torch.int64) - 1) if table is not None else None                            # :193
    for i in range(l):
        bmin_i = scene["bmin"][i] if table is None else table[row, i, 0]
        bmax_i = scene["bmax"][i] if table is None else table[row, i, 1]
        t, xyz, m = stratified_samples(o, d, bmin_i, bmax_i, n1, jitter[i], i == 0, rays.shape[1])
        ts.append(t); masks.append(m)
        xyzs.append(_inverse_edit(xyz, i, scale, shift, pivot, fine=False))
    for i in range(l):
        rgb, sig = run_layer(i, xyzs[i], fine=False)
        if i >= 1 and bool(masks[i].any()) and shown[i]:
            sig = torch.where(ts[i] < 0, torch.zeros_like(sig), sig)                                 # :414
            sig = torch.where(sig < density_threshold, torch.zeros_like(sig), sig)                   # :416-418
        rgbs.append(rgb); sigs.append(sig)
    sigs[0] = torch.where(ts[0] < near, torch.zeros_like(sigs[0]), sigs[0])                          # :422

    def merged(tl, rl, sl, near_cut):
        tm, order = torch.sort(torch.cat(tl, 1), 1)                                                  # :425 / :587
        rm = torch.cat(rl, 1).gather(1, order[..., None].expand(-1, -1, 3))
        sm = torch.cat(sl, 1).gather(1, order)
        if near_cut:
            sm = torch.where(tm < near, torch.zeros_like(sm), sm)                                    # :605
        return composite(tm, rm, sm, boarder)[:3]

    coarse_layer, weights = [], []
    for i in range(l):
        c, dp, a, w = composite(ts[i], rgbs[i], sigs[i], boarder)                                    # :435-444
        coarse_layer.append((c, dp, a)); weights.append(w)
    coarse_mixed = merged(ts, rgbs, sigs, near_cut=False)                                            # :448
    out = {"coarse_mixed": coarse_mixed, "coarse_layer": coarse_layer, "ray_mask": masks,
           "t_coarse": ts, "w_coarse": weights}
    if only_coarse:
        out["fine_mixed"], out["fine_layer"] = coarse_mixed, coarse_layer                            # :721-722
        return out

    # ---- fine pass ----------------------------------------------------------------
    tf, rgbs, sigs = [], [], []
    for i in range(l):
        z = sample_pdf(ts[i], weights[i][:, 1:-1], u[i])                                             # :460
        tfi, _ = torch.sort(torch.cat([ts[i], z], -1), -1)                                           # :462
        tf.append(tfi)
    for i in range(l):
        xyz = tf[i][..., None] * d[:, None, :] + o[:, None, :]                                       # :465
        xyz = _inverse_edit(xyz, i, scale, shift, pivot, fine=True)
        rgb, sig = run_layer(i, xyz, fine=True)
        if i == 0:
            sig = torch.where(sig < bkgd_density_threshold, torch.zeros_like(sig), sig)              # :538-547
        elif bool(masks[i].any()) and shown[i]:
            sig = torch.where(sig < density_threshold, torch.zeros_like(sig), sig)                   # :564-566
            if i == 2:
                sig = sig * alpha2                                                                   # :575-576
        rgbs.append(rgb); sigs.append(sig)
    fine_layer = [composite(tf[i], rgbs[i], sigs[i], boarder)[:3] for i in range(l)]                 # :598-603
    out["fine_mixed"] = merged(tf, rgbs, sigs, near_cut=True)                                        # :605-606
    out["fine_layer"] = fine_layer
    out["t_fine"] = tf
    return out


# --------------------------------------------------------------------------- synthetic inputs (SURVEY 8d)
def corners_from_minmax(bmin, bmax) -> torch.Tensor:
    """Corner order of data/datasets/frame_dataset.py:187-188."""
    x0, y0, z0 = [float(v) for v in bmin]
    x1, y1, z1 = [float(v) for v in bmax]
    return torch.tensor([[x0, y0, z0], [x1, y0, z0], [x1, y1, z0], [x0, y1, z0],
                         [x0, y0, z1], [x1, y0, z1], [x1, y1, z1], [x0, y1, z1]], dtype=F32)


def synthetic_boxes(layer_num: int, n_frames: int = 101):
    """SURVEY 8(d): bkgd box (-6,-6,-1)..(6,6,4); performers 0.8x0.8x1.8 on z=0, centres on x in [-2,2]."""
    bkgd = corners_from_minmax((-6, -6, -1), (6, 6, 4))[None]
    per = []
    for i in range(layer_num):
        cx = 0.0 if layer_num == 1 else -2.0 + 4.0 * i / (layer_num - 1)
        per.append(corners_from_minmax((cx - 0.4, -0.4, 0.0), (cx + 0.4, 0.4, 1.8)))
    per = torch.stack(per, 0)                                         # (L,8,3)
    # a slow drift so fractional frame ids exercise the bbox lerp
    frames = torch.stack([per + 0.002 * f * torch.tensor([1.0, 0.5, 0.0]) for f in range(n_frames)], 0)
    return bkgd, frames


def synthetic_camera(view: int, n_views: int, h: int, w: int):
    """SURVEY 8(d): circle radius 5, height 1.0, looking at (0,0,0.9), up +z, OpenCV c2w; fx=fy=0.78*W."""
    az = 2 * math.pi * view / n_views
    eye = torch.tensor([5 * math.cos(az), 5 * math.sin(az), 1.0], dtype=torch.float64)
    tgt = torch.tensor([0.0, 0.0, 0.9], dtype=torch.float64)
    fwd = tgt - eye; fwd = fwd / fwd.norm()
    up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    right = torch.linalg.cross(fwd, up); right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    T = torch.eye(4, dtype=torch.float64)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, fwd, eye
    K = torch.tensor([[0.78 * w, 0, w / 2], [0, 0.78 * w, h / 2], [0, 0, 1]], dtype=torch.float64)
    return K.to(F32), T.to(F32)


def synthetic_state_dict(layer_num: int, use_space_time: bool, seed: int = 0, gain: float = 1.6):
    """Seeded random weights with the reference's key names/shapes (SURVEY App. B).

    ``gain`` scales the nn.Linear-style uniform init so activations do not collapse to
    zero through 8 layers (keeps sigma/rgb in a range where parity errors are visible).
    Generated with numpy's legacy RandomState so they are identical on every host.
    """
    import numpy as np
    rs = np.random.RandomState(seed)
    sd = {}

    def lin(name, out_f, in_f, g=gain):
        b = g / math.sqrt(in_f)
        sd[name + ".weight"] = torch.from_numpy(rs.uniform(-b, b, (out_f, in_f)).astype(np.float32))
        sd[name + ".bias"] = torch.from_numpy(rs.uniform(-b, b, (out_f,)).astype(np.float32))

    def spacenet(prefix, use_time):
        lin(prefix + "stage1.0", 256, 63)
        for i in (2, 4, 6):
            lin(prefix + "stage1.%d" % i, 256, 256)
        lin(prefix + "stage2.0", 256, 319)
        for i in (2, 4):
            lin(prefix + "stage2.%d" % i, 256, 256)
        lin(prefix + "density_net.0", 1, 256, g=gain * 4)
        lin(prefix + "rgb_net.1", 128, 256 + 27 + (21 if use_time else 0))
        lin(prefix + "rgb_net.3", 3, 128)

    spacenet("bkgd_spacenet.", False)
    spacenet("bkgd_spacenet_fine.", False)
    for i in range(layer_num):
        spacenet("spacenets.%d." % i, use_space_time)
    for i in range(layer_num):
        spacenet("spacenets_fine.%d." % i, use_space_time)
    for i in range(layer_num):
        p = "time_deform_nets.%d.motion_net." % i
        lin(p + "0", 128, 84)
        for j in (2, 4, 6, 8):
            lin(p + "%d" % j, 128, 128)
        lin(p + "10", 3, 128, g=0.1)
    return sd
