"""Test-side restatement of one training forward of the layered model (modeling/layered_rfrender.py:141-734, BBOX sampling,
both ray layouts) in any dtype and on any device, differentiable in every network parameter.  Pinned to the unmodified
reference's float64 gradients by tests/test_train_forward.py (tests/golden/train_grads.npz).

Options for holding an fp32 implementation to float64 (tests/test_gpu_train_forward.py, the method of
test_gpu_composite_grad.py's training chain):
  samples   (t_coarse (l,N,n1), mask (l,N)) fp32: use these depths and hit masks (the points are formed from them in fp32,
            as the fp32 implementations form them) instead of sampling;
  fine_t    per layer (N,n1+n2) fp32: the fine depths to use instead of resampling;
  keep      per network call ("c<i>" / "f<i>" SpaceNet, "mc<i>" / "mf<i>" MotionNet), the points, in hit order, whose
            gradient reaches the weights (the rest are detached);
  flow_at   per performer call: evaluate the SpaceNet at xyz + flow_at[call] with the gradient through this run's own flow;
  kinks     a dict that receives, per network call, the points none of whose hidden pre-activations is near a ReLU kink;
  record    a dict that receives the flows and the SpaceNet outputs (per call) and the fine depths.
"""
from __future__ import annotations

import math

import torch

import test_composite_grad as CG
import test_gpu_nets_train as NT
from oracle import stnerf_oracle as O

F32 = torch.float32


def _ray_box(o, d, bmin, bmax):
    """layers/RaySamplePoint.py:8-62 in the dtype of o (the oracle's, dtype-generic)."""
    n = o.shape[0]
    eps = torch.tensor(2.220446049250313e-16, dtype=o.dtype, device=o.device)
    cand = torch.full((n, 6), -1000.0, dtype=o.dtype, device=o.device)
    col = 0
    for axis in range(3):
        a1, a2 = [a for a in range(3) if a != axis]
        for face in (bmin[..., axis], bmax[..., axis]):
            t = (face - o[:, axis]) / (d[:, axis] + eps)
            p = t[:, None] * d + o
            ok = (p[:, a1] >= bmin[..., a1]) & (p[:, a1] <= bmax[..., a1]) & (p[:, a2] >= bmin[..., a2]) & (p[:, a2] <= bmax[..., a2])
            cand[:, col] = torch.where(ok, t, cand[:, col])
            col += 1
    top = cand.topk(k=2, dim=-1)[0]
    return top[:, 0], top[:, 1]


def _sample(o, d, bmin, bmax, n1, jitter, is_bkgd):
    t_far, t_near = _ray_box(o, d, bmin, bmax)
    start = t_near.clone()
    if is_bkgd:
        start[start <= 0] = 0
    width = ((t_far - start) / n1)[:, None]
    k = torch.arange(0, n1, dtype=o.dtype, device=o.device)[None, :]
    t = (k + jitter) * width + start[:, None]
    return t, (width.abs() > 1e-5)[:, 0]


def _inverse_edit(xyz, i, scale, shift, pivot, fine):
    """layered_rfrender.py:293-303 (coarse) / :467-475 (fine: a None shift entry also skips the scale)."""
    if shift is not None:
        if shift[i] is None:
            if fine:
                return xyz
        else:
            xyz = xyz - torch.tensor(shift[i], dtype=xyz.dtype, device=xyz.device)
    if scale is not None:
        xyz = (xyz - pivot) / scale[i] + pivot
    return xyz


def scene(case, dtype=torch.float64):
    """cases.scene_for(case) with the boxes, their lerp, the edits and the pivot formed in `dtype` (layered_rfrender.py:190-242,
    :123-127 in the retiming branch; a per-frame table of edited boxes for 7-column mixed-frame rays, :193)."""
    import cases as C
    sc = dict(C.scene_for(case))
    bkgd, frames = C.boxes_for(case)
    bkgd, frames = bkgd.to(dtype).reshape(1, 8, 3), frames.to(dtype)
    scale, shift = case.get("scale"), case.get("shift")

    def resolve(frame_ids, lerp):
        boxes = [bkgd[0].clone()]
        for i in range(frames.shape[1]):
            f = torch.tensor(float(frame_ids[i + 1]), dtype=dtype) - 1
            lo, hi = frames[math.floor(f), i], frames[math.ceil(f), i]
            boxes.append(torch.lerp(lo, hi, f - math.floor(f)) if lerp else frames[int(f), i])
        boxes = torch.stack(boxes, 0)
        first = torch.cat([bkgd, frames[0]], 0)
        centre = first.mean(1)
        centre[:, 2] = first[:, 1, 2]
        pivot = None
        if scale is not None:
            pivot = (centre[2] + centre[1]) / 2
            for i in range(len(scale)):
                boxes[i] = (boxes[i] - pivot) * scale[i] + pivot
        if shift is not None:
            for i in range(len(shift)):
                if shift[i] is not None:
                    boxes[i] = boxes[i] + torch.tensor(shift[i], dtype=dtype)
        return boxes[:, 0, :].clone(), boxes[:, 6, :].clone(), pivot

    l = frames.shape[1] + 1
    ids = [case["frame_ids"][0]] * l if case.get("seven") else case["frame_ids"]
    sc["bmin"], sc["bmax"], sc["pivot"] = resolve(ids, not case.get("seven"))
    if case.get("mixed_frames"):
        rows = [resolve([0.0] + [float(f + 1)] * (l - 1), False)[:2] for f in range(frames.shape[0])]
        sc["box_table"] = torch.stack([torch.stack([lo, hi], 1) for lo, hi in rows], 0)
    return sc


def forward(p, scene, rays, n1, n2, jitter, u, only_coarse, thr, bthr, shared_frame, dtype, device,
            samples=None, fine_t=None, keep=None, flow_at=None, kinks=None, record=None):
    """p: state_dict-keyed parameters (any dtype / device; cast here).  scene: cases.scene_for(case).  Returns the 5-tuple."""
    dd = dict(dtype=dtype, device=device)
    rays32 = rays.to(device, F32)
    R = rays32.to(dtype)
    o, d = R[:, :3], R[:, 3:6]
    l = scene["bmin"].shape[0]
    N = rays.shape[0]
    fid = R[:, 6:7].expand(-1, l) if shared_frame else R[:, 6:]
    if shared_frame:
        thr = bthr = float("-inf")                                    # `if self.retiming` (:416,538,564)
    scale, shift = scene.get("scale"), scene.get("shift")
    pivot = None if scene.get("pivot") is None else scene["pivot"].to(**dd)
    shown = scene.get("shown", [True] * l)
    near, alpha2, boarder = float(scene.get("near", 0.0)), float(scene.get("alpha", 1.0)), float(scene.get("boarder", 1e10))
    flows, outputs = {}, {}

    def sub(prefix):
        return {k[len(prefix):]: v.to(**dd) for k, v in p.items() if k.startswith(prefix)}

    def gate(x, key):
        if keep is None or key not in keep:
            return x
        m = keep[key].to(device)[:, None]
        return torch.where(m, x, x.detach())

    def points(t, fine):
        """The marched points of depths t (N,S): in fp32 from fp32 depths (given samples), else in the run's dtype."""
        if samples is not None:
            return (t.to(F32)[..., None] * rays32[:, None, 3:6] + rays32[:, None, :3]).to(dtype)
        return t[..., None] * d[:, None, :] + o[:, None, :]

    def run_layer(i, t, masks, fine):
        S = t.shape[1]
        key = ("f" if fine else "c") + str(i)
        rgb = torch.zeros((N, S, 3), **dd)
        sig = torch.zeros((N, S), **dd)
        idx = torch.ones(N, dtype=torch.bool, device=device) if i == 0 else masks[i].to(device)
        M = int(idx.sum())
        if i > 0 and (M == 0 or not shown[i]):                        # :401 / :556
            return rgb, sig
        xyz = _inverse_edit(points(t, fine), i, scale, shift, pivot, fine)
        q = xyz[idx].reshape(-1, 3)
        dirs = d[idx][:, None, :].expand(M, S, 3).reshape(-1, 3)
        tcol = fid[idx, i][:, None, None].expand(M, S, 1).reshape(-1, 1)
        if i > 0:                                                     # :340-356 / :495-510
            w = sub("time_deform_nets.%d." % (i - 1))
            xyzt = torch.cat([q, tcol], 1)
            if kinks is not None:
                kinks["m" + key] = NT.kink_free(lambda: O.motionnet_forward(w, xyzt.detach()))
            flow = gate(O.motionnet_forward(w, xyzt), "m" + key)
            flows[key] = flow.detach()
            q = q + flow_at[key].to(**dd) + (flow - flow.detach()) if flow_at is not None else q + flow
            w = sub("spacenets%s.%d." % ("_fine" if fine else "", i - 1))
        else:
            w = sub("bkgd_spacenet%s." % ("_fine" if fine else ""))
        times = tcol if w["rgb_net.1.weight"].shape[1] == 256 + 27 + 21 else None
        if kinks is not None:
            kk = NT.kink_free(lambda: O.spacenet_forward(w, q.detach(), dirs, times), NT.KINK_CHAINED if i > 0 else NT.KINK)
            kinks[key] = kk if i == 0 else kk & kinks["m" + key]
            if i > 0:
                kinks["m" + key] = kinks[key]
        r, s = O.spacenet_forward(w, q, dirs, times)
        outputs[key] = (r.detach(), s.detach())
        r, s = gate(r, key), gate(s, key)
        rgb = rgb.index_put((idx,), r.reshape(M, S, 3))
        sig = sig.index_put((idx,), s.reshape(M, S))
        return rgb, sig

    # ---- coarse pass (:249-448) ---------------------------------------------------------------------------------------------
    if samples is not None:
        ts = [samples[0][i].to(device, F32).to(dtype) for i in range(l)]
        masks = [samples[1][i].to(device).bool() for i in range(l)]
    else:
        table = scene.get("box_table") if shared_frame else None
        row = (rays32[:, 6].to(torch.int64) - 1) if table is not None else None
        ts, masks = [], []
        for i in range(l):
            bmin = (scene["bmin"][i] if table is None else table[row.cpu(), i, 0]).to(**dd)
            bmax = (scene["bmax"][i] if table is None else table[row.cpu(), i, 1]).to(**dd)
            t, m = _sample(o, d, bmin, bmax, n1, jitter[i].to(**dd), i == 0)
            ts.append(t); masks.append(m)
    rgbs, sigs = [], []
    for i in range(l):
        rgb, sig = run_layer(i, ts[i], masks, False)
        if i > 0 and bool(masks[i].any()) and shown[i]:
            sig = torch.where(ts[i] < 0, torch.zeros_like(sig), sig)                     # :414
            sig = torch.where(sig < thr, torch.zeros_like(sig), sig)                     # :416-418
        elif i == 0:
            sig = torch.where(ts[0] < near, torch.zeros_like(sig), sig)                  # :422
        rgbs.append(rgb); sigs.append(sig)
    outs = [CG.composite_ref(ts[i], rgbs[i], sigs[i], boarder) for i in range(l)]
    coarse_layer = [x[:3] for x in outs]
    coarse_mixed = CG.merged_ref(ts, rgbs, sigs, boarder, None)
    if record is not None:
        record["flows"], record["outputs"] = flows, outputs
    if only_coarse:
        return coarse_mixed, coarse_mixed, coarse_layer, coarse_layer, masks
    # ---- fine pass (:453-606) -----------------------------------------------------------------------------------------------
    if fine_t is not None:
        tf = [fine_t[i].to(device, F32).to(dtype) for i in range(l)]
    else:
        tf = []
        for i in range(l):
            z = O.sample_pdf(ts[i].detach(), outs[i][3].detach()[:, 1:-1], u[i].to(**dd))
            tf.append(torch.sort(torch.cat([ts[i], z], -1), -1)[0])
    if record is not None:
        record["fine_t"] = [x.detach() for x in tf]
    rgbs, sigs = [], []
    for i in range(l):
        rgb, sig = run_layer(i, tf[i], masks, True)
        if i == 0:
            sig = torch.where(sig < bthr, torch.zeros_like(sig), sig)                    # :538-547
        elif bool(masks[i].any()) and shown[i]:
            sig = torch.where(sig < thr, torch.zeros_like(sig), sig)                     # :564-566
            if i == 2:
                sig = sig * alpha2                                                       # :575-576
        rgbs.append(rgb); sigs.append(sig)
    fine_layer = [CG.composite_ref(tf[i], rgbs[i], sigs[i], boarder)[:3] for i in range(l)]
    fine_mixed = CG.merged_ref(tf, rgbs, sigs, boarder, near)
    return fine_mixed, coarse_mixed, fine_layer, coarse_layer, masks
