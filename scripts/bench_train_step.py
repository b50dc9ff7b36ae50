#!/usr/bin/env python
"""One training step of the layered model on the native path (stnerf_b200.train) against a torch fp32 restatement.

    python scripts/bench_train_step.py [--warmup 3] [--iters 10]

Workload: the taekwondo training configuration -- 2000 rays per batch (SOLVER.BUNCH), 7-column rays with mixed integer frame
ids (boxes per ray by frame), 2 performers, 90 + 30 samples, synthetic weights of the shipped shapes.  A step = forward +
the trainer's loss (layered_trainer.py:216-281, mask losses on) + backward + Adam, in the fine stage and in the coarse stage
(`only_coarse`, COARSE_STAGE).  The torch restatement (TF32 off) takes the same sample depths and hit masks (sampling is
not part of it) and runs networks, scatter, composites, the merged composites and the loss in torch autograd, with the fine
depths from the same native sample_pdf; the two are alternated in one run.  Printed: ms per step and rays/s for both, the
share of the native step spent in the network kernels (a separate torch.profiler run), peak device memory, and the card's
name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "st-nerf_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases as C  # noqa: E402
from oracle import stnerf_oracle as O  # noqa: E402
from stnerf_b200 import ops  # noqa: E402
from tests_support import make_cfg  # noqa: E402

N_RAYS, N1, N2, LAYERS = 2000, 90, 30, 2
MASK_SCALAR = 100000.0
LR = 4e-4
# the kernels of csrc/mlp_train.cu and mlp_train_tc.cu (SpaceNet / MotionNet training forward and backward)
NETWORK_KERNELS = ("gemm_kernel", "tc_gemm_kernel", "reduce_partials_kernel", "rowsum_chunks_kernel", "rowsum_tree_kernel",
                   "spacenet_encode_kernel", "motionnet_encode_kernel", "spacenet_dpos_kernel")


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def trainer_loss(out, rays, labels, target, only_coarse):
    """layered_trainer.py:216-281 with REMOVE_OUTLIERS (epoch < 3) and its `scalar` rule."""
    fine_mixed, coarse_mixed, fine_layer, coarse_layer, _ = out
    loss1 = torch.nn.functional.mse_loss(coarse_mixed[0], target)
    loss2 = torch.nn.functional.mse_loss(fine_mixed[0], target)
    masks = []
    for stage in (coarse_layer, fine_layer):
        outl = torch.cat([stage[i][2][labels == 0] for i in range(1, len(stage))], 0)
        inl = torch.cat([stage[i][2][labels == i] for i in range(len(stage))], 0)
        m = outl.abs().sum() + (1 - inl).abs().sum()
        masks.append(m / MASK_SCALAR if float(m.detach()) > rays.shape[0] * 0.0005 else torch.zeros((1,), device=target.device))
    return loss1 + masks[0] if only_coarse else loss1 + loss2 + masks[0] + masks[1]


def torch_forward(p, rays, t_c, mask, u, only_coarse, near, boarder=1e10):
    """layered_rfrender.py:141-734 restated in torch (7-column rays: no thresholds), on given coarse depths and masks."""
    o, d, fid = rays[:, :3], rays[:, 3:6], rays[:, 6:7]
    N, l = rays.shape[0], t_c.shape[0]

    def sub(prefix):
        return {k[len(prefix):]: v for k, v in p.items() if k.startswith(prefix)}

    def comp(t, rgb, sigma):
        delta = torch.cat([t[:, 1:] - t[:, :-1], torch.full((t.shape[0], 1), boarder, device=t.device)], -1)
        alpha = 1.0 - torch.exp(-torch.relu(sigma) * delta)
        trans = torch.cumprod(torch.cat([torch.ones((t.shape[0], 1), device=t.device), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
        w = alpha * trans
        return (torch.sigmoid(rgb) * w[..., None]).sum(1), (w * t).sum(1, keepdim=True), w.sum(1, keepdim=True), w

    def merged(ts, rgbs, sigmas, near_):
        tm, order = torch.sort(torch.cat(ts, 1), dim=1, stable=True)
        rm = torch.cat(rgbs, 1).gather(1, order[..., None].expand(-1, -1, 3))
        sm = torch.cat(sigmas, 1).gather(1, order)
        if near_ is not None:
            sm = torch.where(tm < near_, torch.zeros_like(sm), sm)
        return comp(tm, rm, sm)[:3]

    def run_pass(ts, fine):
        rgbs, sigmas, outs = [], [], []
        for i in range(l):
            t = ts[i]
            S = t.shape[1]
            idx = mask[i] if i > 0 else torch.ones(N, dtype=torch.bool, device=t.device)
            M = int(idx.sum())
            rgb = torch.zeros((N, S, 3), device=t.device)
            sig = torch.zeros((N, S), device=t.device)
            if M > 0:
                xyz = (t[idx][..., None] * d[idx][:, None, :] + o[idx][:, None, :]).reshape(-1, 3)
                dirs = d[idx][:, None, :].expand(M, S, 3).reshape(-1, 3)
                tm = fid[idx][:, None, :].expand(M, S, 1).reshape(-1, 1)
                sfx = "_fine" if fine else ""
                if i > 0:
                    xyz = xyz + O.motionnet_forward(sub("time_deform_nets.%d." % (i - 1)), torch.cat([xyz, tm], 1))
                    w = sub("spacenets%s.%d." % (sfx, i - 1))
                else:
                    w = sub("bkgd_spacenet%s." % sfx)
                use_time = w["rgb_net.1.weight"].shape[1] == 256 + 27 + 21
                r, s = O.spacenet_forward(w, xyz, dirs, tm if use_time else None)
                rgb = rgb.index_put((idx,), r.reshape(M, S, 3))
                sig = sig.index_put((idx,), s.reshape(M, S))
            if not fine:
                sig = torch.where(t < (0.0 if i > 0 else near), torch.zeros_like(sig), sig)
            rgbs.append(rgb); sigmas.append(sig)
            outs.append(comp(t, rgb, sig))
        return outs, merged(ts, rgbs, sigmas, near if fine else None)

    ts = [t_c[i] for i in range(l)]
    outs_c, mixed_c = run_pass(ts, False)
    layer_c = [x[:3] for x in outs_c]
    if only_coarse:
        return mixed_c, mixed_c, layer_c, layer_c, None
    tf = [ops.sample_pdf(ts[i], outs_c[i][3].detach(), u[i], merge=True)[1] for i in range(l)]
    outs_f, mixed_f = run_pass(tf, True)
    return mixed_f, mixed_c, [x[:3] for x in outs_f], layer_c, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--train-precision", choices=["fp32", "tf32x3"], default="fp32", help="precision of the native networks")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    card, watts = torch.cuda.get_device_name(dev), power_limit()
    print("# %s, power limit %s W; training step, %d rays, %d performers, %d + %d samples, native networks in %s"
          % (card, "%.0f" % watts if watts else "unknown", N_RAYS, LAYERS, N1, N2, args.train_precision))
    import modeling
    case = dict(C.CASES["tkd_train_7col_mixed"], n_rays=N_RAYS, ray_seed=31, n1=N1, n2=N2)
    cfg = make_cfg(LAYERS, N1, N2, True, "fp32")
    cfg.MODEL.B200_TRAINABLE = True
    cfg.MODEL.B200_TRAIN_PRECISION = args.train_precision
    model = modeling.build_layered_model(cfg, 0, None, None)
    model.load_state_dict(O.synthetic_state_dict(LAYERS, True, seed=3))
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model.cuda()
    rays = C.rays_for(case).to(dev)
    g = torch.Generator().manual_seed(5)
    target = torch.rand((N_RAYS, 3), generator=g).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=LR)
    ref_p = {k: v.detach().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ref_opt = torch.optim.Adam(list(ref_p.values()), lr=LR)
    with torch.no_grad():
        out = model(rays, None, None, False)
    labels = out[4][1].long() + 2 * (out[4][2] & ~out[4][1]).long()

    # the restatement's depths and hit masks: the model's own sampling, seen through its `trace` hook
    l = LAYERS + 1
    seen = {}
    model.trace = lambda name, x: seen.__setitem__(name, x.detach().clone()) if name in ("t_coarse", "mask") else None
    model(rays, None, None, True)
    model.trace = None
    t_c, mask = seen["t_coarse"], seen["mask"].bool()
    u = torch.rand((l, N_RAYS, N2), generator=g).to(dev)

    def native_step(only_coarse):
        def run():
            opt.zero_grad()
            loss = trainer_loss(model(rays, labels, None, only_coarse), rays, labels, target, only_coarse)
            loss.backward()
            opt.step()
        return run

    def torch_step(only_coarse, tf32=False):
        def run():
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ref_opt.zero_grad()
            out = torch_forward(ref_p, rays, t_c, mask, u, only_coarse, 0.0)
            loss = trainer_loss(out, rays, labels, target, only_coarse)
            loss.backward()
            ref_opt.step()
            torch.backends.cuda.matmul.allow_tf32 = False
        return run

    def time_ms(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    rows = []
    for stage, only_coarse in (("fine", False), ("coarse", True)):
        times = {"native": [], "torch": [], "torch_1xtf32": []}
        for _ in range(2):                                       # alternated
            torch.cuda.reset_peak_memory_stats(dev)
            times["native"].append(time_ms(native_step(only_coarse)))
            peak_native = torch.cuda.max_memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            times["torch"].append(time_ms(torch_step(only_coarse)))
            peak_torch = torch.cuda.max_memory_allocated(dev)
            # context only: torch with TF32 matmuls (one tf32 product per term, less accurate than tf32x3)
            times["torch_1xtf32"].append(time_ms(torch_step(only_coarse, tf32=True)))
        nat_ms, ref_ms, tf32_ms = min(times["native"]), min(times["torch"]), min(times["torch_1xtf32"])
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            native_step(only_coarse)()
            torch.cuda.synchronize()
        net_us = tot_us = 0.0
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", 0.0)
            tot_us += us
            if any(k in e.key for k in NETWORK_KERNELS):
                net_us += us
        row = dict(stage=stage, train_precision=args.train_precision, native_ms=round(nat_ms, 3), torch_ms=round(ref_ms, 3),
                   torch_1xtf32_ms=round(tf32_ms, 3),
                   native_rays_per_s=round(N_RAYS / nat_ms * 1e3), torch_rays_per_s=round(N_RAYS / ref_ms * 1e3),
                   network_share=round(net_us / tot_us, 3) if tot_us else None,
                   peak_mem_native_gb=round(peak_native / 2 ** 30, 2), peak_mem_torch_gb=round(peak_torch / 2 ** 30, 2),
                   hits=[int(x) for x in mask.sum(1)])
        rows.append(row)
        print("%-6s native %.2f ms (%.0f rays/s), torch %.2f ms (%.0f rays/s), torch 1xTF32 %.2f ms; networks %.0f %% of native "
              "device time; peak %.2f / %.2f GB" % (stage, nat_ms, row["native_rays_per_s"], ref_ms, row["torch_rays_per_s"], tf32_ms,
                                                    100 * (row["network_share"] or 0), row["peak_mem_native_gb"],
                                                    row["peak_mem_torch_gb"]))
        if stage == "fine":
            print("# kernels of one native step:")
            for e in sorted(prof.key_averages(), key=lambda e: -getattr(e, "device_time_total", 0))[:12]:
                print("#   %8.1f us  %s" % (getattr(e, "device_time_total", 0), e.key[:100]))
    print(json.dumps({"card": card, "power_limit_w": watts, "rows": rows}))


if __name__ == "__main__":
    main()
