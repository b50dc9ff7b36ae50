#!/usr/bin/env python
"""Run the UNMODIFIED reference `LayeredRFRender.forward` (modeling/layered_rfrender.py:141) on CPU, in its own process.

TEST INFRASTRUCTURE ONLY.  The native facade packages reuse the reference's top-level import names (`modeling`, `utils`,
`layers`, `engine`), so reference code can never share an interpreter with them: the gpu parity tests and `bench.py` talk to
the reference through this command-line program.

    python oracle/run_reference.py --in job.pt --out result.pt [--threads T] [--workers W] [--time-only]

`job.pt` (torch.save of a dict):
    sd            reference-format state_dict                  L, space_time, n1, n2
    bkgd (1,8,3), frames (F,L,8,3) boxes                       rays (N, 6+l | 7)     jitter (l,N,n1)     u (l,N,n2) | None
    thr (density, bkgd)   near   alpha   hidden [layer ids]   shift   scale   only_coarse
  optional:
    record        True: also return what `sample_pdf` (utils/sample_pdf.py:18-63) saw and produced per layer:
                  z (l,N,n2), denom (l,N,n2) BEFORE the `denom<1e-5 -> 1` branch (:59), bin_lo / bin_hi (l,N,n2) = the two bin
                  centres the sample is interpolated between (:61), cdf_hi (l,N,n2), t_coarse (l,N,n1)
    z_override    (l,N,n2): `sample_pdf` returns these depths instead of its own (the reference's fine pass then runs on
                  exactly the sample positions another implementation chose)
    perturb_seed  int: multiply every coarse weight handed to `sample_pdf` by (1 + s*perturb_rel), s = -1/0/+1 drawn per
                  element from this seed; perturb_rel defaults to 2^-23 (a +-1-ulp perturbation of the resampling input)
    sigma_scale   float: multiply the density every SpaceNet returns (modeling/spacenet.py:139) by this factor -- a coherent
                  relative perturbation of all densities, coarse and fine
    variants      list of dicts, each overriding some of {perturb_seed, perturb_rel, thr, z_override, record}: run the SAME rays
                  once per variant in this one process; the result is {"variants": [result dict per variant]}
    multi         list of {rays, jitter, u}: time SEVERAL inputs in one process (bench.py's steps: one interpreter start-up for
                  the whole run); the result then carries "seconds_each" (per input) and the outputs of the last input only
`result.pt`: {"flat": cases.flatten_outputs schema (numpy), "seconds": wall time of the forward calls, "threads": T, ...}.

Rays are processed in chunks of 3584 like `layered_batchify_ray` (utils/batchify_rays.py:57); `--workers W` splits the rays
over W child processes of this same program (the reference has no cross-ray coupling beyond ray 0's frame ids, SURVEY C.6).
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHUNK = 512 * 7


def _slice_job(job, a, b):
    out = dict(job)
    if "multi" in job:                     # slice every input the same way (relative bounds: a, b are fractions here)
        out["multi"] = [_slice_job(dict(rays=m["rays"], jitter=m["jitter"], u=m.get("u")),
                                   int(a * m["rays"].shape[0]), int(b * m["rays"].shape[0])) for m in job["multi"]]
        return out
    out["rays"] = job["rays"][a:b].clone()
    out["jitter"] = job["jitter"][:, a:b].clone()
    for k in ("u", "z_override"):
        if job.get(k) is not None:
            out[k] = job[k][:, a:b].clone()
    out["ray_base"] = job.get("ray_base", 0) + a
    return out


def _cat_results(parts):
    import numpy as np
    flat = {k: np.concatenate([p["flat"][k] for p in parts], 0) for k in parts[0]["flat"]}
    out = {"flat": flat, "seconds": max(p["seconds"] for p in parts), "cpu_seconds_sum": sum(p["seconds"] for p in parts),
           "threads": sum(p["threads"] for p in parts), "rays": sum(p["rays"] for p in parts)}
    if "record" in parts[0]:
        out["record"] = {k: np.concatenate([p["record"][k] for p in parts], 1) for k in parts[0]["record"]}
    return out


def run_workers(job, workers, threads):
    import torch
    multi = "multi" in job
    n = 0 if multi else job["rays"].shape[0]
    per = (n + workers - 1) // workers
    tmp = tempfile.mkdtemp(prefix="stnerf_refjob_")
    procs = []
    for w in range(workers):
        a, b = (w / workers, (w + 1) / workers) if multi else (w * per, min(n, (w + 1) * per))
        if a >= b:
            break
        jin, jout = os.path.join(tmp, "in%d.pt" % w), os.path.join(tmp, "out%d.pt" % w)
        torch.save(_slice_job(job, a, b), jin)
        procs.append((subprocess.Popen([sys.executable, os.path.abspath(__file__), "--in", jin, "--out", jout,
                                        "--threads", str(max(1, threads // workers))]), jout))
    parts = []
    for p, jout in procs:
        if p.wait() != 0:
            raise RuntimeError("reference worker failed")
        parts.append(torch.load(jout, weights_only=False))
    import shutil
    shutil.rmtree(tmp, ignore_errors=True)
    if multi:
        k = len(parts[0]["seconds_each"])
        return {"seconds_each": [max(p["seconds_each"][i] for p in parts) for i in range(k)],
                "rays_each": [sum(p["rays_each"][i] for p in parts) for i in range(k)], "threads": sum(p["threads"] for p in parts)}
    return _cat_results(parts)


def flatten_outputs(fine_mixed, coarse_mixed, fine_layer, coarse_layer, ray_mask) -> dict:
    """The .npz schema of tests/golden/cases.py::flatten_outputs (kept local: this process must not import the facade tree)."""
    import numpy as np
    d = {}
    f32 = lambda v: np.asarray(v.detach().cpu().reshape(v.shape[0], -1), dtype=np.float32)  # noqa: E731
    for name, trip in (("fine_mixed", fine_mixed), ("coarse_mixed", coarse_mixed)):
        for part, v in zip(("rgb", "depth", "acc"), trip):
            d["%s.%s" % (name, part)] = f32(v)
    for name, lst in (("fine_layer", fine_layer), ("coarse_layer", coarse_layer)):
        for i, trip in enumerate(lst):
            for part, v in zip(("rgb", "depth", "acc"), trip):
                d["%s.%d.%s" % (name, i, part)] = f32(v)
    for i, m in enumerate(ray_mask):
        d["ray_mask.%d" % i] = np.asarray(m.detach().cpu()).astype(np.uint8)
    return d


def run_single(job, threads):
    import numpy as np
    import torch
    torch.set_num_threads(threads)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import reference_shim as R
    m = R.modules()
    import modeling.layered_rfrender as LR          # the reference module whose `sample_pdf` name the wrapper replaces

    model = R.build_model(job["sd"], job["L"], job["n1"], job["n2"], job["space_time"], job["bkgd"], job["frames"],
                          scale=job.get("scale"), shift=job.get("shift"))
    model.near = job.get("near", 0.0)
    model.alpha = job.get("alpha", 1.0)
    for i in job.get("hidden", []):
        model.hide_layer(i)
    if "multi" in job:                      # several inputs, timed one after the other in this one process
        secs, counts = [], []
        for m in job["multi"]:
            sub = dict(job); sub.pop("multi"); sub.update(rays=m["rays"], jitter=m["jitter"], u=m.get("u"))
            r = _run_inputs(sub, model, R, LR, torch, np)
            secs.append(r["seconds"]); counts.append(int(m["rays"].shape[0]))
        return {"seconds_each": secs, "rays_each": counts, "threads": threads}
    if "variants" in job:                   # the same rays under several perturbations / overrides, one process
        outs = []
        for var in job["variants"]:
            sub = dict(job); sub.pop("variants"); sub.update(var)
            outs.append(_run_inputs(sub, model, R, LR, torch, np))
        return {"variants": outs, "threads": threads}
    res = _run_inputs(job, model, R, LR, torch, np)
    res["threads"] = threads
    return res


def _run_inputs(job, model, R, LR, torch, np):
    rays, jit, u = job["rays"], job["jitter"], job.get("u")
    only_coarse = bool(job.get("only_coarse", False))
    record = bool(job.get("record", False))
    z_over = job.get("z_override")
    pseed = job.get("perturb_seed")
    n, l = rays.shape[0], job["L"] + 1
    rec = {k: [[] for _ in range(l)] for k in ("z", "denom", "bin_lo", "bin_hi", "cdf_hi", "t_coarse")} if record else None
    real_sample_pdf = LR.sample_pdf
    state = {"layer": 0, "c0": 0, "c1": 0}

    def wrapped(z_vals, weights, N_samples, det=False, pytest=False):
        i = state["layer"]
        state["layer"] += 1
        if pseed is not None:
            g = torch.Generator().manual_seed(int(pseed) * 1000003 + (job.get("ray_base", 0) + state["c0"]) * 31 + i)
            s = torch.randint(-1, 2, weights.shape, generator=g).to(weights.dtype)
            weights = weights * (1.0 + s * float(job.get("perturb_rel", 2.0 ** -23)))
        z = real_sample_pdf(z_vals, weights, N_samples, det=det, pytest=pytest)
        if record:
            # what utils/sample_pdf.py:20-61 computed on the way (same ops, same order; torch.rand pops the SAME u again
            # because the injection queue is re-primed below)
            uu = state["u_now"][i]
            bins = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
            w = weights + 1e-5
            pdf = w / torch.sum(w, -1, keepdim=True)
            cdf = torch.cumsum(pdf, -1)
            cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
            inds = torch.searchsorted(cdf, uu.contiguous(), right=True)
            below = torch.clamp(inds - 1, min=0)
            above = torch.clamp(inds, max=cdf.shape[-1] - 1)
            cg0, cg1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
            rec["z"][i].append(z.clone()); rec["denom"][i].append(cg1 - cg0)
            rec["bin_lo"][i].append(torch.gather(bins, 1, below)); rec["bin_hi"][i].append(torch.gather(bins, 1, above))
            rec["cdf_hi"][i].append(cg1); rec["t_coarse"][i].append(z_vals.clone())
        if z_over is not None:
            z = z_over[i, state["c0"]:state["c1"]].to(z.dtype).clone()
        return z

    LR.sample_pdf = wrapped
    sig_scale = job.get("sigma_scale")
    hooks = []
    if sig_scale is not None:
        def scale_density(_m, _inp, out):
            return (out[0], out[1] * float(sig_scale))
        nets = [model.bkgd_spacenet, model.bkgd_spacenet_fine] + list(model.spacenets) + list(model.spacenets_fine)
        hooks = [n_.register_forward_hook(scale_density) for n_ in nets]
    outs, secs = [], 0.0
    try:
        for c0 in range(0, n, CHUNK):
            c1 = min(n, c0 + CHUNK)
            state.update(layer=0, c0=c0, c1=c1, u_now=None if u is None else u[:, c0:c1])
            t0 = time.perf_counter()
            out = R.forward(model, rays[c0:c1], jit[:, c0:c1], None if u is None else u[:, c0:c1], only_coarse=only_coarse,
                            density_threshold=job["thr"][0], bkgd_density_threshold=job["thr"][1])
            secs += time.perf_counter() - t0
            outs.append(out)
    finally:
        LR.sample_pdf = real_sample_pdf
        for h in hooks:
            h.remove()
    # concatenate the 5-tuples of the chunks (what layered_batchify_ray does, utils/batchify_rays.py:84-140)
    def cat_trip(get):
        return tuple(torch.cat([get(o)[k] for o in outs], 0) for k in range(3))
    fine_mixed, coarse_mixed = cat_trip(lambda o: o[0]), cat_trip(lambda o: o[1])
    fine_layer = [cat_trip(lambda o, i=i: o[2][i]) for i in range(l)]
    coarse_layer = [cat_trip(lambda o, i=i: o[3][i]) for i in range(l)]
    ray_mask = [torch.cat([o[4][i].reshape(-1) for o in outs], 0) for i in range(l)]
    res = {"flat": flatten_outputs(fine_mixed, coarse_mixed, fine_layer, coarse_layer, ray_mask), "seconds": secs,
           "rays": n, "reference_root": R.REFERENCE_ROOT}
    if record:
        res["record"] = {k: np.stack([torch.cat(v[i], 0).numpy() for i in range(l)], 0) for k, v in rec.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--in", dest="inp", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--workers", type=int, default=1)
    args = ap.parse_args()
    import torch
    threads = args.threads if args.threads > 0 else (os.cpu_count() or 1)
    job = torch.load(args.inp, weights_only=False)
    res = run_workers(job, args.workers, threads) if args.workers > 1 else run_single(job, threads)
    torch.save(res, args.out)


if __name__ == "__main__":
    main()
