"""A/B tool: run the SpaceNet / MotionNet entry points and one small coarse+fine render with the library selected by
STNERF_B200_LIB and dump every output to an .npz, so two builds of the kernel can be compared bit for bit
(`python scripts/dump_networks.py out.npz`, then `python scripts/dump_networks.py --compare a.npz b.npz`).
Synthetic weights and points only (no oracle, no reference): this is a build-vs-build tool."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "st-nerf_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    bad = 0
    for k in A.files:
        x, y = A[k], B[k]
        same = x.shape == y.shape and np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                                     y.view(np.uint32) if y.dtype == np.float32 else y)
        d = float(np.nanmax(np.abs(x.astype(np.float64) - y.astype(np.float64)))) if x.shape == y.shape and x.size else -1.0
        nan = int(np.isnan(x).sum() + np.isnan(y).sum()) if x.dtype.kind == "f" else 0
        print("%-28s %s  max|diff| %.3e  nan %d  n %d" % (k, "bit-identical" if same else "DIFFERENT", d, nan, x.size))
        bad += 0 if same else 1
    print("RESULT: %s" % ("all bit-identical" if bad == 0 else "%d arrays differ" % bad))
    return bad


def main(out):
    import torch
    import cases as C
    from oracle import stnerf_oracle as O      # synthetic weights only
    from stnerf_b200 import NativeRenderer
    from tests_support import run_case_native
    res = {}
    g = torch.Generator().manual_seed(7)
    n = 148 * 128 * 5 + 77                      # several tiles per CTA and a ragged tail
    pos = (torch.rand(n, 3, generator=g) * 4 - 2).cuda()
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1).cuda()
    tm = (torch.rand(n, generator=g) * 20).cuda()
    for prec in ("exact", "exact_cf", "mixed", "fast"):
        sd = O.synthetic_state_dict(1, True, seed=5)
        r = NativeRenderer(2, [False, True], prec)
        r.load_state_dict(sd)
        rgb, sig = r.spacenet(1, False, pos, dirs, tm)
        res["%s.perf.rgb" % prec], res["%s.perf.sigma" % prec] = rgb.cpu().numpy(), sig.cpu().numpy()
        rgb, sig = r.spacenet(0, True, pos, dirs, None)
        res["%s.bkgd.rgb" % prec], res["%s.bkgd.sigma" % prec] = rgb.cpu().numpy(), sig.cpu().numpy()
        flow = r.motionnet(1, torch.cat([pos, tm[:, None]], 1))
        res["%s.flow" % prec] = flow.cpu().numpy()
        r.close()
    # small coarse + fine renders (fused coarse compositing, flow reuse, fine pass); exact_cf adds the corrections first in
    # the coarse pass and the MotionNets, interleaved in the fine pass
    for name, prec in (("syn_L2_64_128", "exact"), ("tkd_edit_frac", "exact"), ("syn_L2_64_128", "exact_cf")):
        if name not in C.CASES:
            continue
        flat = run_case_native(name, prec)
        if flat is None:
            continue
        tag = name if prec == "exact" else "%s.%s" % (name, prec)
        for k, v in flat.items():
            v = np.asarray(v)
            res["%s.%s" % (tag, k)] = v.astype(np.float32) if v.dtype.kind == "f" else v
    for k, v in res.items():
        if v.dtype.kind == "f" and not np.isfinite(v).all():
            print("WARNING: non-finite values in", k)
    np.savez(out, **res)
    print("wrote %s (%d arrays)" % (out, len(res)))


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(1 if compare(sys.argv[2], sys.argv[3]) else 0)
    main(sys.argv[1])
