"""Parity at scale against the UNMODIFIED reference (BASELINE configs[1], configs[2] and the 64+192 sampling of configs[4]).

The committed fixtures `tests/golden/scale_*.npz` hold the reference's own fine images for 16 384 (4 096) rays of a full-size
view (`tests/golden/make_golden_scale.py`).  The tensor-core modes `exact` and `mixed` must match them within the north-star
gate (pixel RGB and opacity within 1e-3) on at least 99.8 % of the rays, with a median error below 5e-5 -- and EVERY ray over
the gate must be attributed to an instability of the reference itself, or the test fails.

Why a few rays exceed the gate (`tests/tools/net_error_probe.py` measures it): the tensor core does not round its fp32
accumulation like an fp32 FFMA chain (`stnerf_selftest_umma_accum`), so the fp16x3 split reproduces sigma slightly less
closely than the reference's own fp32 GEMMs do.  Two steps of the reference amplify such differences without bound:
  * `utils/sample_pdf.py:58-61`: a fine depth is `bin_lo + (u - cdf_lo) / denom * width`; where the coarse pdf of a bin is tiny
    (empty space in front of / behind a surface: denom ~ 1e-5 .. 1e-3) a 1e-6 change of the cdf moves the sample by a visible
    fraction of the bin, and the fine network is steep there;
  * `modeling/layered_rfrender.py:416-418, 538-547, 564-566`: densities below a threshold are zeroed (walking: 20 / 0.8).
Attribution, per ray over the gate (reference re-run out of process from the archive packed by oracle/stash_reference.py):
  A  the reference, re-run with ITS fine depths replaced by the ones the native path chose, reproduces the native pixel (measured:
     to ~1e-6; asserted: a quarter of the gate) -- fine networks, thresholds and compositing agree exactly, the whole difference
     is where the fine samples were placed; and those placements are the reference's own up to its conditioning: every fine
     depth matches the reference's within the shift a cdf change of 1e-4 produces (`|dz| * denom / bin_width <= 1e-4`;
     samples on the `denom < 1e-5` branch point excepted).  A 1.5e-4 shift of ONE sample is enough to flip a pixel by 3e-2 when
     the fine density there sits on a threshold (walking 6-layer, ray 3608).
  or
  C  the reference's OWN pixel moves by more than a quarter of the gate under perturbations of the size of the measured
     disagreement: every density scaled by 1 +- 3e-5 (coherent, like the truncation bias; this also moves densities across the
     thresholds), or the coarse weights it resamples from perturbed by a random relative +-1e-5 (four seeds), while at least
     95 % of ordinary rays move by less than that.
A ray over the gate with neither is a bug and fails the test.  `mixed` (single fp16 pass on the colour-only layer, opt-in)
is held to the same rules except that its colour-only error on per-layer images may reach 2.5e-3 on at most 0.05 % of rays.
"""
import json
import os

import numpy as np
import pytest
import torch

import cases as C
from tests_support import build_case_model

GATE = 1e-3
MAX_OUTLIER_FRACTION = {False: 2e-3, True: 5e-3}     # without / with density thresholds (walking: 20 / 0.8 zero densities below them)
UNSTABLE = GATE / 4
PERTURB_REL = 1e-5
SIGMA_REL = 3e-5                     # ~4 x the rms disagreement of the densities measured by tests/tools/net_error_probe.py
SEEDS = (1, 2, 3, 4)
MAX_ATTRIBUTED = 96                  # rays re-run through the reference per mode (all outliers in every shipped case)
N_CONTROL = 48
_cache = {}


def _render(model, rays, jit, u, case):
    dev = torch.device("cuda", 0)
    model.inject_uniforms(jit.to(dev).contiguous(), u.to(dev).contiguous())
    with torch.no_grad():
        out = model(rays.to(dev), torch.zeros(rays.shape[0], device=dev), None, density_threshold=case["thr"][0],
                    bkgd_density_threshold=case["thr"][1])
    torch.cuda.synchronize()
    return C.flatten_outputs(*out)


def _err(flat, gold, l):
    """Per ray: max |rgb - gold| over the fine mixed image and every fine layer image, and |acc - gold| of the mixed image."""
    err = np.abs(flat["fine_mixed.rgb"] - gold["fine_mixed.rgb"]).max(1)
    for i in range(l):
        err = np.maximum(err, np.abs(flat["fine_layer.%d.rgb" % i] - gold["fine_layer.%d.rgb" % i]).max(1))
    return np.maximum(err, np.abs(flat["fine_mixed.acc"] - gold["fine_mixed.acc"]).max(1))


def _z_from_merged(t_fine, t_coarse):
    """The n2 resampled depths = sorted fine depths minus the (bit-identical) coarse depths, as a sorted array."""
    keep = np.ones(t_fine.shape[0], dtype=bool)
    pos = 0
    for v in t_coarse:
        while pos < t_fine.shape[0] and (t_fine[pos] != v or not keep[pos]):
            pos += 1
        assert pos < t_fine.shape[0], "a coarse depth is missing from the fine depths"
        keep[pos] = False
        pos += 1
    return t_fine[keep]


BAND = 16 * 2.0 ** -24               # cumsum round-off reach around the 1e-5 branch point of utils/sample_pdf.py:59
CDF_EPS = 1e-4                       # agreement of the coarse cdfs the placement check allows for


def _placement_implied_dcdf(z_gpu, z_ref, denom, lo, hi):
    """max over the samples of one (ray, layer) of |dz| * denom / bin_width: the cdf difference that explains the shift."""
    order = np.argsort(z_ref, kind="stable")
    z_ref, denom, lo, hi = z_ref[order], denom[order], lo[order], hi[order]
    band = np.abs(denom - 1e-5) <= BAND
    near_band = band.copy()
    for sft in (1, 2):                   # a moved branch-point sample shifts its neighbours' sorted positions
        near_band[sft:] |= band[:-sft]
        near_band[:-sft] |= band[sft:]
    width = np.maximum(np.abs(hi - lo), 1e-12)
    den_eff = np.where(denom < 1e-5, 1.0, denom)
    implied = np.abs(z_gpu - z_ref) * den_eff / width
    ok = ~near_band
    return float(implied[ok].max()) if ok.any() else 0.0


def attribute_outliers(case, model, rays, jit, u, idx, flat_full, mixed=False):
    """Criteria A / B / C for the rays `idx`.  Returns a report dict; raises AssertionError on an unattributed ray."""
    l, n1, n2 = case["L"] + 1, case["n1"], case["n2"]
    idx = np.asarray(sorted(set(int(i) for i in idx)))[:MAX_ATTRIBUTED]
    ctrl = np.setdiff1d(np.linspace(0, rays.shape[0] - 1, N_CONTROL).astype(np.int64), idx)
    sel = torch.as_tensor(np.concatenate([idx, ctrl]))
    no = idx.size
    r_s, j_s, u_s = rays[sel], jit[:, sel].contiguous(), u[:, sel].contiguous()
    sub = _render(model, r_s, j_s, u_s, case)
    nat = model._ensure_native(torch.device("cuda", 0))
    n = sel.numel()
    tc = [nat.read_depths(False, i, n, n1).cpu().numpy() for i in range(l)]
    tf = [nat.read_depths(True, i, n, n1 + n2).cpu().numpy() for i in range(l)]
    # rays are independent: the sub-render reproduces the pixels of the full render
    assert np.abs(sub["fine_mixed.rgb"] - flat_full["fine_mixed.rgb"][sel.numpy()]).max() <= 2e-6
    key = (case["name"], tuple(idx.tolist()), tuple(np.concatenate([t.reshape(-1) for t in tf])[::97].tolist()))
    if key in _cache:                    # `mixed` places its samples exactly like `exact`: same reference runs
        base, var = _cache[key]
    else:
        base = C.run_reference_job(C.reference_job(case, r_s, j_s, u_s, record=True))
        rec = base["record"]
        z_over = torch.from_numpy(rec["z"].copy())
        for i in range(l):
            for r in range(n):
                if base["flat"]["ray_mask.%d" % i][r] and not (i > 0 and i in case.get("hidden", [])):
                    assert np.array_equal(tc[i][r], rec["t_coarse"][i][r]), "coarse depths differ (layer %d)" % i
                    z_over[i, r] = torch.from_numpy(_z_from_merged(tf[i][r], tc[i][r]))
        variants = [dict(z_override=z_over)]
        variants += [dict(sigma_scale=1.0 + SIGMA_REL), dict(sigma_scale=1.0 - SIGMA_REL)]
        variants += [dict(perturb_seed=sd_, perturb_rel=PERTURB_REL) for sd_ in SEEDS]
        var = C.run_reference_job(C.reference_job(case, r_s, j_s, u_s, variants=variants))["variants"]
        _cache[key] = (base, var)
    ref, rec = base["flat"], base["record"]
    on_native_depths = _err(sub, var[0]["flat"], l)
    score = np.max([_err(v["flat"], ref, l) for v in var[1:]], axis=0)       # how far the reference itself moves
    implied = np.zeros(n)
    for r in range(no):
        for i in range(l):
            if ref["ray_mask.%d" % i][r] and not (i > 0 and i in case.get("hidden", [])):
                implied[r] = max(implied[r], _placement_implied_dcdf(_z_from_merged(tf[i][r], tc[i][r]), rec["z"][i][r], rec["denom"][i][r],
                                                                      rec["bin_lo"][i][r], rec["bin_hi"][i][r]))
    dump = os.path.join(C.ROOT, "gpurun_out")
    if os.path.isdir(dump):              # raw material for offline analysis (scratch, not asserted on)
        np.savez_compressed(os.path.join(dump, "attrib_%s_%s.npz" % (case["name"], model.precision)), sel=sel.numpy(), n_out=no, score=score,
                            on_native_depths=on_native_depths, implied=implied, **{"tc%d" % i: tc[i] for i in range(l)},
                            **{"tf%d" % i: tf[i] for i in range(l)}, **{"sub." + k: v for k, v in sub.items()}, **{"ref." + k: v for k, v in ref.items()})
    labels, unattributed = [], []
    for r in range(no):
        A = on_native_depths[r] <= UNSTABLE and implied[r] <= CDF_EPS
        Cc = score[r] > UNSTABLE
        labels.append("placement" if A else ("unstable" if Cc else "unattributed"))
        if not (A or Cc):
            unattributed.append((int(idx[r]), float(_err(sub, ref, l)[r]), float(on_native_depths[r]), float(score[r])))
    if mixed:        # colour precision of the single-pass layer: small, rare, colour only (acc / depth untouched by construction)
        assert len(unattributed) <= 5e-4 * rays.shape[0] and all(e[1] <= 2.5e-3 for e in unattributed), unattributed
    else:
        assert not unattributed, "rays over the gate that are neither placement-explained nor unstable in the reference: %s" % unattributed
    assert (score[no:] < UNSTABLE).mean() >= 0.95, "ordinary rays are unstable too: %s" % np.sort(score[no:])[-5:]
    return {"rays_attributed": int(no), "labels": {k: labels.count(k) for k in sorted(set(labels))},
            "max_err_of_reference_on_native_depths_vs_native": float(on_native_depths[:no][[lb == "placement" for lb in labels]].max()) if "placement" in labels else None,
            "max_implied_cdf_difference_of_placements": float(implied[:no].max()),
            "reference_move_under_perturbations": {"outliers_median": float(np.median(score[:no])), "controls_median": float(np.median(score[no:])),
                                                   "controls_p95": float(np.sort(score[no:])[int(0.95 * (n - no))])}}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(C.SCALE_CASES))
def test_parity_at_scale_vs_reference(name):
    case = dict(C.SCALE_CASES[name], name=name)
    gold = C.load_golden(name)
    if gold is None or C.state_dict_for(case) is None:
        pytest.skip("fixture or checkpoint copy absent")
    l = case["L"] + 1
    rays, jit, u = C.scale_inputs(case)
    report = {"case": name, "rays": int(rays.shape[0])}
    for prec in ("exact", "exact_cf", "mixed"):
        model = build_case_model(case, precision=prec)
        flat = _render(model, rays, jit, u, case)
        for i in range(l):
            assert np.array_equal(flat["ray_mask.%d" % i], gold["ray_mask.%d" % i])
        err = _err(flat, gold, l)
        dd = np.abs(flat["fine_mixed.depth"] - gold["fine_mixed.depth"])[:, 0]
        depth_off = dd > 2e-2 + 2e-3 * np.abs(gold["fine_mixed.depth"][:, 0])       # depth to the tolerance of test_gpu_render.py
        out = np.nonzero((err > GATE) | depth_off)[0]                               # every such ray must be attributed below
        mse = float(((flat["fine_mixed.rgb"].astype(np.float64) - gold["fine_mixed.rgb"]) ** 2).mean())
        rep = {"max_abs_err": float(err.max()), "rays_over_1e-3": int((err > GATE).sum()), "rays_over_gate_or_depth_tolerance": int(out.size),
               "frac_over_1e-3": float((err > GATE).mean()),
               "median_err": float(np.median(err)), "p999_err": float(np.sort(err)[int(0.999 * err.size)]),
               "psnr_db": 99.0 if mse == 0 else float(10 * np.log10(1.0 / mse))}
        thresholds = case["thr"][0] != 0 or case["thr"][1] != 0
        assert out.size <= MAX_OUTLIER_FRACTION[thresholds] * err.size and rep["median_err"] < 5e-5, rep
        if out.size:
            rep["attribution"] = attribute_outliers(case, model, rays, jit, u, out, flat, mixed=(prec == "mixed"))
        report[prec] = rep
        del model
    dst = os.path.join(C.ROOT, "gpurun_out")
    if os.path.isdir(dst):
        with open(os.path.join(dst, "parity_%s.json" % name), "w") as f:
            json.dump(report, f, indent=1)
    print(json.dumps(report))
