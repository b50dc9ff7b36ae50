"""The float64 restatement the compositing-pass GPU tests compare against (tests/composite_pass_restatement.py) IS the
reference's function: evaluated in fp32 on the CPU it reproduces the reference's own outputs for the committed per-stage
vectors (tests/golden/functions.npz, written by the unmodified reference) bit for bit, and in float64 it lies within fp32
round-off of them.  Runs without a GPU."""
import numpy as np
import torch

import cases as C
import composite_pass_restatement as R

FN = C.load_golden("functions")
IN = C.function_inputs()


def test_composite_is_the_references():
    pix, w = R.composite(IN["comp.t"], IN["comp.rgb"], IN["comp.sigma"], 1e10)
    assert np.array_equal(w.numpy(), FN["comp.w"])
    assert np.array_equal(pix[:, :3].numpy(), FN["comp.color"])
    assert np.array_equal(pix[:, 3:4].numpy(), FN["comp.depth"])
    assert np.array_equal(pix[:, 4:].numpy(), FN["comp.acc"])
    pix, w = R.composite(IN["comp.t"].double(), IN["comp.rgb"].double(), IN["comp.sigma"].double(), 1e10)
    assert np.abs(w.numpy() - FN["comp.w"]).max() < 2e-7
    assert np.abs(pix[:, :3].numpy() - FN["comp.color"]).max() < 5e-7
    assert np.abs(pix[:, 3:4].numpy() - FN["comp.depth"]).max() < 2e-6          # sum of w t with t up to 6
    assert np.abs(pix[:, 4:].numpy() - FN["comp.acc"]).max() < 5e-7


def test_sample_pdf_is_the_references():
    z, _ = R.sample_pdf(IN["pdf.t"], IN["pdf.w"], IN["pdf.u"])
    assert np.array_equal(z.numpy(), FN["pdf.z"])
    z, d = R.sample_pdf(IN["pdf.t"].double(), IN["pdf.w"].double(), IN["pdf.u"].double())
    # float64 against the reference's fp32: the error of a sample is the cdf's round-off over the slope of its bin
    width = (d["ba"] - d["bb"]).abs().numpy()
    tol = width * 2e-6 / d["den"].numpy() + 2e-6
    near_branch = np.abs(d["den_raw"].numpy() - 1e-5) < 4e-6                     # sample_pdf.py:59 may go either way there
    bad = (np.abs(z.numpy() - FN["pdf.z"]) > tol) & ~near_branch
    assert not bad.any(), int(bad.sum())
    assert near_branch.mean() < 0.01


def test_merge_is_a_stable_sort_of_the_concatenation():
    """torch.sort of the reference's merge (layered_rfrender.py:425, 587) leaves equal depths in concatenation order, and counts
    -0.0 and +0.0 as equal: what run_pass restates with a stable argsort."""
    t = torch.tensor([[1.0, 2.0, 2.0, 3.0, 2.0, 0.0, -0.0, 2.0]])
    want = torch.sort(t, dim=-1, stable=True)[1]
    assert want.tolist() == [[5, 6, 0, 1, 2, 4, 7, 3]]
    scene = dict(near=0.0, alpha2=1.0, thr_layer=0.0, thr_bkgd=0.0, boarder=1e10, apply_thr=False, shown=[True, True])
    ts = [t[:, :4].double(), t[:, 4:].double()]
    lg = [torch.full((1, 4, 3), -2.0, dtype=torch.float64), torch.full((1, 4, 3), 2.0, dtype=torch.float64)]
    sg = [torch.full((1, 4), 0.7, dtype=torch.float64), torch.full((1, 4), 0.3, dtype=torch.float64)]
    a = R.merged_pixel(scene, False, ts, lg, sg)
    b = R.merged_pixel(scene, False, ts, lg, sg, reverse_ties=True)
    idx = want[0]
    direct = R.composite(torch.cat(ts, -1)[:, idx], torch.cat(lg, 1)[:, idx], torch.cat(sg, -1)[:, idx], 1e10)[0]
    assert torch.equal(a, direct)
    assert (a - b).abs().max() > 1e-2                                            # the tie order is visible in the pixel


def test_run_pass_matches_its_parts():
    g = torch.Generator().manual_seed(3)
    l, n, S, n2 = 3, 5, 12, 7
    t = torch.sort(torch.rand((l, n, S), generator=g, dtype=torch.float64) * 4 - 0.5, -1)[0]
    raw = torch.randn((l, n, S, 4), generator=g, dtype=torch.float64) * 3
    mask = torch.tensor([[1] * n, [1, 0, 1, 0, 1], [0, 0, 1, 1, 1]]).bool()
    u = torch.rand((l, n, n2), generator=g, dtype=torch.float64)
    scene = dict(near=0.4, alpha2=0.5, thr_layer=0.5, thr_bkgd=1.0, boarder=1e10, apply_thr=True, shown=[True, True, False])
    for fine in (False, True):
        out = R.run_pass(scene, fine, t, raw, mask, None if fine else u)
        img = out["images"]
        assert img[2][~mask[1]].abs().max() == 0 and img[3][~mask[2]].abs().max() == 0
        assert img[3][:, :4].abs().max() == 0                                    # a hidden layer composites zero density
        # ray 1 hits nothing but the background: its merged pixel is the background's own (coarse; fine cuts t < near first)
        if not fine:
            assert torch.allclose(img[0][1], img[1][1], rtol=0, atol=1e-15)
        sg0 = R.mask_density(scene, 0, fine, t[0], raw[0, ..., 3])
        if fine:
            assert torch.equal(sg0, torch.where(raw[0, ..., 3] < 1.0, torch.zeros(()).double(), raw[0, ..., 3]))
        else:
            assert torch.equal(sg0, torch.where(t[0] < 0.4, torch.zeros(()).double(), raw[0, ..., 3]))
    out = R.run_pass(scene, False, t, raw, mask, u)
    assert out["t_fine"].shape == (l, n, S + n2) and (out["t_fine"][..., 1:] >= out["t_fine"][..., :-1]).all()
    lo, hi = out["pdf"][0]["bins"][..., :1], out["pdf"][0]["bins"][..., -1:]
    assert ((out["z"][0] >= lo) & (out["z"][0] <= hi)).all()
