"""GPU parity of each hot-path stage (one C-ABI entry point each) against the reference's golden vectors
(tests/golden/functions.npz) -- SURVEY section 4: per-stage unit tests against the imported reference functions."""
import numpy as np
import pytest
import torch

import cases as C
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

FN = C.load_golden("functions")
IN = C.function_inputs()


def dev(t):
    return t.cuda()


def close(a, b, atol, rtol=0.0, what=""):
    a = np.asarray(a.detach().cpu() if torch.is_tensor(a) else a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b) - rtol * np.abs(b)
    assert err.max() <= atol, "%s max err %.3e" % (what, np.abs(a - b).max())


def test_intersection_bit_exact():
    from stnerf_b200 import ops
    r = IN["isect.rays"]
    _, _, _, tt = ops.intersect_sample(dev(r), IN["isect.bmin"], IN["isect.bmax"], 48, dev(IN["sample.jitter"][0]))
    assert np.array_equal(tt.cpu().numpy(), FN["isect.t"])


@pytest.mark.parametrize("layer", [0, 1])
def test_stratified_samples_bit_exact(layer):
    from stnerf_b200 import ops
    r = IN["isect.rays"]
    t, xyz, m, _ = ops.intersect_sample(dev(r), IN["isect.bmin"], IN["isect.bmax"], 48,
                                        dev(IN["sample.jitter"][layer]), is_bkgd=(layer == 0))
    assert np.array_equal(t.cpu().numpy(), FN["sample.t.%d" % layer])
    assert np.array_equal(xyz.cpu().numpy(), FN["sample.xyz.%d" % layer])
    assert np.array_equal(m.cpu().numpy().astype(np.uint8), FN["sample.mask.%d" % layer])


def test_layers_facade_ray_sample_point():
    import layers
    r = dev(IN["isect.rays"])
    bbox = O.corners_from_minmax(IN["isect.bmin"], IN["isect.bmax"])[None, None].expand(r.shape[0], 2, 8, 3)
    ts, pts, masks = layers.RaySamplePoint(48)(r, bbox)
    assert ts[0].shape == (r.shape[0], 48, 1) and pts[1].shape == (r.shape[0], 48, 3)
    assert np.array_equal(masks[1].cpu().numpy().astype(np.uint8), FN["sample.mask.1"])


def test_composite():
    from stnerf_b200 import ops
    c, d, a, w = ops.composite(dev(IN["comp.t"]), dev(IN["comp.rgb"]), dev(IN["comp.sigma"]))
    close(w, FN["comp.w"], 2e-6, what="w")
    close(c, FN["comp.color"], 5e-6, what="color")
    close(d, FN["comp.depth"], 5e-5, what="depth")
    close(a, FN["comp.acc"], 5e-6, what="acc")


def test_volume_renderer_facade():
    import layers
    vr = layers.VolumeRenderer(boarder_weight=1e10)
    c, d, a, w = vr(dev(IN["comp.t"])[..., None], dev(IN["comp.rgb"]), dev(IN["comp.sigma"])[..., None])
    assert w.shape == (64, 96, 1)
    close(c, FN["comp.color"], 5e-6)


def test_sample_pdf():
    from stnerf_b200 import ops
    z, tf = ops.sample_pdf(dev(IN["pdf.t"]), dev(IN["pdf.w"]), dev(IN["pdf.u"]), merge=True)
    got, want = z.cpu().numpy(), FN["pdf.z"]
    # the `denom < 1e-5 -> 1` branch of utils/sample_pdf.py:59 is discontinuous in cdf round-off: allow a handful
    # of samples to land elsewhere inside their (empty) bin, everything else must agree to fp32 round-off
    bad = np.abs(got - want) > 2e-5
    assert bad.mean() < 0.002, "fraction of mismatching samples %.4f" % bad.mean()
    # sorted merge == torch.sort(cat(t, z))
    ref = np.sort(np.concatenate([IN["pdf.t"].numpy(), got], 1), 1)
    assert np.array_equal(tf.cpu().numpy(), ref)


def test_utils_facade_sample_pdf_shapes():
    import utils
    z = utils.sample_pdf(dev(IN["pdf.t"]), dev(IN["pdf.w"][:, 1:-1]), N_samples=32)
    assert z.shape == (64, 32) and torch.isfinite(z).all()
    lo, hi = IN["pdf.t"].min().item(), IN["pdf.t"].max().item()
    assert z.min().item() >= lo - 1e-4 and z.max().item() <= hi + 1e-4


def test_positional_encoding():
    from stnerf_b200 import ops
    import utils
    close(ops.positional_encoding(dev(IN["pe.x3"]), 10), FN["pe.x3_L10"], 5e-7)
    close(ops.positional_encoding(dev(IN["pe.x3"]), 4), FN["pe.x3_L4"], 5e-7)
    close(ops.positional_encoding(dev(IN["pe.x1"]), 10), FN["pe.x1_L10"], 5e-7)
    close(utils.Trigonometric_kernel(L=10)(dev(IN["pe.x3"])), FN["pe.x3_L10"], 5e-7)


def test_generate_rays():
    from stnerf_b200 import ops
    rays = ops.generate_rays(IN["rays.K"], IN["rays.T"], 24, 40)
    close(rays, FN["rays.rays"], 2e-6)
    # strided rows + frame-id columns (multi-GPU sharding form)
    sub = ops.generate_rays(IN["rays.K"], IN["rays.T"], 24, 40, frame_ids=[0, 7, 8.5], row0=1, row_step=3)
    want = FN["rays.rays"].reshape(24, 40, 6)[1::3].reshape(-1, 6)
    close(sub[:, :6], want, 2e-6)
    assert torch.equal(sub[:, 6:].cpu(), torch.tensor([0, 7, 8.5]).expand(sub.shape[0], 3))


def _renderer(tag, precision):
    from stnerf_b200 import NativeRenderer
    if tag == "syn":
        sd = O.synthetic_state_dict(1, True, seed=5)
    else:
        p = C.find_checkpoint({"tkd": "taekwondo", "walk": "walking"}[tag])
        if p is None:
            pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
        sd = C.replicate_layers(torch.load(p, map_location="cpu")["model"], 1)
    st = sd["spacenets.0.rgb_net.1.weight"].shape[1] == 304
    r = NativeRenderer(2, [False, st], precision)
    r.load_state_dict(sd)
    return r


@pytest.mark.parametrize("precision,sig_tol,rgb_tol", [("fp32", 2e-3, 2e-4), ("exact", 2e-2, 2e-3), ("exact_cf", 2e-2, 2e-3)])
@pytest.mark.parametrize("tag", ["syn", "tkd", "walk"])
def test_networks(tag, precision, sig_tol, rgb_tol):
    """SpaceNet / MotionNet on explicit points vs the reference modules (raw logits: sigma reaches ~1e3, so the
    tolerance is relative-dominated)."""
    if "net.%s.perf.rgb" % tag not in FN:
        pytest.skip("golden for %s not generated" % tag)
    r = _renderer(tag, precision)
    pos, dirs, tm = dev(IN["net.pos"]), dev(IN["net.dirs"]), dev(IN["net.time_int"])
    rgb, sig = r.spacenet(1, False, pos, dirs, tm.reshape(-1))
    close(rgb, FN["net.%s.perf.rgb" % tag], rgb_tol, 2e-4, "perf rgb")
    close(sig, FN["net.%s.perf.sigma" % tag], sig_tol, 2e-4, "perf sigma")
    rgb, sig = r.spacenet(0, True, pos, dirs, None)
    close(rgb, FN["net.%s.bkgd.rgb" % tag], rgb_tol, 2e-4, "bkgd rgb")
    close(sig, FN["net.%s.bkgd.sigma" % tag], sig_tol, 2e-4, "bkgd sigma")
    for kind, tcol in (("int", IN["net.time_int"]), ("frac", IN["net.time_frac"])):
        flow = r.motionnet(1, dev(torch.cat([IN["net.pos"], tcol], 1)))
        close(flow, FN["net.%s.motion_%s" % (tag, kind)], 2e-4, 2e-4, "motion " + kind)
    r.close()


def test_umma_selftest():
    """One 128x256x64 fp16 product through the library's warpgroup-MMA descriptors / swizzled layouts / bulk copy /
    accumulator fragment."""
    import ctypes
    from stnerf_b200 import _lib as L
    err = ctypes.c_float(-1.0)
    L.check(L.lib().stnerf_selftest_umma(ctypes.byref(err)), "stnerf_selftest_umma")
    assert 0.0 <= err.value < 1e-3, err.value
