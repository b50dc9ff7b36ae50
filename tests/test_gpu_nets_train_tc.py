"""SpaceNet / MotionNet in the tf32x3 training precision (csrc/mlp_train_tc.cu) on the device.

The method of test_gpu_nets_train.py and its helpers: float64 truth, the CPU fp32 autograd yardstick, kink-free points.  Every
tensor's rms and max error must stay within 4x the yardstick's (6x through MotionNet -> SpaceNet), plus ULP_FLOOR: the 3xTF32
products carry ~22 significant bits, against fp32's 24.  Scaling the upstream gradients by 1e-20 and 1e+20 must leave the
relative errors where they were (tf32 keeps fp32's exponent).  Batch sizes at tile (128), CTA-tile and weight-gradient chunk
boundaries are compared with the fp32 path, whose indexing they share.
"""
import pytest
import torch

import test_gpu_networks_f64 as NF
import test_gpu_nets_train as NT
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
FACTOR = 4.0
CHAINED_FACTOR = 6.0
RANGE_FACTOR = 1.5
MIN_CHUNK, MAX_SPLIT = 256, 128          # mlp_train.cu: points per weight-gradient chunk, chunks per sum


def _nets():
    from stnerf_b200 import nets
    return nets


def space_module(w, prec="tf32x3"):
    net = _nets().SpaceNet(use_time=NF.uses_time(w), train_precision=prec)
    net.load_state_dict(w)
    return net.to(DEV)


def motion_module(w, prec="tf32x3"):
    net = _nets().MotionNet(c_input=4, input_time=True, train_precision=prec)
    net.load_state_dict(w)
    return net.to(DEV)


def space_grads(w, pos, dirs, tm, prec="tf32x3", scale=1.0):
    net = space_module(w, prec)
    p = pos.to(DEV).requires_grad_(True)
    rgb, sig = net(p, torch.cat([pos, dirs], 1).to(DEV), tm.to(DEV))
    loss = (rgb * (NT._proj(rgb.shape, 1) * scale).to(DEV)).sum() + (sig * (NT._proj(sig.shape, 2) * scale).to(DEV)).sum()
    loss.backward()
    out = {k: v.grad.detach().to(torch.float64) / scale for k, v in net.named_parameters()}
    out["pos"] = p.grad.detach().to(torch.float64) / scale
    return out, rgb.detach(), sig.detach()


def motion_grads(w, xyzt, lerp_mode=-1, prec="tf32x3", scale=1.0):
    net = motion_module(w, prec)
    flow = net(xyzt.to(DEV), lerp_mode)
    (flow * (NT._proj(flow.shape, 3) * scale).to(DEV)).sum().backward()
    return {k: v.grad.detach().to(torch.float64) / scale for k, v in net.named_parameters()}, flow.detach()


@pytest.mark.parametrize("tag", NF.WEIGHTS)
def test_spacenet_gradients_against_float64(tag):
    nets = NT._weights(tag)
    for name in ("bkgd", "perf"):
        w = NF.space_weights(nets, name)
        for s in NT.SETS:
            pos, dirs, tm = NT.points()[s]
            keep = NT.kink_free(lambda: O.spacenet_forward(NT._f64(w), pos.to(DEV, torch.float64), dirs.to(DEV, torch.float64),
                                                           tm.to(DEV, torch.float64) if NF.uses_time(w) else None))
            pos, dirs, tm = pos[keep], dirs[keep], tm[keep]
            truth = NT.oracle_space_grads(w, pos, dirs, tm, DEV, torch.float64)
            ww = NT._f64(w)
            with torch.no_grad():
                rgb64, sig64 = O.spacenet_forward(ww, pos.to(DEV, torch.float64), dirs.to(DEV, torch.float64),
                                                  tm.to(DEV, torch.float64) if NF.uses_time(w) else None)
            got, rgb, sig = space_grads(w, pos, dirs, tm)
            got["rgb"], got["sigma"] = rgb, sig
            truth = dict(truth, rgb=rgb64, sigma=sig64)
            nat = NT.grad_errors(got, truth)
            with torch.no_grad():
                rgb32, sig32 = O.spacenet_forward({k: v.float() for k, v in w.items()}, pos.float(), dirs.float(),
                                                  tm.float() if NF.uses_time(w) else None)
            cpu = NT.grad_errors(dict(NT.oracle_space_grads(w, pos, dirs, tm, "cpu", torch.float32), rgb=rgb32, sigma=sig32),
                                 truth)
            NT.assert_within_twice(nat, cpu, "tf32x3 %s/%s/%s" % (tag, name, s), FACTOR)


@pytest.mark.parametrize("tag", NF.WEIGHTS)
def test_motionnet_gradients_against_float64(tag):
    w = NT._weights(tag)["motion"][0]
    for s in NT.SETS:
        pos, _, tm = NT.points()[s]
        xyzt = torch.cat([pos, tm], 1)
        for lerp_mode in (-1, 0, 1):
            lerp = NF.lerp_of(tm, lerp_mode)
            keep = NT.kink_free(lambda: NF.motion_forward(NT._f64(w), xyzt.to(DEV, torch.float64), lerp))
            x = xyzt[keep]
            truth = NT.oracle_motion_grads(w, x, lerp, DEV, torch.float64)
            with torch.no_grad():
                truth["flow"] = NF.motion_forward(NT._f64(w), x.to(DEV, torch.float64), lerp)
                flow32 = NF.motion_forward({k: v.float() for k, v in w.items()}, x.float(), lerp)
            got, flow = motion_grads(w, x, lerp_mode)
            got["flow"] = flow
            nat = NT.grad_errors(got, truth)
            cpu = NT.grad_errors(dict(NT.oracle_motion_grads(w, x, lerp, "cpu", torch.float32), flow=flow32), truth)
            NT.assert_within_twice(nat, cpu, "tf32x3 %s/%s/lerp%d" % (tag, s, lerp_mode), FACTOR)


@pytest.mark.parametrize("tag", ["syn_t", "tkd"])
def test_chained_motionnet_gradients_against_float64(tag):
    """MotionNet -> SpaceNet(xyz + flow), as test_gpu_nets_train's chained test, both networks in tf32x3."""
    nets = NT._weights(tag)
    for s in ("rays", "times"):
        pos, dirs, tm = NT.points()[s]
        xyzt = torch.cat([pos, tm], 1)
        mw, sw = nets["motion"][0], nets["space"][0]

        def f64():
            x = xyzt.to(DEV, torch.float64)
            O.spacenet_forward(NT._f64(sw), x[:, :3] + O.motionnet_forward(NT._f64(mw), x), dirs.to(DEV, torch.float64),
                               x[:, 3:] if NF.uses_time(sw) else None)
        keep = NT.kink_free(f64, NT.KINK_CHAINED)
        x, d = xyzt[keep], dirs[keep]
        mn, sn = motion_module(mw), space_module(sw)
        xd = x.to(DEV)
        flow = mn(xd)
        rgb, sig = sn(xd[:, :3] + flow, torch.cat([x[:, :3], d], 1).to(DEV), xd[:, 3:])
        ((rgb * NT._proj(rgb.shape, 1).to(DEV)).sum() + (sig * NT._proj(sig.shape, 2).to(DEV)).sum()).backward()
        nat = {k: v.grad.detach() for k, v in mn.named_parameters()}
        cpu, flow_cpu = NT._chained(mw, sw, x, d, "cpu", torch.float32, False)
        nat = NT.grad_errors(nat, NT._chained(mw, sw, x, d, DEV, torch.float64, False, flow_at=flow.detach())[0])
        cpu = NT.grad_errors(cpu, NT._chained(mw, sw, x, d, DEV, torch.float64, False, flow_at=flow_cpu)[0])
        NT.assert_within_twice(nat, cpu, "tf32x3 chained %s/%s" % (tag, s), CHAINED_FACTOR)


def test_upstream_gradients_scaled_by_1e20_and_1e_minus_20():
    """The lo halves of terms near 1e-20 x 2^-11 and products up to 1e20 x |W| stay normal fp32 / tf32: the relative errors
    of the scaled runs match the unscaled run's."""
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sw, mw = w["space"][0], w["motion"][0]
    pos, dirs, tm = NT.points()["gauss"]
    keep = NT.kink_free(lambda: O.spacenet_forward(NT._f64(sw), pos.to(DEV, torch.float64), dirs.to(DEV, torch.float64),
                                                   tm.to(DEV, torch.float64)))
    pos, dirs, tm = pos[keep], dirs[keep], tm[keep]
    truth = NT.oracle_space_grads(sw, pos, dirs, tm, DEV, torch.float64)
    xyzt = torch.cat([pos, tm + 0.25], 1)
    lerp = NF.lerp_of(tm + 0.25, -1)
    mtruth = NT.oracle_motion_grads(mw, xyzt, lerp, DEV, torch.float64)
    base = NT.grad_errors(space_grads(sw, pos, dirs, tm)[0], truth)
    mbase = NT.grad_errors(motion_grads(mw, xyzt)[0], mtruth)
    for scale in (1e-20, 1e20):
        got = NT.grad_errors(space_grads(sw, pos, dirs, tm, scale=scale)[0], truth)
        mgot = NT.grad_errors(motion_grads(mw, xyzt, scale=scale)[0], mtruth)
        for e, b, what in ((got, base, "spacenet"), (mgot, mbase, "motionnet")):
            ratio = max(max(e[k][i] / max(b[k][i], NT.ULP_FLOOR) for i in (0, 1)) for k in e)
            print("scale %g %s: worst error ratio to unscaled %.3f" % (scale, what, ratio))
            for k in e:
                for i in (0, 1):
                    assert e[k][i] <= RANGE_FACTOR * b[k][i] + NT.ULP_FLOOR, (scale, what, k, e[k][i], b[k][i])


def _rel(a, b):
    a, b = a.to(torch.float64), b.to(torch.float64)
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


def _kink_free_points(sw, mw, P, seed):
    """P random points none of whose float64 pre-activations, in the SpaceNet or the MotionNet, sits at a ReLU kink (see
    test_gpu_nets_train.kink_free): there the fp32 and the tf32x3 forward may take different sides, which moves a gradient
    by a whole point's share."""
    g = torch.Generator().manual_seed(seed)
    n = P + P // 4 + 64
    pos = torch.randn((n, 3), generator=g) * 0.7
    dirs = torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=1)
    tm = torch.full((n, 1), 3.0) + torch.rand((n, 1), generator=g)
    xyzt = torch.cat([pos, tm], 1)
    lerp = NF.lerp_of(tm, -1)
    keep = NT.kink_free(lambda: O.spacenet_forward(NT._f64(sw), pos.to(DEV, torch.float64), dirs.to(DEV, torch.float64),
                                                   tm.to(DEV, torch.float64)))
    keep &= NT.kink_free(lambda: NF.motion_forward(NT._f64(mw), xyzt.to(DEV, torch.float64), lerp))
    idx = keep.nonzero()[:, 0][:P]
    assert idx.numel() == P
    return pos[idx], dirs[idx], tm[idx]


@pytest.mark.parametrize("P", [1, 7, 63, 64, 65, 127, 128, 129, MIN_CHUNK * MAX_SPLIT - 1, MIN_CHUNK * MAX_SPLIT + 1,
                               (1 << 20) + 3])
def test_batch_sizes_at_tile_and_chunk_boundaries(P):
    """Outputs, d_pos and parameter gradients against the fp32 path on the same kink-free points: an indexing error would show
    as an O(1) difference, the arithmetic differs at ~1e-6."""
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sw, mw = w["space"][0], w["motion"][0]
    pos, dirs, tm = _kink_free_points(sw, mw, P, P)
    a, rgb_a, sig_a = space_grads(sw, pos, dirs, tm)
    b, rgb_b, sig_b = space_grads(sw, pos, dirs, tm, prec="fp32")
    worst = max([_rel(rgb_a, rgb_b), _rel(sig_a, sig_b)] + [_rel(a[k], b[k]) for k in a])
    xyzt = torch.cat([pos, tm], 1)
    ma, fa = motion_grads(mw, xyzt)
    mb, fb = motion_grads(mw, xyzt, prec="fp32")
    mworst = max([_rel(fa, fb)] + [_rel(ma[k], mb[k]) for k in ma])
    print("P = %d: worst relative difference to fp32, spacenet %.3g, motionnet %.3g" % (P, worst, mworst))
    assert worst < 2e-3 and mworst < 2e-3, (worst, mworst)


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def test_identical_calls_and_rows_independent_of_batch():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    pos, dirs, tm = NT.points()["gauss"]
    a, b = space_grads(w["space"][0], pos, dirs, tm)[0], space_grads(w["space"][0], pos, dirs, tm)[0]
    assert all(_same(a[k], b[k]) for k in a)
    xyzt = torch.cat([pos, tm + 0.25], 1)
    a, b = motion_grads(w["motion"][0], xyzt)[0], motion_grads(w["motion"][0], xyzt)[0]
    assert all(_same(a[k], b[k]) for k in a)
    sn, mn = space_module(w["space"][0]), motion_module(w["motion"][0])
    g = torch.Generator().manual_seed(5)
    n = 5 * 128 * 132 + 77
    pos = (torch.randn((n, 3), generator=g) * 1.5).to(DEV)
    rays = torch.cat([pos, torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=1).to(DEV)], 1)
    tm = torch.full((n, 1), 12.0, device=DEV)
    xyzt = torch.cat([pos, tm], 1)
    with torch.no_grad():
        rgb, sig = sn(pos, rays, tm)
        flow = mn(xyzt, 0)
        for sl in [slice(0, k) for k in (1, 127, 128, 129, 1000)] + [slice(k, n) for k in (1, 8, 16, 64, 128)]:
            r2, s2 = sn(pos[sl], rays[sl], tm[sl])
            assert _same(r2, rgb[sl]) and _same(s2, sig[sl]), sl
            assert _same(mn(xyzt[sl], 0), flow[sl]), sl
        perm = torch.randperm(n, generator=g).to(DEV)
        r2, s2 = sn(pos[perm], rays[perm], tm[perm])
        assert _same(r2, rgb[perm]) and _same(s2, sig[perm])
        assert _same(mn(xyzt[perm], 0), flow[perm])


def test_zero_points_bad_precision_and_short_scratch():
    from stnerf_b200 import _lib as L
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sn, mn = space_module(w["space"][0]), motion_module(w["motion"][0])
    pos = torch.zeros((0, 3), device=DEV, requires_grad=True)
    rgb, sig = sn(pos, torch.zeros((0, 6), device=DEV), torch.zeros((0, 1), device=DEV))
    (rgb.sum() + sig.sum()).backward()
    assert rgb.shape == (0, 3) and pos.grad.shape == (0, 3)
    assert all(float(p.grad.abs().max()) == 0.0 for p in sn.parameters())
    flow = mn(torch.zeros((0, 4), device=DEV))
    flow.sum().backward()
    assert all(float(p.grad.abs().max()) == 0.0 for p in mn.parameters())

    lib, P, tp = L.lib(), 300, L.TRAIN_TC_3XTF32
    assert lib.stnerf_train_scratch_bytes_prec(0, 1, P, 7) == 0
    assert lib.stnerf_train_scratch_bytes_prec(0, 1, P, tp) == lib.stnerf_train_scratch_bytes(0, 1, P)
    W = torch.cat([p.detach().reshape(-1) for p in sn.parameters()])
    MW = torch.cat([p.detach().reshape(-1) for p in mn.parameters()])
    x = torch.rand((P, 4), device=DEV)
    pos, dirs, times = x[:, :3].contiguous(), x[:, 1:].contiguous(), x[:, 3].contiguous()
    saved = torch.empty(lib.stnerf_train_saved_floats(0, 1, P), device=DEV)
    msaved = torch.empty(lib.stnerf_train_saved_floats(1, 0, P), device=DEV)
    rgb, sig, d3 = (torch.zeros((P, 3), device=DEV), torch.zeros(P, device=DEV), torch.zeros((P, 3), device=DEV))
    dW, dMW = torch.empty_like(W), torch.empty_like(MW)
    nb = lib.stnerf_train_scratch_bytes_prec(0, 1, P, tp)
    mnb = lib.stnerf_train_scratch_bytes_prec(1, 0, P, tp)
    scratch = torch.empty(max(nb, mnb), dtype=torch.uint8, device=DEV)
    s = L.stream_ptr()
    ptr = L.ptr
    for prec, ok in ((7, False), (-1, False), (tp, True)):
        rc = lib.stnerf_spacenet_train_forward_prec(ptr(W), 1, ptr(pos), ptr(dirs), ptr(times), P, ptr(rgb), ptr(sig),
                                                    ptr(saved), prec, s)
        assert (rc == 0) == ok, (prec, rc)
        rc = lib.stnerf_spacenet_backward_prec(ptr(W), 1, P, ptr(saved), ptr(d3), ptr(sig), ptr(dW), ptr(d3), ptr(scratch), nb,
                                               prec, s)
        assert (rc == 0) == ok, (prec, rc)
        rc = lib.stnerf_motionnet_train_forward_prec(ptr(MW), ptr(x), P, -1, ptr(d3), ptr(msaved), ptr(scratch), mnb, prec, s)
        assert (rc == 0) == ok, (prec, rc)
        rc = lib.stnerf_motionnet_backward_prec(ptr(MW), P, ptr(msaved), ptr(d3), ptr(dMW), ptr(scratch), mnb, prec, s)
        assert (rc == 0) == ok, (prec, rc)
    einval = -1                                          # STNERF_EINVAL
    assert lib.stnerf_spacenet_backward_prec(ptr(W), 1, P, ptr(saved), ptr(d3), ptr(sig), ptr(dW), ptr(d3), ptr(scratch), nb - 1,
                                             tp, s) == einval
    assert lib.stnerf_motionnet_train_forward_prec(ptr(MW), ptr(x), P, -1, ptr(d3), ptr(msaved), ptr(scratch), mnb - 1, tp,
                                                   s) == einval
    assert lib.stnerf_motionnet_backward_prec(ptr(MW), P, ptr(msaved), ptr(d3), ptr(dMW), ptr(scratch), mnb - 1, tp, s) == einval
    torch.cuda.synchronize()
