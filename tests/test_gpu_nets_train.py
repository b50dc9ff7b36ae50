"""Trainable SpaceNet / MotionNet (stnerf_b200.nets over csrc/mlp_train.cu) on the device.

Forward: the training forward's outputs are bit-identical to `stnerf_spacenet` / `stnerf_motionnet` in `fp32` mode, and a
point's outputs do not depend on the batch around it.
Gradients: d_pos and every parameter gradient against float64 autograd of the oracle's restatement with the same fp32 weights
and points (pinned to the reference's own gradients by tests/test_nets_train.py).  Weights: synthetic with and without a time
input, and both shipped checkpoints when their copies are present; points: the rays / gauss / far / times sets of
test_gpu_networks_f64.py (first YARD_POINTS of each); loss: a seeded random projection of the outputs.  The budget is
self-calibrating: twice the error of the CPU oracle's own fp32 autograd on the same points, on the rms AND the max of each
tensor's error (relative to that tensor's rms / max magnitude).
"""
import numpy as np
import pytest
import torch

import cases as C
import test_gpu_networks_f64 as NF
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

YARD_POINTS = 4096
KINK = 1e-4
ULP_FLOOR = 8 * 2.0 ** -24
# chained: the SpaceNet's input xyz + flow carries the MotionNet forward's rounding, which PE(pos)'s 2^9 frequency magnifies, so
# its pre-activations sit further from the float64 ones and the band of ambiguous ReLU masks is wider
KINK_CHAINED = 1e-3
# the chained MotionNet gradients sum d_pos terms that cancel strongly (relative error ~1e-5 for both fp32 paths); the native
# path's worst ratio to the CPU yardstick measured 2.3 (taekwondo weights, `times` points, one H100 80GB HBM3 at 700 W)
CHAINED_FACTOR = 3.0
SETS = ("rays", "gauss", "far", "times")
DEV = "cuda"
_POINTS = {}


def points():
    if not _POINTS:
        for k, (pos, dirs, tm) in NF.point_sets().items():
            _POINTS[k] = (pos[:YARD_POINTS].contiguous(), dirs[:YARD_POINTS].contiguous(), tm[:YARD_POINTS].contiguous())
    return _POINTS


def _nets():
    from stnerf_b200 import nets
    return nets


def space_module(w):
    net = _nets().SpaceNet(use_time=NF.uses_time(w))
    net.load_state_dict(w)
    return net.to(DEV)


def motion_module(w):
    net = _nets().MotionNet(c_input=4, input_time=True)
    net.load_state_dict(w)
    return net.to(DEV)


def _proj(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g)


# ---------------------------------------------------------------------------------------------------------------------
# gradients: native, float64 truth, CPU fp32 yardstick
# ---------------------------------------------------------------------------------------------------------------------
def native_space_grads(w, pos, dirs, tm):
    net = space_module(w)
    p = pos.to(DEV).requires_grad_(True)
    rgb, sig = net(p, torch.cat([pos, dirs], 1).to(DEV), tm.to(DEV))
    loss = (rgb * _proj(rgb.shape, 1).to(DEV)).sum() + (sig * _proj(sig.shape, 2).to(DEV)).sum()
    loss.backward()
    out = {k: v.grad.detach().clone() for k, v in net.named_parameters()}
    out["pos"] = p.grad.detach().clone()
    return out


def oracle_space_grads(w, pos, dirs, tm, device, dtype):
    ww = {k: v.detach().to(device, dtype).clone().requires_grad_(True) for k, v in w.items()}
    p = pos.detach().to(device, dtype).clone().requires_grad_(True)
    rgb, sig = O.spacenet_forward(ww, p, dirs.to(device, dtype), tm.to(device, dtype) if NF.uses_time(w) else None)
    loss = (rgb * _proj(rgb.shape, 1).to(device, dtype)).sum() + (sig * _proj(sig.shape, 2).to(device, dtype)).sum()
    loss.backward()
    out = {k: v.grad.detach() for k, v in ww.items()}
    out["pos"] = p.grad.detach()
    return out


def native_motion_grads(w, xyzt, lerp_mode=-1):
    net = motion_module(w)
    flow = net(xyzt.to(DEV), lerp_mode)
    (flow * _proj(flow.shape, 3).to(DEV)).sum().backward()
    return {k: v.grad.detach().clone() for k, v in net.named_parameters()}


def oracle_motion_grads(w, xyzt, lerp, device, dtype):
    ww = {k: v.detach().to(device, dtype).clone().requires_grad_(True) for k, v in w.items()}
    flow = NF.motion_forward(ww, xyzt.to(device, dtype), lerp)
    (flow * _proj(flow.shape, 3).to(device, dtype)).sum().backward()
    return {k: v.grad.detach() for k, v in ww.items()}


def grad_errors(got, truth):
    """per tensor: (rms error / rms truth, max error / max |truth|)"""
    out = {}
    for k, t in truth.items():
        e = got[k].to(t.device, torch.float64) - t
        out[k] = (float(e.pow(2).mean().sqrt() / t.pow(2).mean().sqrt().clamp(min=1e-300)),
                  float(e.abs().max() / t.abs().max().clamp(min=1e-300)))
    return out


def assert_within_twice(nat, cpu, what, factor=2.0):
    """rms and max of every tensor within twice the CPU fp32 yardstick's, plus ULP_FLOOR: a few roundings of the result
    itself, the level at which two correct fp32 summation orders of the same sum differ at random (a bias gradient is one
    sum of P terms)."""
    bad = {k: (nat[k], cpu[k]) for k in nat
           if nat[k][0] > factor * cpu[k][0] + ULP_FLOOR or nat[k][1] > factor * cpu[k][1] + ULP_FLOOR}
    worst = max(nat[k][1] / max(cpu[k][1], 1e-12) for k in nat)
    worst_rms = max(nat[k][0] / max(cpu[k][0], 1e-12) for k in nat)
    print("%s: worst ratio native / cpu fp32: rms %.2f, max %.2f" % (what, worst_rms, worst))
    assert not bad, (what, bad)


def kink_free(fwd, kink=None):
    """Points none of whose float64 hidden pre-activations (every Linear wider than 3 outputs) lies within KINK x that layer's
    rms of the ReLU's kink.  There the derivative jumps, and an fp32 forward may land on either side of it: the native path and
    the CPU yardstick each flip a few such (point, unit) masks, at different points, and one flip moves a weight gradient by a
    whole point's contribution (~1/P of it).  Those points are set aside for both, so the budget compares arithmetic."""
    zs, real = [], O.F.linear

    def rec(x, w, b=None):
        z = real(x, w, b)
        if w.shape[0] > 3:
            zs.append(z)
        return z
    O.F.linear = rec
    try:
        with torch.no_grad():
            fwd()
    finally:
        O.F.linear = real
    ok = torch.ones(zs[0].shape[0], dtype=torch.bool, device=zs[0].device)
    for z in zs:
        ok &= (z.abs() >= (kink or KINK) * z.pow(2).mean().sqrt()).all(1)
    return ok.cpu()


def _f64(w):
    return {k: v.to(DEV, torch.float64) for k, v in w.items()}


def _weights(tag):
    sd = NF.state_dict(tag)
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    return O.split_state_dict(sd, 1)


@pytest.mark.parametrize("tag", NF.WEIGHTS)
def test_spacenet_gradients_against_float64(tag):
    nets = _weights(tag)
    for name in ("bkgd", "perf"):
        w = NF.space_weights(nets, name)
        for s in SETS:
            pos, dirs, tm = points()[s]
            keep = kink_free(lambda: O.spacenet_forward(_f64(w), pos.to(DEV, torch.float64), dirs.to(DEV, torch.float64),
                                                        tm.to(DEV, torch.float64) if NF.uses_time(w) else None))
            pos, dirs, tm = pos[keep], dirs[keep], tm[keep]
            truth = oracle_space_grads(w, pos, dirs, tm, DEV, torch.float64)
            nat = grad_errors(native_space_grads(w, pos, dirs, tm), truth)
            cpu = grad_errors(oracle_space_grads(w, pos, dirs, tm, "cpu", torch.float32), truth)
            assert_within_twice(nat, cpu, "%s/%s/%s" % (tag, name, s))


@pytest.mark.parametrize("tag", NF.WEIGHTS)
def test_motionnet_gradients_against_float64(tag):
    w = _weights(tag)["motion"][0]
    for s in SETS:
        pos, _, tm = points()[s]
        xyzt = torch.cat([pos, tm], 1)
        for lerp_mode in (-1, 0, 1):
            lerp = NF.lerp_of(tm, lerp_mode)
            keep = kink_free(lambda: NF.motion_forward(_f64(w), xyzt.to(DEV, torch.float64), lerp))
            x = xyzt[keep]
            truth = oracle_motion_grads(w, x, lerp, DEV, torch.float64)
            nat = grad_errors(native_motion_grads(w, x, lerp_mode), truth)
            cpu = grad_errors(oracle_motion_grads(w, x, lerp, "cpu", torch.float32), truth)
            assert_within_twice(nat, cpu, "%s/%s/lerp%d" % (tag, s, lerp_mode))


def _chained(mw, sw, xyzt, dirs, device, dtype, native, flow_at=None):
    """MotionNet's parameter gradients (and its flow) for a loss on SpaceNet(xyz + flow).  flow_at: evaluate the SpaceNet at
    xyz + flow_at instead, with the gradient still taken through this chain's own flow (the float64 truth of an fp32 path)."""
    if native:
        mn, sn = motion_module(mw), space_module(sw)
        x = xyzt.to(DEV)
        flow = mn(x)
        rgb, sig = sn(x[:, :3] + flow, torch.cat([xyzt[:, :3], dirs], 1).to(DEV), x[:, 3:])
        params = dict(mn.named_parameters())
    else:
        params = {k: v.detach().to(device, dtype).clone().requires_grad_(True) for k, v in mw.items()}
        sww = {k: v.to(device, dtype) for k, v in sw.items()}
        x = xyzt.to(device, dtype)
        flow = O.motionnet_forward(params, x)
        s_in = x[:, :3] + (flow if flow_at is None else flow_at.to(device, dtype) + (flow - flow.detach()))
        rgb, sig = O.spacenet_forward(sww, s_in, dirs.to(device, dtype), x[:, 3:] if NF.uses_time(sw) else None)
    loss = (rgb * _proj(rgb.shape, 1).to(rgb.device, rgb.dtype)).sum() + (sig * _proj(sig.shape, 2).to(sig.device, sig.dtype)).sum()
    loss.backward()
    return {k: v.grad.detach() for k, v in params.items()}, flow.detach()


@pytest.mark.parametrize("tag", ["syn_t", "tkd"])
def test_chained_motionnet_gradients_against_float64(tag):
    """flow = MotionNet(xyzt), then SpaceNet(xyz + flow): a loss on the SpaceNet reaches the MotionNet's weights via d_pos.
    Each fp32 path (native, CPU yardstick) is held to the float64 chain evaluated at ITS OWN SpaceNet input xyz + flow: the
    forward's rounding of the flow moves the point on PE(pos)'s 2^9 x terms, which is a property of the point, not of the
    gradient arithmetic under test."""
    nets = _weights(tag)
    for s in ("rays", "times"):
        pos, dirs, tm = points()[s]
        xyzt = torch.cat([pos, tm], 1)
        mw, sw = nets["motion"][0], nets["space"][0]

        def f64():
            x = xyzt.to(DEV, torch.float64)
            O.spacenet_forward(_f64(sw), x[:, :3] + O.motionnet_forward(_f64(mw), x), dirs.to(DEV, torch.float64),
                               x[:, 3:] if NF.uses_time(sw) else None)
        keep = kink_free(f64, KINK_CHAINED)
        args = (mw, sw, xyzt[keep], dirs[keep])
        nat, flow_nat = _chained(*args, DEV, torch.float32, True)
        cpu, flow_cpu = _chained(*args, "cpu", torch.float32, False)
        nat = grad_errors(nat, _chained(*args, DEV, torch.float64, False, flow_at=flow_nat)[0])
        cpu = grad_errors(cpu, _chained(*args, DEV, torch.float64, False, flow_at=flow_cpu)[0])
        assert_within_twice(nat, cpu, "chained %s/%s" % (tag, s), CHAINED_FACTOR)


# ---------------------------------------------------------------------------------------------------------------------
# forward: bit-identical to the fp32 inference kernels, independent of the batch
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("tag", ["syn_t", "syn", "tkd"])
def test_forward_bit_identical_to_fp32_mode(tag):
    from stnerf_b200 import NativeRenderer
    sd = NF.state_dict(tag)
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    nets = O.split_state_dict(sd, 1)
    r = NativeRenderer(2, [False, NF.uses_time(nets["space"][0])], "fp32")
    r.load_state_dict(sd)
    with torch.no_grad():
        for s in SETS:
            pos, dirs, tm = (x.to(DEV) for x in NF.point_sets()[s])
            for name, layer, fine in NF.SPACE_NETS:
                w = NF.space_weights(nets, name)
                rgb, sig = space_module(w)(pos, torch.cat([pos, dirs], 1), tm)
                rgb0, sig0 = r.spacenet(layer, fine, pos, dirs, tm if NF.uses_time(w) else None)
                assert _same(rgb, rgb0) and _same(sig, sig0), (tag, s, name)
            xyzt = torch.cat([pos, tm], 1)
            for lerp_mode in (-1, 0, 1):
                flow = motion_module(nets["motion"][0])(xyzt, lerp_mode)
                assert _same(flow, r.motionnet(1, xyzt, lerp_mode)), (tag, s, lerp_mode)
    r.close()


def test_forward_rows_independent_of_batch():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sn, mn = space_module(w["space"][0]), motion_module(w["motion"][0])
    g = torch.Generator().manual_seed(5)
    n = 5 * 128 * 132 + 77                                      # several CTAs' worth of tiles + a partial tile
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


def test_repeated_calls_give_identical_gradients():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    pos, dirs, tm = points()["gauss"]
    a, b = native_space_grads(w["space"][0], pos, dirs, tm), native_space_grads(w["space"][0], pos, dirs, tm)
    assert all(_same(a[k], b[k]) for k in a)
    xyzt = torch.cat([pos, tm + 0.25], 1)
    a, b = native_motion_grads(w["motion"][0], xyzt), native_motion_grads(w["motion"][0], xyzt)
    assert all(_same(a[k], b[k]) for k in a)


def test_zero_points():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sn, mn = space_module(w["space"][0]), motion_module(w["motion"][0])
    pos = torch.zeros((0, 3), device=DEV, requires_grad=True)
    rgb, sig = sn(pos, torch.zeros((0, 6), device=DEV), torch.zeros((0, 1), device=DEV))
    (rgb.sum() + sig.sum()).backward()
    assert rgb.shape == (0, 3) and sig.shape == (0, 1) and pos.grad.shape == (0, 3)
    assert all(float(p.grad.abs().max()) == 0.0 for p in sn.parameters())
    flow = mn(torch.zeros((0, 4), device=DEV))
    flow.sum().backward()
    assert flow.shape == (0, 3) and all(float(p.grad.abs().max()) == 0.0 for p in mn.parameters())


def test_bins_mode_and_box_normalisation_shapes():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    sn, mn = space_module(w["space"][0]), motion_module(w["motion"][0])
    pos = torch.randn((7, 5, 3), device=DEV)
    rays = torch.randn((7, 6), device=DEV)
    tm = torch.full((7, 1), 3.0, device=DEV)
    maxs, mins = torch.full((3,), 2.0, device=DEV), torch.full((3,), -2.0, device=DEV)
    rgb, sig = sn(pos, rays, tm, maxs, mins)
    assert rgb.shape == (7, 5, 3) and sig.shape == (7, 5, 1)
    flat_rgb, _ = sn(((pos.reshape(-1, 3) - mins) / (maxs - mins) - 0.5) * 2,
                     rays[:, None].expand(-1, 5, -1).reshape(-1, 6), tm[:, None].expand(-1, 5, -1).reshape(-1, 1))
    assert _same(rgb.reshape(-1, 3), flat_rgb)
    assert mn(torch.randn((7, 5, 4), device=DEV)).shape == (7, 5, 3)


# ---------------------------------------------------------------------------------------------------------------------
# closing the loop: fine-tune, write back, render
# ---------------------------------------------------------------------------------------------------------------------
ADAM_STEPS = 50
# final-loss gap between the native modules and the fp32 torch restatement after ADAM_STEPS steps, relative to the latter
ADAM_REL_TOL = 1.2e-2      # measured 5.7e-3 on one H100 80GB HBM3 (700 W power limit)


def _fit(native, sw, mw, xyzt, dirs, target_rgb, target_sig):
    torch.backends.cuda.matmul.allow_tf32 = False
    if native:
        sn, mn = space_module(sw), motion_module(mw)
        params = list(sn.parameters()) + list(mn.parameters())

        def run():
            flow = mn(xyzt)
            return sn(xyzt[:, :3] + flow, torch.cat([xyzt[:, :3], dirs], 1), xyzt[:, 3:])
    else:
        sp = {k: v.detach().to(DEV).clone().requires_grad_(True) for k, v in sw.items()}
        mp = {k: v.detach().to(DEV).clone().requires_grad_(True) for k, v in mw.items()}
        params = list(sp.values()) + list(mp.values())

        def run():
            flow = O.motionnet_forward(mp, xyzt)
            return O.spacenet_forward(sp, xyzt[:, :3] + flow, dirs, xyzt[:, 3:] if NF.uses_time(sw) else None)
    opt = torch.optim.Adam(params, lr=2e-4)
    losses = []
    for _ in range(ADAM_STEPS):
        opt.zero_grad()
        rgb, sig = run()
        loss = (torch.sigmoid(rgb) - target_rgb).pow(2).mean() + 1e-3 * (sig - target_sig).pow(2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    return losses, (sn, mn) if native else None


def test_adam_steps_decrease_the_loss_like_torch():
    w = O.split_state_dict(NF.state_dict("syn_t"), 1)
    g = torch.Generator().manual_seed(9)
    n = 4096
    pos = torch.randn((n, 3), generator=g)
    dirs = torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=1)
    xyzt = torch.cat([pos, torch.full((n, 1), 20.0)], 1).to(DEV)
    dirs = dirs.to(DEV)
    target_rgb = (0.5 + 0.4 * torch.sin(2.0 * pos)).to(DEV)
    target_sig = (10.0 * torch.exp(-pos.pow(2).sum(1, keepdim=True))).to(DEV)
    nat, _ = _fit(True, w["space"][0], w["motion"][0], xyzt, dirs, target_rgb, target_sig)
    ref, _ = _fit(False, w["space"][0], w["motion"][0], xyzt, dirs, target_rgb, target_sig)
    gap = abs(nat[-1] - ref[-1]) / ref[-1]
    print("adam: loss %.6g -> %.6g native, %.6g -> %.6g torch fp32, relative gap %.3g" % (nat[0], nat[-1], ref[0], ref[-1], gap))
    assert nat[-1] < 0.9 * nat[0]
    assert gap < ADAM_REL_TOL, gap


def test_fine_tuned_weights_round_trip_into_a_render():
    from stnerf_b200 import nets
    from tests_support import build_case_model
    name = "syn_L2_64_128"
    case = C.CASES[name]
    model = build_case_model(name, "fp32")
    d = nets.from_layered(model).to(DEV)
    opt = torch.optim.Adam(d.parameters(), lr=1e-3)
    pos = torch.randn((512, 3), device=DEV)
    rays = torch.cat([pos, torch.nn.functional.normalize(torch.randn((512, 3), device=DEV), dim=1)], 1)
    tm = torch.full((512, 1), 5.0, device=DEV)
    for _ in range(3):
        opt.zero_grad()
        rgb, sig = d["spacenets"][0](pos + d["time_deform_nets"][0](torch.cat([pos, tm], 1)), rays, tm)
        rgb2, sig2 = d["bkgd_spacenet_fine"](pos, rays, tm)
        (rgb.pow(2).mean() + sig.pow(2).mean() + rgb2.pow(2).mean() + sig2.pow(2).mean()).backward()
        opt.step()
    sd = d.state_dict()
    model.load_state_dict(sd)
    fresh = build_case_model(name, "fp32", sd=model.state_dict())
    rays_c = C.rays_for(case).to(DEV)
    jit, u = C.uniforms_for(case)
    outs = []
    for m in (model, fresh):
        m.inject_uniforms(jit.to(DEV), None if u is None else u.to(DEV))
        with torch.no_grad():
            outs.append(C.flatten_outputs(*m(rays_c, torch.zeros(rays_c.shape[0], device=DEV), None,
                                             density_threshold=case["thr"][0], bkgd_density_threshold=case["thr"][1])))
    before = build_case_model(name, "fp32")
    assert not torch.equal(sd["spacenets.0.stage1.0.weight"].cpu(), before.state_dict()["spacenets.0.stage1.0.weight"])
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), k
