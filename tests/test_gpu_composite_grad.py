"""Differentiable compositing (stnerf_b200.volume over csrc/composite.cu composite_backward_kernel) on the device.

Gradients: d_rgb and d_sigma against float64 autograd of the restatement in tests/test_composite_grad.py (pinned there to the
unmodified reference's own gradients), on random rays, on the coarse / fine depths of a scale fixture with sigma and rgb from the
native networks, and on the golden edge cases; every S in SIZES and every subset of upstream gradients.  The budget follows
tests/test_gpu_nets_train.py: rms and max error within twice the torch fp32 autograd error on the same inputs, plus ULP_FLOOR
(the larger of the CPU's and the GPU's, see `yardstick`).
Bits: the forward is ops.composite's, repeated backward calls agree, a ray's gradients do not depend on its batch, and the
layers facade returns what it returned before it became differentiable.
Merged: composite_merged against float64 with ties in depth, each tie's gradient on the sample the stable order put last.
Training chain: one step of a two-layer synthetic scene from native parts only, every parameter gradient against float64.
"""
import itertools

import pytest
import torch

import cases as C
import test_composite_grad as CG
import test_gpu_nets_train as NT
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
SIZES = (1, 31, 32, 33, 64, 90, 192, 256, 1000)
UPSTREAMS = ("color", "depth", "acc", "w")


def _vol():
    from stnerf_b200 import volume
    return volume


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def random_set(N, S, seed):
    """fp32 t (N,S) ascending, rgb (N,S,3), sigma (N,S): negative, zero, small and opaque densities, rays opaque early."""
    g = torch.Generator().manual_seed(seed)
    t = 1.0 + torch.cumsum(torch.rand((N, S), generator=g) * 0.08 + 0.002, 1)
    rgb = torch.randn((N, S, 3), generator=g) * 2.0
    sigma = torch.randn((N, S), generator=g) * 6.0
    sigma[torch.rand((N, S), generator=g) < 0.05] = 0.0
    dense = torch.rand((N,), generator=g) < 0.2
    sigma[dense] = sigma[dense].abs() * 40.0
    opaque = torch.rand((N, S), generator=g) < 0.01
    sigma[opaque] = 2.0e3
    return t, rgb, sigma


def upstreams(N, S, seed):
    g = torch.Generator().manual_seed(seed)
    return {"color": torch.randn((N, 3), generator=g), "depth": torch.randn((N, 1), generator=g),
            "acc": torch.randn((N, 1), generator=g), "w": torch.randn((N, S), generator=g)}


def _loss(outs, ups):
    return sum((outs[UPSTREAMS.index(k)] * v).sum() for k, v in ups.items())


def _leaf(x, device, dtype):
    return x.detach().to(device, dtype).clone().requires_grad_(True)


def native_grads(t, rgb, sigma, ups):
    r, s = _leaf(rgb, DEV, torch.float32), _leaf(sigma, DEV, torch.float32)
    outs = _vol().composite(t.to(DEV), r, s)
    torch.autograd.backward([outs[UPSTREAMS.index(k)] for k in ups], [v.to(DEV) for v in ups.values()])
    return {"d_rgb": r.grad, "d_sigma": s.grad}


def ref_grads(t, rgb, sigma, ups, device, dtype):
    r, s = _leaf(rgb, device, dtype), _leaf(sigma, device, dtype)
    _loss(CG.composite_ref(t.to(device, dtype), r, s), {k: v.to(device, dtype) for k, v in ups.items()}).backward()
    return {"d_rgb": torch.zeros_like(r) if r.grad is None else r.grad, "d_sigma": s.grad}    # no d_color: rgb unused


def check_against_f64(t, rgb, sigma, ups, what):
    truth = ref_grads(t, rgb, sigma, ups, DEV, torch.float64)
    got = native_grads(t, rgb, sigma, ups)
    for k in got:
        fin = torch.isfinite(truth[k])
        assert bool(torch.isfinite(got[k])[fin].all()), (what, k, "non-finite where float64 is finite")
    nat = NT.grad_errors(got, truth)
    yard = yardstick(NT.grad_errors(ref_grads(t, rgb, sigma, ups, "cpu", torch.float32), truth),
                     NT.grad_errors(ref_grads(t, rgb, sigma, ups, DEV, torch.float32), truth))
    NT.assert_within_twice(nat, yard, what)


def yardstick(cpu, gpu):
    """Per tensor, the larger error of torch fp32 autograd on the CPU and on the GPU.  The CPU's cumprod / cumsum accumulate
    in double, the GPU's (where the reference trains) in fp32 like the native kernels; a scan-heavy gradient can be several
    times more accurate on the CPU than the reference's own arithmetic on the device."""
    return {k: (max(cpu[k][0], gpu[k][0]), max(cpu[k][1], gpu[k][1])) for k in cpu}


def _subsets():
    return [c for n in range(1, 5) for c in itertools.combinations(UPSTREAMS, n)]


@pytest.mark.parametrize("S", SIZES)
def test_random_rays_every_upstream_subset(S):
    N = max(64, 4096 // S)
    t, rgb, sigma = random_set(N, S, 100 + S)
    ups = upstreams(N, S, 200 + S)
    for sub in _subsets():
        check_against_f64(t, rgb, sigma, {k: ups[k] for k in sub}, "random S=%d %s" % (S, "+".join(sub)))


def test_no_upstream_gives_zero_gradients():
    """Every upstream pointer NULL: the gradients are exact zeros (through the C ABI, which autograd never calls so)."""
    from stnerf_b200 import _lib as L
    t, rgb, sigma = (x.to(DEV) for x in random_set(40, 33, 7))
    d_rgb, d_sigma = torch.full((40, 33, 3), 7.0, device=DEV), torch.full((40, 33), 7.0, device=DEV)
    L.check(L.lib().stnerf_composite_backward(L.ptr(t), L.ptr(rgb), L.ptr(sigma), 40, 33, 1e10, None, None, None, None,
                                              L.ptr(d_rgb), L.ptr(d_sigma), L.stream_ptr()))
    torch.cuda.synchronize()
    assert float(d_rgb.abs().max()) == 0.0 and float(d_sigma.abs().max()) == 0.0


@pytest.mark.parametrize("S", CG.G.SAMPLE_COUNTS)
def test_golden_edge_cases(S):
    """Negative sigma, sigma = 0, transmittance underflowing behind opaque samples, a tiny sigma on the border sample."""
    t, rgb, sigma, proj = CG.golden_case(S)
    ups = {"color": proj["color"].float(), "depth": proj["depth"].float(), "acc": proj["acc"].float(), "w": proj["w"].float()}
    got = native_grads(t, rgb, sigma, ups)
    assert all(bool(torch.isfinite(v).all()) for v in got.values()), S
    check_against_f64(t, rgb, sigma, ups, "golden S=%d" % S)
    for sub in _subsets():
        check_against_f64(t, rgb, sigma, {k: ups[k] for k in sub}, "golden S=%d %s" % (S, "+".join(sub)))


@pytest.mark.parametrize("S", SIZES)
def test_border_and_underflow_hazards_stay_finite(S):
    t, rgb, sigma = random_set(16, S, 300 + S)
    sigma[0, :] = -1.0                     # transparent in front of the border sample: T = 1 there
    sigma[0, -1] = 1e-12                   # border: alpha ~ 0.01, delta = 1e10 -> d_sigma ~ 1e10, finite
    sigma[1, -1] = 5.0                     # border: alpha = 1, f = 1e-10
    sigma[2, :] = 5.0e3                    # every sample opaque: T underflows to 0 after four samples
    sigma[3, :] = -1.0
    ups = upstreams(16, S, 400 + S)
    got = native_grads(t, rgb, sigma, ups)
    truth = ref_grads(t, rgb, sigma, ups, DEV, torch.float64)
    for k in got:
        assert bool(torch.isfinite(got[k]).all()) and bool(torch.isfinite(truth[k]).all()), (S, k)
    assert float(got["d_sigma"][3].abs().max()) == 0.0
    if S > 1:
        rel = float((got["d_sigma"][0, -1].double() - truth["d_sigma"][0, -1]).abs() / truth["d_sigma"][0, -1].abs())
        assert rel < 1e-4, rel


def _scale_point_sets():
    """Coarse (64) and fine (192) depths of the first scale fixture's rays through the background and performer boxes, with
    rgb and sigma from native SpaceNets (synthetic weights) and the fine depths from ops.sample_pdf on the coarse weights."""
    from stnerf_b200 import ops
    case = C.SCALE_CASES["scale_tkd2_16k"]
    rays, jit, u = C.scale_inputs(case)
    sc = C.scene_for(case)
    keep = torch.arange(0, rays.shape[0], 4)
    rays, jit, u = rays[keep].to(DEV), jit[:, keep].to(DEV), u[:, keep, :].to(DEV)
    sd = O.synthetic_state_dict(1, True, seed=21)
    nn_ = O.split_state_dict(sd, 1)
    out = []
    for i, w in ((0, nn_["bkgd"]), (1, nn_["space"][0])):
        net = NT.space_module(w)
        t, xyz, mask, _ = ops.intersect_sample(rays, sc["bmin"][i], sc["bmax"][i], case["n1"], jit[i], is_bkgd=(i == 0))
        t, xyz = t[mask], xyz[mask]
        n = t.shape[0]
        dirs = rays[mask][:, None, 3:6].expand(n, t.shape[1], 3).reshape(-1, 3)
        tm = rays[mask][:, 6 + i:7 + i][:, None].expand(n, t.shape[1], 1).reshape(-1, 1)
        with torch.no_grad():
            rgb, sig = net(xyz.reshape(-1, 3), torch.cat([xyz.reshape(-1, 3), dirs], 1), tm)
            out.append((t, rgb.reshape(n, -1, 3), sig.reshape(n, -1)))
            w_c = ops.composite(t, rgb.reshape(n, -1, 3), sig.reshape(n, -1))[3]
            _, tf = ops.sample_pdf(t, w_c, u[i][mask], merge=True)
            xf = rays[mask][:, None, :3] + tf[..., None] * rays[mask][:, None, 3:6]
            dirs = rays[mask][:, None, 3:6].expand(n, tf.shape[1], 3).reshape(-1, 3)
            tm = rays[mask][:, 6 + i:7 + i][:, None].expand(n, tf.shape[1], 1).reshape(-1, 1)
            rgb, sig = net(xf.reshape(-1, 3), torch.cat([xf.reshape(-1, 3), dirs], 1), tm)
            out.append((tf, rgb.reshape(n, -1, 3), sig.reshape(n, -1)))
    return [(t.cpu(), r.cpu(), s.cpu()) for t, r, s in out]


def test_scale_fixture_depths_with_native_network_outputs():
    for k, (t, rgb, sigma) in enumerate(_scale_point_sets()):
        N, S = t.shape
        ups = upstreams(N, S, 500 + k)
        check_against_f64(t, rgb, sigma, ups, "scale set %d (S=%d, %d rays)" % (k, S, N))
        check_against_f64(t, rgb, sigma, {"color": ups["color"], "acc": ups["acc"]}, "scale set %d color+acc" % k)


# ---------------------------------------------------------------------------------------------------------------------
# bit identities
# ---------------------------------------------------------------------------------------------------------------------
def test_forward_is_ops_composite_bit_for_bit():
    from stnerf_b200 import ops
    for S in SIZES:
        t, rgb, sigma = (x.to(DEV) for x in random_set(100, S, 600 + S))
        want = ops.composite(t, rgb, sigma)
        got = _vol().composite(t, rgb.clone().requires_grad_(True), sigma.clone().requires_grad_(True))
        assert all(_same(a, b) for a, b in zip(got, want)), S
        with torch.no_grad():
            got = _vol().composite(t, rgb.clone().requires_grad_(True), sigma)
        assert all(_same(a, b) for a, b in zip(got, want)), S


def test_repeated_backward_calls_identical():
    for S in (33, 192, 1000):
        t, rgb, sigma = random_set(300, S, 700 + S)
        ups = upstreams(300, S, 800 + S)
        a, b = native_grads(t, rgb, sigma, ups), native_grads(t, rgb, sigma, ups)
        assert all(_same(a[k], b[k]) for k in a), S


def test_rays_independent_of_batch():
    for S in (1, 33, 192):
        n = 5000
        t, rgb, sigma = random_set(n, S, 900 + S)
        ups = upstreams(n, S, 1000 + S)
        full = native_grads(t, rgb, sigma, ups)
        for sl in [slice(0, k) for k in (1, 7, 8, 9, 2049)] + [slice(k, n) for k in (1, 8, 31, 256)]:
            part = native_grads(t[sl], rgb[sl], sigma[sl], {k: v[sl] for k, v in ups.items()})
            assert all(_same(part[k], full[k][sl.start:sl.stop]) for k in part), (S, sl)
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(S))
        part = native_grads(t[perm], rgb[perm], sigma[perm], {k: v[perm] for k, v in ups.items()})
        assert all(_same(part[k], full[k][perm.to(DEV)]) for k in part), S


def test_layers_facade_values_unchanged():
    import layers
    from layers.render_layer import gen_weight
    from stnerf_b200 import ops
    for S in (2, 64, 192):
        t, rgb, sigma = (x.to(DEV) for x in random_set(50, S, 1100 + S))
        want = ops.composite(t, rgb, sigma)
        vr = layers.VolumeRenderer(boarder_weight=1e10)
        for grad in (False, True):
            r, s = rgb.clone().requires_grad_(grad), sigma[..., None].clone().requires_grad_(grad)
            c, d, a, w = vr(t[..., None], r, s)
            assert _same(c, want[0]) and _same(d, want[1]) and _same(a, want[2]) and _same(w[..., 0], want[3]), (S, grad)
            if grad:
                (c.sum() + w.sum()).backward()
                assert r.grad.shape == r.shape and s.grad.shape == s.shape
        delta = torch.cat([t[:, 1:] - t[:, :-1], torch.full((50, 1), 1e10, device=DEV)], 1)
        tt = torch.cumsum(torch.cat([torch.zeros_like(delta[:, :1]), delta[:, :-1]], 1), 1)
        want_w = ops.composite(tt, torch.zeros((50, S, 3), device=DEV), sigma, 1e10)[3]
        s = sigma[..., None].clone().requires_grad_(True)
        assert _same(gen_weight(s, delta), want_w)
        with pytest.raises(NotImplementedError):
            gen_weight(s, delta.clone().requires_grad_(True))


# ---------------------------------------------------------------------------------------------------------------------
# merged composite: ties route the gradient like the stable (t, cat index) order
# ---------------------------------------------------------------------------------------------------------------------
def _merged_grads(ts, rgbs, sigmas, near, device, dtype, native):
    rs = [_leaf(r, device, dtype) for r in rgbs]
    ss = [_leaf(s, device, dtype) for s in sigmas]
    tt = [t.to(device, dtype) for t in ts]
    fn = _vol().composite_merged if native else CG.merged_ref
    c, d, a = fn(tt, rs, ss, 1e10, near)
    g = torch.Generator().manual_seed(77)
    (c * torch.randn(c.shape, generator=g).to(device, dtype)).sum().backward(retain_graph=True)
    (d * torch.randn(d.shape, generator=g).to(device, dtype) + a * torch.randn(a.shape, generator=g).to(device, dtype)).sum().backward()
    out = {}
    for i, (r, s) in enumerate(zip(rs, ss)):
        out["d_rgb%d" % i], out["d_sigma%d" % i] = r.grad, s.grad
    return out


@pytest.mark.parametrize("near", [None, 1.5])
def test_merged_gradients_with_ties(near):
    N, S = 256, 64
    t0, r0, _ = random_set(N, S, 1200)
    t1, r1, _ = random_set(N, S, 1201)
    g = torch.Generator().manual_seed(1202)
    s0, s1 = torch.rand((N, S), generator=g) * 2.0 + 0.2, torch.rand((N, S), generator=g) * 2.0 + 0.2
    dup = torch.zeros((N, S), dtype=torch.bool)
    dup[:, 10:50:5] = True
    t1 = torch.where(dup, t0, t1)                                   # duplicated depths across the two layers
    t1, order = torch.sort(t1, 1)
    dup = dup.gather(1, order)
    missed = torch.arange(N) % 7 == 3                               # a missed layer: every depth equal, sigma 0
    t2 = torch.where(missed[:, None], torch.full((N, S), 2.0), t1 + 0.013)
    r2, s2 = torch.randn((N, S, 3)), torch.where(missed[:, None], torch.zeros((N, S)), s1 * 0.5)
    ts, rgbs, sigmas = [t0, t1, t2], [r0, r1, r2], [s0, s1, s2]
    truth = _merged_grads(ts, rgbs, sigmas, near, DEV, torch.float64, False)
    nat = NT.grad_errors(_merged_grads(ts, rgbs, sigmas, near, DEV, torch.float32, True), truth)
    yard = yardstick(NT.grad_errors(_merged_grads(ts, rgbs, sigmas, near, "cpu", torch.float32, False), truth),
                     NT.grad_errors(_merged_grads(ts, rgbs, sigmas, near, DEV, torch.float32, False), truth))
    NT.assert_within_twice(nat, yard, "merged near=%s" % near)
    got = _merged_grads(ts, rgbs, sigmas, near, DEV, torch.float32, True)
    # a tie (layer 0 sample, layer 1 sample) sorts layer 0 first: its delta is 0, so only the layer-1 sample absorbs
    d0 = got["d_sigma0"].cpu()
    d1 = got["d_sigma1"].cpu()
    src0 = torch.zeros((N, S), dtype=torch.bool)
    for r in range(N):
        src0[r] = torch.isin(t0[r], t1[r][dup[r]])
    assert float(d0[src0].abs().max()) == 0.0
    live = dup & (t1 >= (near if near is not None else -1e30))
    assert float((d1[live] != 0).float().mean()) > 0.8
    # the missed layer's equal depths: every one but the last of the tie has delta 0 and no sigma gradient
    assert float(got["d_sigma2"].cpu()[missed].abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# empty and invalid calls
# ---------------------------------------------------------------------------------------------------------------------
def test_empty_and_invalid_calls():
    from stnerf_b200 import _lib as L
    vol = _vol()
    r = torch.zeros((0, 8, 3), device=DEV, requires_grad=True)
    s = torch.zeros((0, 8), device=DEV, requires_grad=True)
    c, d, a, w = vol.composite(torch.zeros((0, 8), device=DEV), r, s)
    assert c.shape == (0, 3) and d.shape == (0, 1) and a.shape == (0, 1) and w.shape == (0, 8)
    (c.sum() + w.sum()).backward()
    assert r.grad.shape == (0, 8, 3) and s.grad.shape == (0, 8)
    lib = L.lib()
    assert lib.stnerf_composite_backward(None, None, None, 0, 8, 1e10, None, None, None, None, None, None, None) == 0
    x = torch.zeros((2, 8), device=DEV)
    x3 = torch.zeros((2, 8, 3), device=DEV)
    p = L.ptr
    assert lib.stnerf_composite_backward(p(x), p(x3), p(x), -1, 8, 1e10, None, None, None, None, p(x3), p(x), None) == -1
    assert lib.stnerf_composite_backward(p(x), p(x3), p(x), 2, 0, 1e10, None, None, None, None, p(x3), p(x), None) == -1
    assert lib.stnerf_composite_backward(p(x), p(x3), None, 2, 8, 1e10, None, None, None, None, p(x3), p(x), None) == -1
    assert lib.stnerf_composite_backward(p(x), p(x3), p(x), 2, 8, 1e10, None, None, None, None, None, p(x), None) == -1
    t = torch.zeros((2, 8), device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError):
        vol.composite(t, x3.clone().requires_grad_(True), x)
    with pytest.raises(NotImplementedError):
        vol.CompositeFunction.apply(t, x3, x, 1e10)
    with torch.no_grad():
        assert _same(vol.composite(t, x3, x)[3], vol.composite(t.detach(), x3, x)[3])


# ---------------------------------------------------------------------------------------------------------------------
# training chain: sampling -> MotionNet -> SpaceNet -> per-layer + merged composite -> sample_pdf -> fine pass -> loss
# ---------------------------------------------------------------------------------------------------------------------
CHAIN_CASE = dict(weights="synthetic", seed=31, L=1, space_time=True, n1=64, n2=128, seven=True, frame_ids=[10, 10],
                  thr=(20.0, 0.8), n_rays=192, ray_seed=41)
MASK_SCALAR = 100000.0                                          # layered_trainer.py:236 `scalar_max`
ADAM_STEPS = 30
ADAM_LR = 5e-4
# final-loss gap between the native chain and the torch fp32 restatement after ADAM_STEPS steps, relative to the latter
ADAM_REL_TOL = 1e-3        # measured 3.1e-5 on one H100 80GB HBM3 (700 W power limit)


def chain_inputs():
    from tests_support import build_case_model
    from stnerf_b200 import ops
    model = build_case_model(CHAIN_CASE, "fp32")
    rays = C.rays_for(CHAIN_CASE).to(DEV)
    jit, u = C.uniforms_for(CHAIN_CASE)
    jit, u = jit.to(DEV), u.to(DEV)
    bk, frames = C.boxes_for(CHAIN_CASE)
    f = int(float(rays[0, 6])) - 1                               # index_select(frame_id - 1) (layered_rfrender.py:193)
    boxes = [bk.reshape(8, 3), frames[f, 0]]
    samp = []
    for i, b in enumerate(boxes):
        t, xyz, mask, _ = ops.intersect_sample(rays, b[0], b[6], CHAIN_CASE["n1"], jit[i], is_bkgd=(i == 0))
        samp.append((t, xyz, mask if i > 0 else torch.ones_like(mask)))
    labels = samp[1][2].long()                                   # label 1 where the ray meets the performer's box
    g = torch.Generator().manual_seed(5)
    target = (0.5 + 0.4 * torch.sin(3.0 * rays[:, 3:6].cpu() + torch.rand((rays.shape[0], 3), generator=g))).to(DEV)
    return model, rays, jit, u, samp, labels, target


class NativeNets:
    def __init__(self, model):
        from stnerf_b200 import nets
        d = nets.from_layered(model).to(DEV)
        self.d = d
        self.space = [d["bkgd_spacenet"], d["spacenets"][0]]
        self.space_fine = [d["bkgd_spacenet_fine"], d["spacenets_fine"][0]]
        self.motion = d["time_deform_nets"][0]

    def params(self):
        return dict(self.d.named_parameters())

    def spacenet(self, i, fine, pos, dirs, times):
        net = (self.space_fine if fine else self.space)[i]
        return net(pos, torch.cat([pos.detach(), dirs], 1), times)

    def motionnet(self, xyzt):
        return self.motion(xyzt)


class RefNets:
    """The oracle's restatement with its own parameter tensors (any dtype / device), keyed like NativeNets.params()."""

    def __init__(self, model, device, dtype):
        self.p = {k: v.detach().to(device, dtype).clone().requires_grad_(True) for k, v in model.state_dict().items()
                  if k.split(".")[0] in ("spacenets", "spacenets_fine", "bkgd_spacenet", "bkgd_spacenet_fine", "time_deform_nets")}
        self.flow_at = None

    def _sub(self, prefix):
        return {k[len(prefix):]: v for k, v in self.p.items() if k.startswith(prefix)}

    def params(self):
        return self.p

    def spacenet(self, i, fine, pos, dirs, times):
        pre = ("bkgd_spacenet" + ("_fine" if fine else "") + ".") if i == 0 else ("spacenets" + ("_fine" if fine else "") + ".0.")
        w = self._sub(pre)
        return O.spacenet_forward(w, pos, dirs, times if NT.NF.uses_time(w) else None)

    def motionnet(self, xyzt):
        return O.motionnet_forward(self._sub("time_deform_nets.0."), xyzt)


def run_chain(nets, rays, samp, u_fine, labels, target, dtype, device, comp, merged, keep=None, flow_at=None,
              fine_t=None, record=None):
    """One training forward.  comp / merged: the compositing functions (native volume.* or the restatement).  keep: per
    network call, the points whose gradient flows into the weights (the rest are set aside, detached).  flow_at: evaluate each
    SpaceNet at xyz + flow_at[call] (float64 truth of an fp32 chain), with the gradient through this chain's own flow.
    fine_t: the fine depths to use (None: resample with ops.sample_pdf on the detached coarse weights).
    Returns loss, coarse per-layer images, coarse merged image, fine depths, flows."""
    from stnerf_b200 import ops
    rays = rays.to(device, dtype)
    o, d, fid = rays[:, :3], rays[:, 3:6], rays[:, 6:7]
    N = rays.shape[0]
    flows = {}

    def gate(x, k):
        if keep is None or k not in keep:
            return x
        m = keep[k].to(device)[:, None]
        return torch.where(m, x, x.detach())

    def layer(i, fine, t, xyz, mask):
        S = t.shape[1]
        idx = mask.to(device)
        M = int(idx.sum())
        rgb = torch.zeros((N, S, 3), dtype=dtype, device=device)
        sig = torch.zeros((N, S), dtype=dtype, device=device)
        if M == 0:
            return rgb, sig
        p = xyz[idx].reshape(-1, 3)
        dirs = d[idx][:, None, :].expand(M, S, 3).reshape(-1, 3)
        tm = fid[idx][:, None, :].expand(M, S, 1).reshape(-1, 1)
        key = "%s%d" % ("f" if fine else "c", i)
        if i > 0:
            flow = gate(nets.motionnet(torch.cat([p, tm], 1)), "m" + key)
            flows[key] = flow.detach()
            if flow_at is not None:
                p = p + flow_at[key].to(device, dtype) + (flow - flow.detach())
            else:
                p = p + flow
        r, s = nets.spacenet(i, fine, p, dirs, tm)
        r, s = gate(r, key), gate(s.reshape(-1, 1), key)
        rgb = rgb.index_put((idx,), r.reshape(M, S, 3))
        sig = sig.index_put((idx,), s.reshape(M, S))
        return rgb, sig

    ts, rgbs, sigs, layer_c = [], [], [], []
    for i, (t, xyz, mask) in enumerate(samp):
        t, xyz = t.to(device, dtype), xyz.to(device, dtype)
        rgb, sig = layer(i, False, t, xyz, mask)
        if i > 0:
            sig = torch.where(t < 0, torch.zeros_like(sig), sig)                       # layered_rfrender.py:414
        else:
            sig = torch.where(t < 0.0, torch.zeros_like(sig), sig)                     # :422 (near = 0)
        ts.append(t); rgbs.append(rgb); sigs.append(sig)
        layer_c.append(comp(t, rgb, sig))
    merged_c = merged(ts, rgbs, sigs, 1e10, None)
    if fine_t is None:
        fine_t = [ops.sample_pdf(ts[i].float().contiguous(), layer_c[i][3].detach().float(), u_fine[i], merge=True)[1]
                  for i in range(len(samp))]                                           # :459-462
    tf, rgbf, sigf, layer_f = [], [], [], []
    for i, (_, _, mask) in enumerate(samp):
        t = fine_t[i].to(device, dtype)
        xyz = t[..., None] * d[:, None, :] + o[:, None, :]                             # :465
        rgb, sig = layer(i, True, t, xyz, mask)
        tf.append(t); rgbf.append(rgb); sigf.append(sig)
        layer_f.append(comp(t, rgb, sig))
    merged_f = merged(tf, rgbf, sigf, 1e10, 0.0)                                       # :605-606 (near = 0)
    tgt = target.to(device, dtype)
    loss1 = torch.nn.functional.mse_loss(merged_c[0], tgt)
    loss2 = torch.nn.functional.mse_loss(merged_f[0], tgt)
    lab = labels.to(device)
    masks = []
    for stage in (layer_c, layer_f):                                                   # layered_trainer.py:216-281
        out = torch.cat([stage[i][2][lab == 0] for i in range(1, len(samp))], 0)
        inl = torch.cat([stage[i][2][lab == i] for i in range(len(samp))], 0)
        masks.append((out.abs().sum() + (1 - inl).abs().sum()) / MASK_SCALAR)
    loss = loss1 + loss2 + masks[0] + masks[1]
    if record is not None:
        record.update(layer_c=layer_c, merged_c=merged_c, fine_t=[x.detach().float() for x in fine_t], flows=flows,
                      mask_losses=[float(m) * MASK_SCALAR for m in masks])
    return loss


def _ref_comp(t, rgb, sig):
    return CG.composite_ref(t, rgb, sig)


def _ref_merged(ts, rgbs, sigs, boarder, near):
    return CG.merged_ref(ts, rgbs, sigs, boarder, near)


def _native_comp(t, rgb, sig):
    return _vol().composite(t, rgb, sig)


def _native_merged(ts, rgbs, sigs, boarder, near):
    return _vol().composite_merged(ts, rgbs, sigs, boarder, near)


def _kink_keep(model, rays, samp, fine_t):
    """Per network call: points none of whose float64 hidden pre-activations lies near a ReLU kink (NT.kink_free), for the
    MotionNet and for the SpaceNet it feeds (NT.KINK_CHAINED there: its input carries the MotionNet's rounding)."""
    ref = RefNets(model, DEV, torch.float64)
    keep = {}
    real_space, real_motion = ref.spacenet, ref.motionnet

    def space(i, fine, pos, dirs, times):
        key = "%s%d" % ("f" if fine else "c", i)
        kk = NT.kink_free(lambda: real_space(i, fine, pos.detach(), dirs, times), NT.KINK_CHAINED if i > 0 else NT.KINK)
        keep[key] = kk if i == 0 else kk & keep.pop("_m")
        return real_space(i, fine, pos, dirs, times)

    def motion(xyzt):
        keep["_m"] = NT.kink_free(lambda: real_motion(xyzt.detach()))
        return real_motion(xyzt)
    ref.spacenet, ref.motionnet = space, motion
    with torch.no_grad():
        run_chain(ref, rays, samp, None, torch.zeros(rays.shape[0], dtype=torch.long), torch.zeros((rays.shape[0], 3)),
                  torch.float64, DEV, _ref_comp, _ref_merged, fine_t=fine_t)
    for k in [k for k in keep if not k.endswith("0")]:
        keep["m" + k] = keep[k]                                  # the flow of a set-aside point is set aside with it
    return keep


def _grads(params):
    return {k: (v.grad.detach().clone() if v.grad is not None else torch.zeros_like(v)) for k, v in params.items()}


def test_training_chain_forward_matches_layered_rf_render():
    """The chain's coarse per-layer and merged images are LayeredRFRender.forward's (fp32 mode, same rays and jitter)."""
    model, rays, jit, u, samp, labels, target = chain_inputs()
    rec = {}
    with torch.no_grad():
        run_chain(NativeNets(model), rays, samp, u, labels, target, torch.float32, DEV, _native_comp, _native_merged,
                  record=rec)
        model.inject_uniforms(jit, u)
        fine_mixed, coarse_mixed, fine_layer, coarse_layer, ray_mask = model(rays, torch.zeros(rays.shape[0], device=DEV), None)
    assert torch.equal(ray_mask[1].cpu(), samp[1][2].cpu())
    worst = 0.0
    for got, want in [(rec["merged_c"], coarse_mixed)] + list(zip(rec["layer_c"], coarse_layer)):
        for a, b in zip(got[:3], want):
            worst = max(worst, float((a.reshape(b.shape) - b).abs().max()))
    print("chain vs LayeredRFRender.forward coarse images: max |diff| %.3g" % worst)
    assert worst <= 1e-5, worst
    assert int(samp[1][2].sum()) > 20 and int((~samp[1][2]).sum()) > 20


def test_training_chain_gradients_against_float64():
    torch.backends.cuda.matmul.allow_tf32 = False
    model, rays, jit, u, samp, labels, target = chain_inputs()
    nat_nets = NativeNets(model)
    rec = {}
    run_chain(nat_nets, rays, samp, u, labels, target, torch.float32, DEV, _native_comp, _native_merged, record=rec)
    fine_t = rec["fine_t"]
    keep = _kink_keep(model, rays, samp, fine_t)
    print("chain: kept points per call %s" % {k: "%d/%d" % (int(v.sum()), v.numel()) for k, v in keep.items()})
    assert min(rec["mask_losses"]) > rays.shape[0] * 0.0005          # the trainer's condition for a nonzero mask loss (:254)

    nat_nets.d.zero_grad()
    rec = {}
    run_chain(nat_nets, rays, samp, u, labels, target, torch.float32, DEV, _native_comp, _native_merged, keep=keep,
              fine_t=fine_t, record=rec).backward()
    nat = _grads(nat_nets.params())
    flows_nat = rec["flows"]
    cpu_nets = RefNets(model, "cpu", torch.float32)
    rec = {}
    run_chain(cpu_nets, rays.cpu(), [(t.cpu(), x.cpu(), m.cpu()) for t, x, m in samp], None, labels.cpu(), target.cpu(),
              torch.float32, "cpu", _ref_comp, _ref_merged, keep=keep, fine_t=[x.cpu() for x in fine_t], record=rec).backward()
    cpu = _grads(cpu_nets.params())
    flows_cpu = rec["flows"]
    gpu_nets = RefNets(model, DEV, torch.float32)
    rec = {}
    run_chain(gpu_nets, rays, samp, None, labels, target, torch.float32, DEV, _ref_comp, _ref_merged, keep=keep,
              fine_t=fine_t, record=rec).backward()
    gpu = _grads(gpu_nets.params())
    flows_gpu = rec["flows"]
    truths = []
    for flows in (flows_nat, flows_cpu, flows_gpu):
        ref = RefNets(model, DEV, torch.float64)
        run_chain(ref, rays, samp, None, labels, target, torch.float64, DEV, _ref_comp, _ref_merged, keep=keep,
                  flow_at=flows, fine_t=fine_t).backward()
        truths.append(_grads(ref.params()))
    used = [k for k in truths[0] if float(truths[0][k].abs().max()) > 0]
    assert any(k.startswith("time_deform_nets") for k in used) and any(k.startswith("bkgd_spacenet_fine") for k in used)
    e_nat = NT.grad_errors({k: nat[k] for k in used}, {k: truths[0][k] for k in used})
    e_cpu = NT.grad_errors({k: cpu[k] for k in used}, {k: truths[1][k] for k in used})
    e_gpu = NT.grad_errors({k: gpu[k] for k in used}, {k: truths[2][k] for k in used})
    NT.assert_within_twice(e_nat, yardstick(e_cpu, e_gpu), "training chain", NT.CHAINED_FACTOR)


def _fit(native, model, rays, samp, u, labels, target):
    torch.backends.cuda.matmul.allow_tf32 = False
    nets = NativeNets(model) if native else RefNets(model, DEV, torch.float32)
    params = list(nets.params().values())
    opt = torch.optim.Adam(params, lr=ADAM_LR)
    comp, merged = (_native_comp, _native_merged) if native else (_ref_comp, _ref_merged)
    losses = []
    for _ in range(ADAM_STEPS):
        opt.zero_grad()
        loss = run_chain(nets, rays, samp, u, labels, target, torch.float32, DEV, comp, merged)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    return losses


def test_training_chain_adam_steps_decrease_the_loss_like_torch():
    model, rays, jit, u, samp, labels, target = chain_inputs()
    nat = _fit(True, model, rays, samp, u, labels, target)
    ref = _fit(False, model, rays, samp, u, labels, target)
    gap = abs(nat[-1] - ref[-1]) / ref[-1]
    print("chain adam: loss %.6g -> %.6g native, %.6g -> %.6g torch fp32, relative gap %.3g" % (nat[0], nat[-1], ref[0], ref[-1], gap))
    assert nat[-1] < 0.9 * nat[0]
    assert gap < ADAM_REL_TOL, gap
