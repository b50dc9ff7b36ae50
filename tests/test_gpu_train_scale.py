"""The training networks at training batch sizes, against float64, in both training precisions (fp32, tf32x3).

test_gpu_nets_train*.py hold the gradients to float64 at 4096 points, where a weight gradient is 16 chunks of 256 points.
The chunking of csrc/mlp_train.cu changes with the batch size P: up to MIN_CHUNK * MAX_SPLIT = 32 768 points a chunk is 256
points; above, there are ~128 chunks of roundup16(ceil(P / 128)) points with a ragged last one.  Saved activations are
feature-major (row r of point p at r * P + p), so from P ~ 1.057 M a SpaceNet's last rows lie past 2^31 elements.  Here:

1. Dense gradients (every point with an upstream gradient) at P = 32 767, 32 769, 240 007 (the taekwondo fine background
   call) and 1 190 007 (a ragged last chunk; SpaceNet saved rows from h7's 206th on past 2^31 elements, the direction / time
   encoding rows among them), for synthetic weights with and without a time
   input and both shipped checkpoints where their copies are present, background and performer SpaceNets; the MotionNet at
   the chunk cap with lerp modes -1 and 1.  The float64 truth is the oracle's restatement run on the device in chunks of 2^16
   points, its parameter gradients accumulated in float64.  The yardstick is torch fp32 autograd of the same restatement on
   the device over the whole batch in one call (cuBLAS, TF32 off): what a user would otherwise train with.  Bars: the rms
   and the max of every tensor within 2x the yardstick's (fp32) or 4x (tf32x3), plus ULP_FLOOR.
2. Sparse-upstream probes: the upstream gradients are zero except on a few hundred probe points (first, second and last
   point of every weight-gradient chunk, both sides of 64- and 128-point tile edges, P - 2 and P - 1, and the points whose
   saved offset r * P + p is the first past 2^30 and 2^31 for some row r).  A point with zero upstream adds exactly nothing
   to any sum in both precisions, so the parameter gradients are those of the probes alone, held to float64 of the probes at
   the small-P bar; d_pos of every other point is exactly zero; the probes' outputs and d_pos equal, bit for bit, those of
   the probes run as a batch of their own.  This catches a dropped, doubled or misplaced point that an rms comparison over
   10^6 points cannot see.
3. A full training step at the taekwondo batch of scripts/bench_train_step.py (2000 rays, 7-column rays with mixed integer
   frame ids and per-ray boxes, 2 performers, 90 + 30 samples) against float64, the fine and the only_coarse stage, by
   test_gpu_train_forward.float64_step_check.  One tf32x3 tensor is a known defect (KNOWN below), held apart.

All point sets are kink-free (test_gpu_nets_train.kink_free, evaluated in chunks): no float64 pre-activation of a point lies
within KINK x its layer's rms of a ReLU kink, so each probe is its own nearest kink-free point.  Each leg (native, yardstick,
truth) frees its device memory before the next.  The module prints its wall time, its peak device memory and the card.
"""
import subprocess
import time

import pytest
import torch

import cases as C
import make_golden_train_grads as TG
import test_gpu_networks_f64 as NF
import test_gpu_nets_train as NT
import test_gpu_nets_train_tc as TC
import test_gpu_train_forward as TF
from oracle import stnerf_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
PRECS = ("fp32", "tf32x3")
# (factor, chained factor) of the bars per training precision: test_gpu_nets_train.py and test_gpu_nets_train_tc.py
FACTORS = {"fp32": (2.0, NT.CHAINED_FACTOR), "tf32x3": (TC.FACTOR, TC.CHAINED_FACTOR)}
MIN_CHUNK, MAX_SPLIT, TK = 256, 128, 16              # mlp_train.cu: weight-gradient chunking
CAP = MIN_CHUNK * MAX_SPLIT
SPACE_P = (CAP - 1, CAP + 1, 240_007, 1_190_007)
MOTION_P = (CAP - 1, CAP + 1)
BIG_DEPTHS = 112         # background depths per ray of the scale fixture's 16 384 rays: 1 835 008 points before kink filtering
CHUNK = 1 << 16          # points per chunk of the float64 legs
HID, HEAD, PE_POS = 256, 128, 63


def grad_chunk(P):
    """mlp_train.cu grad_chunk: points per weight-gradient chunk, a function of P alone."""
    c = -(-P // MAX_SPLIT)
    return MIN_CHUNK if c < MIN_CHUNK else -(-c // TK) * TK


def saved_rows(use_time):
    """rows of a SpaceNet's saved activations: h1-h4, PE(pos), h5-h7, ENC = PE(dir) [+ PE(t)], h8"""
    return 7 * HID + PE_POS + 27 + (21 if use_time else 0) + HEAD


class NoTF32:
    def __enter__(self):
        self.flag = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32 = self.flag


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return "%.0f W" % float(out.strip().splitlines()[0])
    except Exception:
        return "unknown"


@pytest.fixture(scope="module", autouse=True)
def _wall_time_and_peak_memory():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    print("\ntest_gpu_train_scale: wall time %.0f s, peak device memory %.2f GiB (%s, power limit %s)"
          % (time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30, torch.cuda.get_device_name(),
             _power_limit()))


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# points
# ---------------------------------------------------------------------------------------------------------------------
def kink_free_chunked(fwd, n, kink=NT.KINK):
    """test_gpu_nets_train.kink_free over n points, run CHUNK points at a time: fwd(sl) evaluates the float64 network on
    points sl.  Per layer, each point's smallest |pre-activation| is kept and compared at the end with kink x that layer's
    rms over all n points, so the mask is the one a single call would give."""
    real, mins, sq, width = O.F.linear, [], None, None
    for s in range(0, n, CHUNK):
        zs = []

        def rec(x, w, b=None):
            z = real(x, w, b)
            if w.shape[0] > 3:
                zs.append(z)
            return z
        O.F.linear = rec
        try:
            with torch.no_grad():
                fwd(slice(s, min(n, s + CHUNK)))
        finally:
            O.F.linear = real
        mins.append(torch.stack([z.abs().min(1).values for z in zs], 1))
        part = torch.stack([z.pow(2).sum() for z in zs])
        sq = part if sq is None else sq + part
        width = torch.tensor([z.shape[1] for z in zs], dtype=torch.float64, device=part.device)
    rms = (sq / (n * width)).sqrt()
    return (torch.cat(mins) >= kink * rms).all(1).cpu()


def _dev64(x, sl=slice(None)):
    return x[sl].to(DEV, torch.float64)


def _ray_set(n_rays, n_depths, seed):
    """test_gpu_networks_f64's `rays` set: background depths along the scale fixture's rays, n_rays of them spread over the
    view, ray-major (point = ray * n_depths + depth)."""
    rays, _, _ = C.scale_inputs(C.SCALE_CASES["scale_tkd2_16k"])
    rays = rays[torch.linspace(0, rays.shape[0] - 1, n_rays).long()]
    g = torch.Generator().manual_seed(seed)
    t = (torch.arange(n_depths)[None] + torch.rand((n_rays, n_depths), generator=g)) * 0.2 + 0.5
    pos = (rays[:, None, :3] + t[..., None] * rays[:, None, 3:6]).reshape(-1, 3)
    dirs = rays[:, None, 3:6].expand(-1, n_depths, -1).reshape(-1, 3)
    return pos.contiguous(), dirs.contiguous(), torch.full((pos.shape[0], 1), 10.0)


def _gauss_set(n, seed):
    """test_gpu_networks_f64's `gauss` set"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, 3), generator=g) * 1.5, NF._unit(g, n), torch.full((n, 1), 37.25)


def space_points(w, key, P):
    """P kink-free points for the SpaceNet w: the gauss set below the chunk cap, the rays set above it (every ray of the scale
    fixture for the largest P).  key: (weights, net, P), for the printout."""
    if P < CAP:
        pos, dirs, tm = _gauss_set(P + P // 2, P)
    elif P >= 1_000_000:
        pos, dirs, tm = _ray_set(16384, BIG_DEPTHS, P)
    else:
        pos, dirs, tm = _ray_set(-(-3 * P // (2 * 64)), 64, P)
    w64 = NT._f64(w)
    keep = kink_free_chunked(lambda sl: O.spacenet_forward(w64, _dev64(pos, sl), _dev64(dirs, sl),
                                                           _dev64(tm, sl) if NF.uses_time(w) else None), pos.shape[0])
    idx = keep.nonzero()[:, 0]
    print("%s: %d of %d points kink-free, %d used" % (key, idx.numel(), keep.numel(), P))
    assert idx.numel() >= P, (key, idx.numel())
    idx = idx[:P]
    return pos[idx].contiguous(), dirs[idx].contiguous(), tm[idx].contiguous()


def motion_points(w, P, lerp_mode):
    """P kink-free MotionNet points: gauss positions; integer frame ids for lerp mode -1 (the batch then does not lerp), the
    `times` set's mix of integer, fractional and negative times for the forced lerp."""
    g = torch.Generator().manual_seed(P + 7)
    n = P + P // 2
    pos = torch.randn((n, 3), generator=g) * 1.5
    if lerp_mode < 0:
        tm = torch.randint(0, 120, (n, 1), generator=g).float()
    else:
        tm = torch.where(torch.rand((n, 1), generator=g) < 0.5, torch.randint(-5, 120, (n, 1), generator=g).float(),
                         torch.rand((n, 1), generator=g) * 130.0 - 8.0)
    xyzt = torch.cat([pos, tm], 1)
    lerp = NF.lerp_of(tm, lerp_mode)
    w64 = NT._f64(w)
    keep = kink_free_chunked(lambda sl: NF.motion_forward(w64, _dev64(xyzt, sl), lerp), n)
    idx = keep.nonzero()[:, 0]
    assert idx.numel() >= P
    return xyzt[idx[:P]].contiguous(), lerp


def _proj(n, cols, seed):
    return torch.randn((n, cols), generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------------------------------------------------------------
# the three legs
# ---------------------------------------------------------------------------------------------------------------------
def native_space(w, pos, dirs, tm, prgb, psig, prec):
    """(gradients incl. d_pos, rgb, sigma) of the native SpaceNet for the loss sum(rgb * prgb) + sum(sigma * psig)"""
    net = TC.space_module(w, prec)
    p = pos.to(DEV).requires_grad_(True)
    rgb, sig = net(p, torch.cat([pos, dirs], 1).to(DEV), tm.to(DEV))
    ((rgb * prgb.to(DEV)).sum() + (sig * psig.to(DEV)).sum()).backward()
    out = {k: v.grad.detach().clone() for k, v in net.named_parameters()}
    out["pos"] = p.grad.detach()
    rgb, sig = rgb.detach(), sig.detach()
    del net, p
    _free()
    return out, rgb, sig


def oracle_space(w, pos, dirs, tm, prgb, psig, dtype, chunk):
    """The oracle's SpaceNet in dtype on the device, `chunk` points per call; parameter gradients accumulated across calls"""
    ww = {k: v.detach().to(DEV, dtype).clone().requires_grad_(True) for k, v in w.items()}
    dpos = []
    for s in range(0, pos.shape[0], chunk):
        sl = slice(s, s + chunk)
        p = pos[sl].to(DEV, dtype).requires_grad_(True)
        rgb, sig = O.spacenet_forward(ww, p, dirs[sl].to(DEV, dtype), tm[sl].to(DEV, dtype) if NF.uses_time(w) else None)
        ((rgb * prgb[sl].to(DEV, dtype)).sum() + (sig * psig[sl].to(DEV, dtype)).sum()).backward()
        dpos.append(p.grad.detach())
        del rgb, sig, p
    out = {k: v.grad.detach() for k, v in ww.items()}
    out["pos"] = torch.cat(dpos)
    del ww, dpos
    _free()
    return out


def native_motion(w, xyzt, pflow, lerp_mode, prec):
    net = TC.motion_module(w, prec)
    flow = net(xyzt.to(DEV), lerp_mode)
    (flow * pflow.to(DEV)).sum().backward()
    out = {k: v.grad.detach().clone() for k, v in net.named_parameters()}
    flow = flow.detach()
    del net
    _free()
    return out, flow


def oracle_motion(w, xyzt, pflow, lerp, dtype, chunk):
    ww = {k: v.detach().to(DEV, dtype).clone().requires_grad_(True) for k, v in w.items()}
    for s in range(0, xyzt.shape[0], chunk):
        sl = slice(s, s + chunk)
        (NF.motion_forward(ww, xyzt[sl].to(DEV, dtype), lerp) * pflow[sl].to(DEV, dtype)).sum().backward()
    out = {k: v.grad.detach() for k, v in ww.items()}
    del ww
    _free()
    return out


def yardstick_space(w, pos, dirs, tm, prgb, psig):
    with NoTF32():
        return oracle_space(w, pos, dirs, tm, prgb, psig, torch.float32, pos.shape[0])


def yardstick_motion(w, xyzt, pflow, lerp):
    with NoTF32():
        return oracle_motion(w, xyzt, pflow, lerp, torch.float32, xyzt.shape[0])


def within(nat, yard, factor):
    """test_gpu_nets_train.assert_within_twice's bar: (tensors over it, worst rms ratio, worst max ratio)"""
    bad = {k: (nat[k], yard[k]) for k in nat
           if nat[k][0] > factor * yard[k][0] + NT.ULP_FLOOR or nat[k][1] > factor * yard[k][1] + NT.ULP_FLOOR}
    return (bad, max(nat[k][0] / max(yard[k][0], 1e-12) for k in nat), max(nat[k][1] / max(yard[k][1], 1e-12) for k in nat))


def _check_all(results):
    """results: [(what, bad)]; fails with every case over its bar"""
    bad = [(what, b) for what, b in results if b]
    assert not bad, bad


def _space_cases():
    for tag in NF.WEIGHTS:
        for name in ("bkgd", "perf"):
            yield tag, name


def _space_weights(tag, name):
    sd = NF.state_dict(tag)
    if sd is None:
        pytest.skip("checkpoint copy not present (oracle/_ref/ckpt)")
    return NF.space_weights(O.split_state_dict(sd, 1), name)


# ---------------------------------------------------------------------------------------------------------------------
# 1. dense gradients against float64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["bkgd", "perf"])
@pytest.mark.parametrize("tag", NF.WEIGHTS)
@pytest.mark.parametrize("P", SPACE_P)
def test_spacenet_dense_gradients_against_float64(P, tag, name):
    w = _space_weights(tag, name)
    pos, dirs, tm = space_points(w, (tag, name, P), P)
    prgb, psig = _proj(P, 3, 1), _proj(P, 1, 2)
    truth = oracle_space(w, pos, dirs, tm, prgb, psig, torch.float64, CHUNK)
    yard = NT.grad_errors(yardstick_space(w, pos, dirs, tm, prgb, psig), truth)
    results = []
    for prec in PRECS:
        nat = NT.grad_errors(native_space(w, pos, dirs, tm, prgb, psig, prec)[0], truth)
        bad, rms, mx = within(nat, yard, FACTORS[prec][0])
        k = max(nat, key=lambda k: nat[k][1] / max(yard[k][1], 1e-12))
        print("P = %d %s %s/%s: worst ratio native / device fp32: rms %.2f, max %.2f (%s)" % (P, prec, tag, name, rms, mx, k))
        results.append(("%s P=%d %s/%s" % (prec, P, tag, name), bad))
    del truth
    _free()
    _check_all(results)


@pytest.mark.parametrize("lerp_mode", [-1, 1])
@pytest.mark.parametrize("tag", NF.WEIGHTS)
@pytest.mark.parametrize("P", MOTION_P)
def test_motionnet_dense_gradients_against_float64(P, tag, lerp_mode):
    w = NT._weights(tag)["motion"][0]
    xyzt, lerp = motion_points(w, P, lerp_mode)
    pflow = _proj(P, 3, 3)
    truth = oracle_motion(w, xyzt, pflow, lerp, torch.float64, CHUNK)
    yard = NT.grad_errors(yardstick_motion(w, xyzt, pflow, lerp), truth)
    results = []
    for prec in PRECS:
        nat = NT.grad_errors(native_motion(w, xyzt, pflow, lerp_mode, prec)[0], truth)
        bad, rms, mx = within(nat, yard, FACTORS[prec][0])
        print("P = %d %s motion %s lerp %d: worst ratio native / device fp32: rms %.2f, max %.2f" % (P, prec, tag, lerp_mode,
                                                                                                   rms, mx))
        results.append(("%s P=%d %s lerp %d" % (prec, P, tag, lerp_mode), bad))
    _check_all(results)


# ---------------------------------------------------------------------------------------------------------------------
# 2. sparse-upstream probes
# ---------------------------------------------------------------------------------------------------------------------
def probes(P, rows=None):
    """Sorted probe indices: the first, second and last point of every weight-gradient chunk, both sides of a few 64- and
    128-point tile edges, P - 2 and P - 1, and for saved rows `rows` the first point of each row r whose offset r * P + p is
    past 2^30 or 2^31 elements, with its neighbour before."""
    ch = grad_chunk(P)
    idx = set()
    for z in range(-(-P // ch)):
        a, b = z * ch, min((z + 1) * ch, P)
        idx.update((a, a + 1, b - 1))
    for e in (64, 128, 64 * 3, 128 * 5, (P // 3) // 64 * 64, (P // 2) // 128 * 128, (P - 1) // 128 * 128):
        idx.update((e - 1, e))
    idx.update((P - 2, P - 1))
    if rows:
        for lim in (1 << 30, 1 << 31):
            r = lim // P
            if r < rows:
                p = lim - r * P
                idx.update((p - 1, p) if p > 0 else (p,))
    return torch.tensor(sorted(i for i in idx if 0 <= i < P))


def _sparse(proj, idx):
    out = torch.zeros_like(proj)
    out[idx] = proj[idx]
    return out


@pytest.mark.parametrize("tag", ["syn_t", "syn"])
@pytest.mark.parametrize("P", SPACE_P)
def test_spacenet_probe_gradients(P, tag):
    """Upstream gradients on the probes only: parameter gradients against float64 of the probes alone, d_pos exactly zero
    off the probes, the probes' outputs and d_pos bit for bit those of the probes as a batch of their own."""
    results = []
    for name in ("bkgd", "perf"):
        w = _space_weights(tag, name)
        pos, dirs, tm = space_points(w, (tag, name, P), P)
        rows = saved_rows(NF.uses_time(w))
        idx = probes(P, rows)
        crossing = [r for r in range(rows) if r * P < (1 << 31) < (r + 1) * P]
        prgb, psig = _proj(P, 3, 11), _proj(P, 1, 12)
        sub = (pos[idx], dirs[idx], tm[idx], prgb[idx], psig[idx])
        truth = oracle_space(w, *sub, torch.float64, CHUNK)
        yard = NT.grad_errors(yardstick_space(w, *sub), truth)
        off = torch.ones(P, dtype=torch.bool)
        off[idx] = False
        for prec in PRECS:
            got, rgb, sig = native_space(w, pos, dirs, tm, _sparse(prgb, idx), _sparse(psig, idx), prec)
            dpos = got["pos"]
            assert float(dpos[off.to(DEV)].abs().max()) == 0.0, (prec, P, tag, name, "d_pos off the probes")
            rgb, sig, dpos = rgb[idx.to(DEV)], sig[idx.to(DEV)], dpos[idx.to(DEV)]
            got["pos"] = dpos
            nat = NT.grad_errors(got, truth)
            del got
            own, rgb1, sig1 = native_space(w, *sub, prec)
            what = "%s P=%d %s/%s (%d probes, saved row crossing 2^31: %s)" % (prec, P, tag, name, idx.numel(), crossing)
            assert NT._same(rgb, rgb1) and NT._same(sig, sig1), (what, "outputs")
            assert NT._same(dpos, own["pos"]), (what, "d_pos")
            bad, rms, mx = within(nat, yard, FACTORS[prec][0])
            print("%s: worst ratio native / device fp32: rms %.2f, max %.2f" % (what, rms, mx))
            results.append((what, bad))
            del rgb, sig, dpos
            _free()
    _check_all(results)


@pytest.mark.parametrize("P", MOTION_P)
def test_motionnet_probe_gradients(P):
    results = []
    w = NT._weights("syn_t")["motion"][0]
    for lerp_mode in (-1, 1):
        xyzt, lerp = motion_points(w, P, lerp_mode)
        idx = probes(P)
        pflow = _proj(P, 3, 13)
        truth = oracle_motion(w, xyzt[idx], pflow[idx], lerp, torch.float64, CHUNK)
        yard = NT.grad_errors(yardstick_motion(w, xyzt[idx], pflow[idx], lerp), truth)
        for prec in PRECS:
            got, flow = native_motion(w, xyzt, _sparse(pflow, idx), lerp_mode, prec)
            _, flow1 = native_motion(w, xyzt[idx], pflow[idx], lerp_mode, prec)
            what = "motion %s P=%d lerp %d (%d probes)" % (prec, P, lerp_mode, idx.numel())
            assert NT._same(flow[idx.to(DEV)], flow1), (what, "flow")
            bad, rms, mx = within(NT.grad_errors(got, truth), yard, FACTORS[prec][0])
            print("%s: worst ratio native / device fp32: rms %.2f, max %.2f" % (what, rms, mx))
            results.append((what, bad))
    _check_all(results)


def test_probe_placement():
    """The probes sit where the test says they do."""
    P = SPACE_P[-1]
    ch = grad_chunk(P)
    assert P % 16 and P % 128 and P % ch and -(-P // ch) == MAX_SPLIT
    for use_time in (False, True):
        rows = saved_rows(use_time)
        assert (rows - 1) * P + P - 1 >= 1 << 31
        idx = set(probes(P, rows).tolist())
        r = (1 << 31) // P
        assert (1 << 31) - r * P in idx and (1 << 31) - r * P - 1 in idx
        assert {0, 1, ch - 1, ch, ch + 1, P - 2, P - 1} <= idx and 300 <= len(idx) <= 500
    assert grad_chunk(CAP - 1) == MIN_CHUNK and grad_chunk(CAP + 1) == MIN_CHUNK + TK       # either side of the cap
    assert saved_rows(True) == 2031 and saved_rows(False) == 2010


# ---------------------------------------------------------------------------------------------------------------------
# 3. a full training step at the taekwondo batch
# ---------------------------------------------------------------------------------------------------------------------
# scripts/bench_train_step.py's workload: synthetic weights of the shipped shapes, no edits
TKD_BATCH = dict(weights="synthetic", seed=3, L=2, space_time=True, n1=90, n2=30, seven=True, mixed_frames=(3, 60),
                 frame_ids=[10, 10, 10], thr=(1e-4, 0.0), n_rays=2000, ray_seed=31)


# A known defect of tf32x3, held apart from the other tensors of its step: the coarse background SpaceNet's density bias
# gradient, the sum of d_sigma over that call's 153 524 kept points, misses float64 by 10.1x the fp32 yardstick's error
# (bar 4x).  The tf32x3 forward's sigma errors there are biased: their mean is -0.54x their rms (fp32 native +0.01x, torch
# fp32 +0.03x), so they add up coherently through the compositing backward instead of averaging out.  Every other tensor of
# the step is asserted at its bar.  This one must stay under KNOWN_CEILING x the yardstick, and the test fails once it meets
# its bar, so that the exception is removed with the defect.
KNOWN = {"tf32x3": ("bkgd_spacenet.density_net.0.bias",)}
KNOWN_CEILING = 15.0


@pytest.mark.parametrize("only_coarse", [False, True], ids=["fine", "only_coarse"])
@pytest.mark.parametrize("prec", PRECS)
def test_training_step_at_the_taekwondo_batch(prec, only_coarse):
    case = dict(TKD_BATCH, only_coarse=only_coarse)
    known = TF.float64_step_check(case, TG.case_inputs(case), prec, *FACTORS[prec], known=KNOWN.get(prec, ()))
    over = {}
    for k, (nat, yard, f) in known.items():
        ratio = max(nat[i] / max(yard[i], 1e-12) for i in (0, 1))
        print("%s known: %s ratio %.2f (native %.3g / %.3g, yardstick %.3g / %.3g)" % (prec, k, ratio, *nat, *yard))
        assert nat[0] <= KNOWN_CEILING * yard[0] and nat[1] <= KNOWN_CEILING * yard[1], (k, nat, yard)
        if nat[0] > f * yard[0] + NT.ULP_FLOOR or nat[1] > f * yard[1] + NT.ULP_FLOOR:
            over[k] = ratio
    assert set(over) == set(known), ("now within its bar: drop it from KNOWN", set(known) - set(over))
    if over:
        pytest.xfail("tf32x3 sigma bias: %s" % over)
