"""The trainable LayeredRFRender (stnerf_b200.train) on the device.

Values: under grad, in fp32 mode with injected uniforms, the 5-tuple equals LayeredRFRender.forward's (fp32) on every golden
case whose weights are present, and meets test_gpu_render's tolerances against the reference's goldens; without injection a
grad and a no-grad forward with the same seed give the same images.
Gradients: on the cases of the reference golden (tests/golden/train_grads.npz: a 7-column mixed-frame batch with per-ray
boxes and edits; retiming rays with fractional frame ids, thresholds, a scale / shift edit with a None shift entry, alpha, a
near plane and a hidden layer; an only_coarse batch), the trainer's loss with its `scalar` rule, every parameter gradient within
2x (3x through a MotionNet) of the larger fp32 torch error against float64 -- the float64 restatement pinned to the reference
there.  On the two-layer chain of test_gpu_composite_grad the model's gradients also equal the chain's bit for bit; that chain
adds its mask losses unconditionally (no `scalar` rule), and so does `_chain_loss` here.  Identical calls give bit-identical gradients, with injected and with Philox uniforms,
on a batch whose hit lists cross compaction blocks.
Training: Adam steps against the torch fp32 restatement (on that chain case: one performer, 64 + 128 samples, 192 rays, lr
4e-4 -- not the full taekwondo batch, which scripts/bench_train_step.py times), one step under anomaly detection, the optimiser sees every parameter.
Round trip: after a step the no-grad render uses the new weights, bit-identical to a fresh LayeredRFRender loaded with them,
and a checkpoint saved as the trainer saves it loads through checkpoint_io.
Edges: a performer with no hit ray, a hidden performer, N = 2, 90 + 30 samples, CPU rays, a bad ray width.
"""
import numpy as np
import pytest
import torch

import cases as C
import test_gpu_composite_grad as CG
import test_gpu_nets_train as NT
from oracle import stnerf_oracle as O
from tests_support import make_cfg

pytestmark = pytest.mark.gpu

DEV = "cuda"
VALUE_TOL = 1e-5               # grad forward vs LayeredRFRender.forward, fp32 mode (measured: see the printed differences)
ADAM_STEPS = 30
ADAM_LR = 4e-4                 # configs/config_taekwondo.yml SOLVER.BASE_LR
ADAM_REL_TOL = 1e-3


def _model(case, precision="fp32", trainable=True, sd=None, train_precision=None):
    import modeling
    cfg = make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], precision)
    cfg.MODEL.B200_TRAINABLE = trainable
    if train_precision is not None:
        cfg.MODEL.B200_TRAIN_PRECISION = train_precision
    model = modeling.build_layered_model(cfg, 0, case.get("scale"), case.get("shift"))
    sd = C.state_dict_for(case) if sd is None else sd
    if sd is None:
        return None
    model.load_state_dict(sd)
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model.near = case.get("near", 0.0)
    model.alpha = case.get("alpha", 1.0)
    for i in case.get("hidden", []):
        model.hide_layer(i)
    return model.cuda()


def _run(model, case, rays=None, uniforms=None, inject=True, seed=None, grad=True):
    rays = (C.rays_for(case) if rays is None else rays).to(DEV)
    if inject:
        jit, u = C.uniforms_for(case) if uniforms is None else uniforms
        model.inject_uniforms(jit.to(DEV).contiguous(), None if u is None else u.to(DEV).contiguous())
    if seed is not None:
        model.seed = seed
    with torch.set_grad_enabled(grad):
        return model(rays, torch.zeros(rays.shape[0], device=DEV), None, only_coarse=case.get("only_coarse", False),
                     density_threshold=case["thr"][0], bkgd_density_threshold=case["thr"][1])


def _max_diff(a, b):
    fa, fb = C.flatten_outputs(*a), C.flatten_outputs(*b)
    worst = 0.0
    for k in fb:
        if k.startswith("ray_mask"):
            assert np.array_equal(fa[k], fb[k]), k
        else:
            worst = max(worst, float(np.abs(fa[k].astype(np.float64) - fb[k]).max()))
    return worst


def _grads(model):
    return {k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)) for k, p in model.named_parameters()}


def _bits_equal(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


# ---------------------------------------------------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(C.CASES))
def test_grad_forward_equals_render_fp32(name):
    case = C.CASES[name]
    trainable = _model(case)
    if trainable is None:
        pytest.skip("checkpoint for %s not present" % name)
    plain = _model(case, trainable=False)
    got = _run(trainable, case)
    assert got[0][0].requires_grad and got[1][0].requires_grad
    want = _run(plain, case, grad=False)
    worst = _max_diff(got, want)
    print("%s: grad forward vs LayeredRFRender.forward (fp32): max |diff| %.3g" % (name, worst))
    assert worst <= VALUE_TOL, worst
    gold = C.load_golden(name)
    if gold is not None:                                   # test_gpu_render's tolerances against the reference
        flat = C.flatten_outputs(*got)
        for k in gold:
            if k.startswith("ray_mask"):
                assert np.array_equal(flat[k], gold[k]), k
            elif k.endswith("rgb") or k.endswith("acc"):
                assert float(np.abs(flat[k].astype(np.float64) - gold[k]).max()) <= 1e-3, k
            elif k.endswith("depth"):
                assert (np.abs(flat[k].astype(np.float64) - gold[k]) <= 2e-2 + 2e-3 * np.abs(gold[k])).all(), k


def test_philox_grad_and_nograd_forwards_place_the_same_samples():
    case = C.CASES["syn_L2_64_128"]
    model = _model(case)
    got = _run(model, case, inject=False, seed=41)
    want = _run(model, case, inject=False, seed=41, grad=False)
    worst = _max_diff(got, want)
    print("philox: grad vs no-grad forward, same seed: max |diff| %.3g" % worst)
    assert worst <= VALUE_TOL, worst
    other = _run(model, case, inject=False, seed=42, grad=False)
    assert _max_diff(other, want) > 0                      # the seed does select the draws


# ---------------------------------------------------------------------------------------------------------------------
# gradients: the training chain of test_gpu_composite_grad (held to float64 there) through the model
# ---------------------------------------------------------------------------------------------------------------------
def _chain_loss(out, labels, target):
    """run_chain's loss (layered_trainer.py:216-281 with the mask losses always on) from the 5-tuple."""
    fine_mixed, coarse_mixed, fine_layer, coarse_layer, _ = out
    loss = torch.nn.functional.mse_loss(coarse_mixed[0], target) + torch.nn.functional.mse_loss(fine_mixed[0], target)
    for stage in (coarse_layer, fine_layer):
        outl = torch.cat([stage[i][2][labels == 0] for i in range(1, len(stage))], 0)
        inl = torch.cat([stage[i][2][labels == i] for i in range(len(stage))], 0)
        loss = loss + (outl.abs().sum() + (1 - inl).abs().sum()) / CG.MASK_SCALAR
    return loss


def _chain_model():
    model0, rays, jit, u, samp, labels, target = CG.chain_inputs()
    model = _model(CG.CHAIN_CASE, sd=model0.state_dict())
    return model, model0, rays, jit, u, samp, labels, target


def _model_step(model, rays, jit, u, labels, target):
    model.zero_grad(set_to_none=True)
    model.inject_uniforms(jit, u)
    out = model(rays, labels, None, False)
    loss = _chain_loss(out, labels, target)
    loss.backward()
    return loss, out


def test_gradients_equal_the_native_training_chain():
    model, model0, rays, jit, u, samp, labels, target = _chain_model()
    loss, _ = _model_step(model, rays, jit, u, labels, target)
    got = _grads(model)
    nets = CG.NativeNets(model0)
    chain_loss = CG.run_chain(nets, rays, samp, u, labels, target, torch.float32, DEV, CG._native_comp, CG._native_merged)
    chain_loss.backward()
    want = _grads(nets.d)
    assert set(got) == set(want)
    used = [k for k in want if float(want[k].abs().max()) > 0]
    assert any(k.startswith("time_deform_nets") for k in used) and any(k.startswith("bkgd_spacenet_fine") for k in used)
    worst = max(float((got[k] - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30)) for k in used)
    print("model vs native chain: loss %.9g / %.9g, worst relative gradient difference %.3g" % (float(loss), float(chain_loss), worst))
    assert abs(float(loss) - float(chain_loss)) <= 1e-6 * abs(float(chain_loss))
    assert worst <= 1e-5, worst
    for k in want:
        if k not in used:
            assert float(got[k].abs().max()) == 0.0, k


def test_identical_calls_give_identical_gradients():
    # three quarters of rays_for's rays are aimed at the performer boxes, alternating layers: > 256 hit rays per layer
    case = dict(C.CASES["syn_L2_64_128"], n_rays=1600, ray_seed=77, n2=64, thr=(1e-4, 0.0))
    model = _model(case, sd=O.synthetic_state_dict(2, True, seed=23))
    rays = C.rays_for(case).to(DEV)
    jit, u = (x.to(DEV).contiguous() for x in C.uniforms_for(case))
    for inject in (True, False):
        grads, hits = [], None
        for _ in range(2):
            model.zero_grad(set_to_none=True)
            if inject:
                model.inject_uniforms(jit, u)
            model.seed = 7
            out = model(rays, None, None, False, density_threshold=case["thr"][0])
            (out[0][0].square().sum() + out[1][0].sum() + sum(o[2].sum() for o in out[2])).backward()
            grads.append(_grads(model))
            hits = [int(m.sum()) for m in out[4]]
        print("determinism (inject=%s): hit rays per layer %s" % (inject, hits))
        assert min(hits[1:]) > 256                       # the ordered compaction spans several blocks
        assert _bits_equal(grads[0], grads[1])


# ---------------------------------------------------------------------------------------------------------------------
# training loop
# ---------------------------------------------------------------------------------------------------------------------
def test_adam_steps_follow_the_torch_restatement():
    torch.backends.cuda.matmul.allow_tf32 = False
    model, model0, rays, jit, u, samp, labels, target = _chain_model()
    opt = torch.optim.Adam(model.parameters(), lr=ADAM_LR)
    assert sum(len(g["params"]) for g in opt.param_groups) == len(model0.state_dict())
    nat = []
    for step in range(ADAM_STEPS):
        opt.zero_grad()
        with torch.autograd.set_detect_anomaly(step == 0):
            loss, _ = _model_step(model, rays, jit, u, labels, target)
        opt.step()
        nat.append(float(loss))
    ref_nets = CG.RefNets(model0, DEV, torch.float32)
    ropt = torch.optim.Adam(list(ref_nets.params().values()), lr=ADAM_LR)
    ref = []
    for _ in range(ADAM_STEPS):
        ropt.zero_grad()
        loss = CG.run_chain(ref_nets, rays, samp, u, labels, target, torch.float32, DEV, CG._ref_comp, CG._ref_merged)
        loss.backward()
        ropt.step()
        ref.append(float(loss))
    gap = abs(nat[-1] - ref[-1]) / ref[-1]
    print("adam: loss %.6g -> %.6g native model, %.6g -> %.6g torch fp32, relative gap %.3g" % (nat[0], nat[-1], ref[0], ref[-1], gap))
    assert nat[-1] < 0.9 * nat[0]
    assert gap < ADAM_REL_TOL, gap


# ---------------------------------------------------------------------------------------------------------------------
# round trip
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "exact"])
def test_no_grad_render_uses_the_trained_weights(precision, tmp_path):
    from stnerf_b200 import checkpoint_io
    case = C.CASES["syn_L2_64_128"]
    model = _model(case, precision=precision)
    before = _run(model, case, grad=False)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    out = _run(model, case)
    (out[0][0].sum() + out[1][2].sum()).backward()
    opt.step()
    after = _run(model, case, grad=False)
    fresh = _model(case, precision=precision, trainable=False, sd=model.state_dict())
    want = _run(fresh, case, grad=False)
    assert _max_diff(after, want) == 0.0
    assert _max_diff(after, before) > 0.0
    path = tmp_path / "layered_rfnr_checkpoint_1.pt"
    torch.save({"model": model.state_dict()}, str(path))            # engine/layered_trainer.py:347 (ModelCheckpoint)
    loaded = _model(case, precision=precision, trainable=False)
    assert checkpoint_io.load_checkpoint(loaded, str(path)) == []
    assert _max_diff(_run(loaded, case, grad=False), want) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------
def _equal_to_render(case, rays=None, uniforms=None, what=""):
    trainable, plain = _model(case), _model(case, trainable=False)
    got = _run(trainable, case, rays=rays, uniforms=uniforms)
    (got[0][0].sum() + got[1][0].sum()).backward()
    for k, p in trainable.named_parameters():
        assert p.grad is None or bool(torch.isfinite(p.grad).all()), (what, k)
    worst = _max_diff(got, _run(plain, case, rays=rays, uniforms=uniforms, grad=False))
    print("%s: max |diff| %.3g" % (what, worst))
    assert worst <= VALUE_TOL, (what, worst)
    return trainable, got


def test_performer_without_hit_rays():
    case = C.CASES["syn_L2_64_128"]
    rays = C.rays_for(case)
    jit, u = C.uniforms_for(case)
    miss = torch.arange(4)                                 # the four image corners miss every performer
    trainable, got = _equal_to_render(case, rays[miss], (jit[:, miss].contiguous(), u[:, miss].contiguous()), "no hit ray")
    assert all(int(m.sum()) == 0 for m in got[4][1:])
    assert all(trainable.spacenets[i].stage1[0].weight.grad is None for i in range(2))


def test_hidden_performer():
    case = dict(C.CASES["syn_L2_64_128"], hidden=[1])
    trainable, _ = _equal_to_render(case, what="hidden performer")
    assert trainable.spacenets[0].stage1[0].weight.grad is None
    assert trainable.spacenets[1].stage1[0].weight.grad is not None


def test_two_rays_and_90_30_samples():
    case = C.CASES["syn_L2_64_128"]
    rays = C.rays_for(case)
    jit, u = C.uniforms_for(case)
    pick = torch.tensor([50, 120])
    _equal_to_render(case, rays[pick], (jit[:, pick].contiguous(), u[:, pick].contiguous()), "N = 2")
    case = dict(C.CASES["syn_L2_64_128"], n1=90, n2=30, thr=(1e-4, 0.0))
    _equal_to_render(case, what="90 + 30")


def test_only_coarse_and_edits():
    _equal_to_render(C.CASES["syn_L1_coarse"], what="only_coarse")
    case = dict(C.CASES["syn_L2_64_128"], shift=[[0, 0, 0], [0, 0.3, 0], None], scale=[1, 0.8, 1.2], alpha=0.5, near=0.5,
                thr=(1e-4, 0.0))
    _equal_to_render(case, what="edits with a None shift entry")


def test_bad_inputs_and_the_plain_model():
    from stnerf_b200 import _lib as L
    case = C.CASES["syn_L2_64_128"]
    model = _model(case)
    rays = C.rays_for(case)
    with pytest.raises(L.StnerfError):
        model(rays, None, None)
    with pytest.raises(ValueError):
        model(rays[:, :8].to(DEV), None, None)
    plain = _model(case, trainable=False)
    assert len(list(plain.parameters())) == 0
    out = _run(plain, case)
    assert not any(t.requires_grad for t in out[0] + out[1])


# ---------------------------------------------------------------------------------------------------------------------
# gradients against float64 on the cases of the reference golden (tests/golden/train_grads.npz): the trainer's loss, the
# method of test_gpu_composite_grad's training chain -- points near a ReLU kink set aside in every run, the fine depths fixed
# to the native run's, each SpaceNet of the float64 truth evaluated at the fp32 run's own deformed points (flow_at)
# ---------------------------------------------------------------------------------------------------------------------
import make_golden_train_grads as TG  # noqa: E402
import train_restatement as TR  # noqa: E402


def _native_trace(model, keep=None):
    rec = {}

    def trace(name, x):
        if name in ("t_coarse", "mask") or name.startswith("t_fine."):
            rec[name] = x.detach().clone()
            return None
        kind, call = name.split(".")
        rec[name] = x.detach().clone()
        if kind == "flow":
            call = "m" + call
        if keep is not None and call in keep:
            return torch.where(keep[call].to(x.device)[:, None] if x.dim() > 1 else keep[call].to(x.device), x, x.detach())
        return None
    model.trace = trace
    return rec


def float64_step_check(case, inputs, train_precision="fp32", factor=2.0, chained_factor=NT.CHAINED_FACTOR, known=()):
    """One training step of the trainable model on `case` (a case dict of make_golden_train_grads' form) with
    inputs = make_golden_train_grads.case_inputs(case), native networks in `train_precision`: every parameter gradient
    within `factor` (chained_factor through a MotionNet) of the larger torch fp32 error against float64, CPU or device.
    Also printed: each SpaceNet call's sigma error, rms and mean over its kept points relative to the float64 sigma's rms.
    Parameters named in `known` are left out of the assertion; their (native, yardstick) errors and bar are returned."""
    flag = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return _float64_step_check(case, inputs, train_precision, factor, chained_factor, known)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = flag


def _outputs_of(rec):
    """the native run's SpaceNet outputs per call, from its trace"""
    return {k[4:]: (v, rec["sigma." + k[4:]]) for k, v in rec.items() if k.startswith("rgb.")}


def _sigma_errors(got, truth, keep):
    """per SpaceNet call over its kept points: (rms, mean) of sigma - float64 sigma, relative to the float64 sigma's rms"""
    out = {}
    for k, (_, s64) in truth.items():
        if k not in got:
            continue
        m = keep[k].to(s64.device)
        t = s64.reshape(-1)[m]
        e = got[k][1].reshape(-1).to(t.device, torch.float64)[m] - t
        den = float(t.pow(2).mean().sqrt()) or 1.0
        out[k] = "%.2g/%+.2g" % (float(e.pow(2).mean().sqrt()) / den, float(e.mean()) / den)
    return out


def _float64_step_check(case, inputs, train_precision, factor, chained_factor, known):
    rays, jit, u, labels, target, sd = inputs
    only_coarse, l = bool(case.get("only_coarse", False)), case["L"] + 1
    model = _model(case, sd=sd, train_precision=train_precision)
    assert all(m.train_precision == train_precision for m in model.modules() if hasattr(m, "train_precision"))
    name = "%s %s %d rays" % (train_precision, "only_coarse" if only_coarse else "fine", rays.shape[0])
    lab, tgt = labels.to(DEV), target.to(DEV)

    def native(keep):
        model.zero_grad(set_to_none=True)
        rec = _native_trace(model, keep)
        model.inject_uniforms(jit.to(DEV).contiguous(), None if u is None else u.to(DEV).contiguous())
        out = model(rays.to(DEV), lab, None, only_coarse, density_threshold=case["thr"][0], bkgd_density_threshold=case["thr"][1])
        TG.trainer_loss(out, lab, tgt, only_coarse, rays.shape[0]).backward()
        model.trace = None
        return _grads(model), rec

    _, rec = native(None)
    samples = (rec["t_coarse"], rec["mask"])
    fine_t = None if only_coarse else [rec["t_fine.%d" % i] for i in range(l)]
    sc = C.scene_for(case)

    def restated(dtype, device, keep=None, flow_at=None, kinks=None):
        p = {k: v.to(device, dtype).clone().requires_grad_(True) for k, v in sd.items()}
        r = {}
        out = TR.forward(p, sc, rays, case["n1"], case["n2"], jit, u, only_coarse, case["thr"][0], case["thr"][1],
                         bool(case.get("seven")), dtype, device, samples=samples, fine_t=fine_t, keep=keep, flow_at=flow_at,
                         kinks=kinks, record=r)
        if kinks is not None:
            return None, None
        TG.trainer_loss(out, labels.to(device), target.to(device, dtype), only_coarse, rays.shape[0]).backward()
        return {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}, r

    keep = {}
    with torch.no_grad():
        restated(torch.float64, DEV, kinks=keep)
    print("%s: kept points per call %s" % (name, {k: "%d/%d" % (int(v.sum()), v.numel()) for k, v in keep.items()}))
    nat, rec = native(keep)
    flows_nat = {k[5:]: v for k, v in rec.items() if k.startswith("flow.")}
    cpu, rec_cpu = restated(torch.float32, "cpu", keep)
    gpu, rec_gpu = restated(torch.float32, DEV, keep)
    truths = [restated(torch.float64, DEV, keep, flow_at=f) for f in (flows_nat, rec_cpu["flows"], rec_gpu["flows"])]
    print("%s: sigma error rms/mean per call, native %s, device fp32 %s"
          % (name, _sigma_errors(_outputs_of(rec), truths[0][1]["outputs"], keep),
             _sigma_errors(rec_gpu["outputs"], truths[2][1]["outputs"], keep)))
    truths = [t[0] for t in truths]
    used = [k for k in truths[0] if float(truths[0][k].abs().max()) > 0]
    assert used
    out = {}
    for group, f in (([k for k in used if not k.startswith("time_deform_nets")], factor),
                     ([k for k in used if k.startswith("time_deform_nets")], chained_factor)):
        if not group:
            continue
        e_nat = NT.grad_errors({k: nat[k] for k in group}, {k: truths[0][k] for k in group})
        e_cpu = NT.grad_errors({k: cpu[k] for k in group}, {k: truths[1][k] for k in group})
        e_gpu = NT.grad_errors({k: gpu[k] for k in group}, {k: truths[2][k] for k in group})
        yard = CG.yardstick(e_cpu, e_gpu)
        out.update({k: (e_nat[k], yard[k], f) for k in group if k in known})
        NT.assert_within_twice({k: v for k, v in e_nat.items() if k not in known}, yard, "%s (%d tensors)" % (name, len(group)), f)
    for k in nat:
        if k not in used:
            assert float(nat[k].abs().max()) == 0.0, k
    return out


@pytest.mark.parametrize("name", list(TG.CASES))
def test_gradients_against_float64_on_the_reference_cases(name):
    float64_step_check(TG.CASES[name], TG.case_inputs(name))
