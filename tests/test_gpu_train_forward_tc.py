"""The trainable LayeredRFRender with train_precision="tf32x3" on the device.

Gradients on the cases of the reference golden (tests/golden/train_grads.npz) against float64, by the method of
test_gpu_train_forward.py: within 4x the fp32 torch yardstick (6x through a MotionNet).  Identical calls give identical
gradient bits.  Adam steps on the two-layer chain stay as close to the torch fp32 restatement as 4x the fp32 native path's own
distance.  The no-grad render after training uses the trained weights, and the default model still trains in fp32.
"""
import pytest
import torch

import cases as C
import test_gpu_composite_grad as CG
import test_gpu_train_forward as TF
import make_golden_train_grads as TG
from tests_support import make_cfg

pytestmark = pytest.mark.gpu

DEV = "cuda"
FACTOR, CHAINED_FACTOR = 4.0, 6.0
ADAM_FACTOR = 4.0


def _model(case, train_precision="tf32x3", sd=None, set_knob=True):
    import modeling
    cfg = make_cfg(case["L"], case["n1"], case["n2"], case["space_time"], "fp32")
    cfg.MODEL.B200_TRAINABLE = True
    if set_knob:
        cfg.MODEL.B200_TRAIN_PRECISION = train_precision
    model = modeling.build_layered_model(cfg, 0, case.get("scale"), case.get("shift"))
    model.load_state_dict(C.state_dict_for(case) if sd is None else sd)
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    model.near = case.get("near", 0.0)
    model.alpha = case.get("alpha", 1.0)
    for i in case.get("hidden", []):
        model.hide_layer(i)
    return model.cuda()


@pytest.mark.parametrize("name", list(TG.CASES))
def test_gradients_against_float64_on_the_reference_cases(name):
    TF.float64_step_check(TG.CASES[name], TG.case_inputs(name), "tf32x3", FACTOR, CHAINED_FACTOR)


def test_identical_calls_give_identical_gradients():
    model, model0, rays, jit, u, samp, labels, target = _chain()
    grads = []
    for _ in range(2):
        TF._model_step(model, rays, jit, u, labels, target)
        grads.append(TF._grads(model))
    assert TF._bits_equal(grads[0], grads[1])


def _chain(train_precision="tf32x3"):
    model0, rays, jit, u, samp, labels, target = CG.chain_inputs()
    model = _model(CG.CHAIN_CASE, train_precision, sd=model0.state_dict())
    return model, model0, rays, jit, u, samp, labels, target


def _params_distance(a, b, start):
    num = sum(float((a[k].double() - b[k].double()).pow(2).sum()) for k in b)
    den = sum(float((b[k].double() - start[k].double()).pow(2).sum()) for k in b)
    return (num / den) ** 0.5


def test_adam_steps_follow_the_torch_restatement():
    """30 Adam steps: the parameters' distance from the torch fp32 restatement's, relative to how far that moved, is at most
    4x the fp32 native path's own distance."""
    torch.backends.cuda.matmul.allow_tf32 = False
    model0, rays, jit, u, samp, labels, target = CG.chain_inputs()
    start = {k: v.detach().to(DEV).clone() for k, v in model0.state_dict().items()}
    ref_nets = CG.RefNets(model0, DEV, torch.float32)
    ropt = torch.optim.Adam(list(ref_nets.params().values()), lr=TF.ADAM_LR)
    for _ in range(TF.ADAM_STEPS):
        ropt.zero_grad()
        CG.run_chain(ref_nets, rays, samp, u, labels, target, torch.float32, DEV, CG._ref_comp, CG._ref_merged).backward()
        ropt.step()
    ref = {k: v.detach() for k, v in ref_nets.params().items()}
    dist, losses, trained = {}, {}, {}
    for tp in ("fp32", "tf32x3"):
        model = _model(CG.CHAIN_CASE, tp, sd=model0.state_dict())
        opt = torch.optim.Adam(model.parameters(), lr=TF.ADAM_LR)
        first = None
        for _ in range(TF.ADAM_STEPS):
            opt.zero_grad()
            loss, _ = TF._model_step(model, rays, jit, u, labels, target)
            opt.step()
            first = float(loss) if first is None else first
        losses[tp] = (first, float(loss))
        dist[tp] = _params_distance(dict(model.named_parameters()), ref, start)
        trained[tp] = model
    print("adam: relative parameter distance from the torch fp32 restatement: fp32 %.3g, tf32x3 %.3g (ratio %.2f); "
          "losses fp32 %.6g -> %.6g, tf32x3 %.6g -> %.6g" % (dist["fp32"], dist["tf32x3"], dist["tf32x3"] / dist["fp32"],
                                                             *losses["fp32"], *losses["tf32x3"]))
    assert losses["tf32x3"][1] < 0.9 * losses["tf32x3"][0]
    assert dist["tf32x3"] <= ADAM_FACTOR * dist["fp32"], dist

    # the no-grad render of the trained model is a fresh LayeredRFRender's with the trained weights
    model = trained["tf32x3"]
    case = dict(CG.CHAIN_CASE)
    jit_c, u_c = jit.contiguous(), u.contiguous()
    with torch.no_grad():
        model.inject_uniforms(jit_c, u_c)
        after = model(rays, None, None, False)
        fresh = TF._model(case, precision="fp32", trainable=False, sd=model.state_dict())
        fresh.inject_uniforms(jit_c, u_c)
        want = fresh(rays, None, None, False)
    assert TF._max_diff(after, want) == 0.0


def test_default_model_trains_in_fp32():
    """No knob: fp32 training, bit-identical gradients to B200_TRAIN_PRECISION="fp32"."""
    model0, rays, jit, u, samp, labels, target = CG.chain_inputs()
    grads = []
    for set_knob in (False, True):
        model = _model(CG.CHAIN_CASE, "fp32", sd=model0.state_dict(), set_knob=set_knob)
        assert all(m.train_precision == "fp32" for m in model.modules() if hasattr(m, "train_precision"))
        TF._model_step(model, rays, jit, u, labels, target)
        grads.append(TF._grads(model))
    assert TF._bits_equal(grads[0], grads[1])
