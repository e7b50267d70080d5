"""-m gpu parity tests of the IoUNet row (SURVEY.md 8(f).1): the IoU feature branch of the network plan, `predict_iou` with its
analytic box gradient, and the on-device refinement loops -- against outputs of the UNMODIFIED reference modules on the same seeded
weights and inputs (PyTorch-CPU autograd, the oracle's PrRoIPool restatement; tests/golden/iou_tomp_ref.npz, recorded by
oracle/gen_iou_tomp_golden.py).  The plug-in seam test runs the reference's own autograd code above the engine and needs a reference
checkout."""
import numpy as np
import pytest
import torch

from ref_weights import GOLDEN, iou_inputs, iou_state_dict

pytestmark = pytest.mark.gpu


def _gold():
    return np.load(GOLDEN)


def _ref_net():
    """The unmodified reference DiMP-50 network with the golden's weights (for the plug-in seam test only)."""
    from baseline import ref_env
    if not ref_env.reference_available():
        pytest.skip("reference tree not staged (baseline/_ref)")
    from oracle import ref_shims
    ref_shims.install()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from baseline import ref_tracker
    net = ref_tracker.build_dimp_net("resnet50", seed=0)
    net.load_state_dict(iou_state_dict(_gold()), strict=False)
    return net.eval()


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _rel_elem(a, b, floor):
    """element-wise relative error, with the denominator floored at `floor` x the largest reference magnitude"""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=floor * b.abs().max())).max())


def _sampled_rel(mine, gold, name, floor=None):
    """Relative error of `mine` at the golden's sampled indices: against the full reference maximum, or element-wise with the
    denominator floored at `floor` x that maximum."""
    a = mine.detach().double().cpu().reshape(-1)[torch.from_numpy(gold[name + "_idx"])]
    b = torch.from_numpy(gold[name]).double()
    amax = float(gold[name + "_amax"])
    if floor is None:
        return float((a - b).abs().max() / amax)
    return float(((a - b).abs() / b.abs().clamp(min=floor * amax)).max())


def test_iou_feature_branch_matches_reference_get_iou_feat():
    gold = _gold()
    sd = iou_state_dict(gold)
    from pytracking_b200 import synth
    from pytracking_b200.engine import BackboneEngine
    im = synth.make_crop(3, 2, 288)
    eng = BackboneEngine(sd, arch="resnet50", max_batch=2, crop_size=288)
    eng.attach_iou_head(sd)
    out = eng.forward(im.cuda(), want=("layer2", "layer3", "iou3", "iou4"))
    again = eng.iou_features(2)                                   # the branch alone, from the arena
    assert torch.equal(again[0], out["iou3"]) and torch.equal(again[1], out["iou4"])
    for mine, name in ((out["iou3"], "feat_c3"), (out["iou4"], "feat_c4")):
        assert _sampled_rel(mine, gold, name) < 1e-4, (name, _sampled_rel(mine, gold, name))
        # element-wise: entries above 1 % of the map's maximum to 2e-3 (two more 3x3 layers after layer2 / layer3)
        assert _sampled_rel(mine, gold, name, 1e-2) < 2e-3, (name, _sampled_rel(mine, gold, name, 1e-2))
    eng.close()


def test_predict_iou_and_box_gradient_match_reference_autograd():
    gold = _gold()
    from pytracking_b200.iou import IoUPredictor
    pred = IoUPredictor(iou_state_dict(gold))
    for seed, R in ((0, 10), (1, 1), (2, 16)):
        mod, feat, boxes = iou_inputs(seed, R)
        iou, grad = pred.predict_iou([m.cuda() for m in mod], [f.cuda() for f in feat], boxes.cuda(), return_grad=True)
        ref_i, ref_g = torch.from_numpy(gold["piou_%d_iou" % seed]), torch.from_numpy(gold["piou_%d_grad" % seed])
        assert _rel(iou, ref_i) < 1e-4, (seed, _rel(iou, ref_i))
        assert _rel(grad, ref_g) < 1e-4, (seed, _rel(grad, ref_g))
        assert _rel_elem(iou, ref_i, 1e-3) < 1e-3
    pred.close()


@pytest.mark.parametrize("relative", [False, True])
def test_refinement_loop_matches_reference_optimize_boxes(relative):
    gold = _gold()
    from pytracking_b200.iou import IoUPredictor
    pred = IoUPredictor(iou_state_dict(gold))
    mod, feat, boxes = iou_inputs(7, 10)
    iters, step = (10, 2.5e-3) if relative else (5, 1.0)
    ref_boxes = torch.from_numpy(gold["refine_%d_%d_boxes" % (iters, relative)])
    ref_iou = torch.from_numpy(gold["refine_%d_%d_iou" % (iters, relative)])
    b, iou = pred.refine([m.cuda() for m in mod], [f.cuda() for f in feat], boxes.cuda(), iters, step, 1, relative)
    assert _rel(b, ref_boxes) < 1e-4, _rel(b, ref_boxes)
    assert float((b.cpu() - ref_boxes).abs().max()) < 2e-2            # pixels, after 5 / 10 ascent steps of O(1..10) px each
    assert _rel(iou, ref_iou) < 1e-3, _rel(iou, ref_iou)
    moved = float((ref_boxes - boxes.reshape(-1, 4)).abs().max())
    assert moved > 0.5, moved                                           # the loop really moved the boxes
    pred.close()


def _ref_iou_and_grad(net, mod, feat, boxes, device):
    netd = net.to(device)
    bb = boxes.clone().to(device).requires_grad_(True)
    iou = netd.bb_regressor.predict_iou([m.to(device) for m in mod], [f.to(device) for f in feat], bb)
    iou.backward(gradient=torch.ones_like(iou))
    return iou.detach().cpu(), bb.grad.detach().cpu()


def test_plugin_predict_iou_seam_keeps_the_trackers_autograd_code_working():
    net = _ref_net()
    from pytracking_b200 import plugin
    mod, feat, boxes = iou_inputs(11, 10)
    i_cpu, g_cpu = _ref_iou_and_grad(net, mod, feat, boxes, "cpu")
    plugin.install()
    plugin.stats.clear()
    try:
        i_eng, g_eng = _ref_iou_and_grad(net, mod, feat, boxes, "cuda")         # dimp.py:737-742 verbatim: predict_iou + backward
        assert plugin.stats.get("predict_iou", 0) == 1 and not plugin.stats.get("prroi_pooling_forward")
    finally:
        plugin.uninstall()
        net.cpu()
    assert _rel(i_eng, i_cpu) < 1e-4 and _rel(g_eng, g_cpu) < 1e-4, (_rel(i_eng, i_cpu), _rel(g_eng, g_cpu))
