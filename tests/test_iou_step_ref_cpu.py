"""tests/iou_step_ref.py pinned on the CPU: its float64 predict_iou, box gradient and ascent steps against the unmodified reference's
float32 autograd runs in tests/golden/iou_tomp_ref.npz; its PrRoIPool forward and coordinate gradient against oracle/prroi_oracle.py and
against central differences of its own forward on the geometry grid of tests/test_iou_steps_f64_gpu.py; the reference's known-answer
test (PrRoIPool equals avg_pool2d on integer-aligned RoIs)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import iou_step_ref as R
from ref_weights import GOLDEN, iou_inputs, iou_state_dict

GRID = [(36, 36, 1.0 / 8), (18, 18, 1.0 / 16)]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def net(gold):
    return R.IoUNet64(iou_state_dict(gold))


def _lists(mod, feat):
    return [m.reshape(-1) for m in mod], [f for f in feat]


@pytest.mark.parametrize("seed,n", [(0, 10), (1, 1), (2, 16)])
def test_predict_iou_and_gradient_vs_reference_golden(net, gold, seed, n):
    """Per box: the golden is a float32 run, so each IoU is held to 2e-6 of its magnitude term and each gradient entry to 2e-5 of its."""
    mod, feat, boxes = iou_inputs(seed, n)
    mod, feat = _lists(mod, feat)
    out = net.evaluate(mod, feat, boxes.reshape(-1, 4), yardstick=False)
    gi, gg = torch.from_numpy(gold["piou_%d_iou" % seed]).reshape(-1).double(), torch.from_numpy(gold["piou_%d_grad" % seed]).reshape(-1, 4).double()
    ei = ((out["iou"] - gi).abs() / out["iouN"]).max()
    eg = ((out["grad"] - gg).abs() / out["gradN"]).max()
    assert ei < 2e-6 and eg < 2e-5, (float(ei), float(eg))


@pytest.mark.parametrize("iters,relative", [(5, False), (10, True)])
def test_refinement_vs_reference_golden(net, gold, iters, relative):
    """The float64 steps from the same initial boxes end, per box and coordinate, within 1e-4 of the path the coordinate travelled
    (sum_k |d_k|) plus 8 ulp per step of the coordinate of the reference's float32 loop: the golden's gradients carry float32 errors of
    about 1e-6 of their magnitude, which the steps carry and the later steps' Jacobians amplify (observed 1.1e-5 / 2.0e-5 of the path).
    The IoUs of the last forward are held to 1e-5 of their magnitude term."""
    mod, feat, boxes = iou_inputs(7, 10)
    mod, feat = _lists(mod, feat)
    b = boxes.reshape(-1, 4).double()
    sz = b[0, 2:].clone()
    step = 2.5e-3 if relative else 1.0
    path = torch.zeros_like(b)
    for _ in range(iters):
        out = net.evaluate(mod, feat, b.float(), yardstick=False)
        d = R.box_step(b, out["grad"], step, relative, sz)
        path += d.abs()
        b = b + d
    ref_b, ref_i = torch.from_numpy(gold["refine_%d_%d_boxes" % (iters, int(relative))]).double(), torch.from_numpy(gold["refine_%d_%d_iou" % (iters, int(relative))]).double()
    err = (b - ref_b).abs()
    assert bool((err <= 1e-4 * path + 8 * iters * R.U * ref_b.abs()).all()), float((err / path).max())
    assert float(((out["iou"] - ref_i).abs() / out["iouN"]).max()) < 1e-5
    assert float((ref_b - boxes.reshape(-1, 4)).abs().max()) > 0.5


def test_yardstick_runs_the_reference_order(net, gold):
    """The float32 yardstick is a float32 computation of the same function: within 1e-5 (IoU) / 1e-4 (gradient) of float64, per box."""
    mod, feat, boxes = iou_inputs(0, 10)
    mod, feat = _lists(mod, feat)
    out = net.evaluate(mod, feat, boxes.reshape(-1, 4))
    assert float(((out["iou32"].double() - out["iou"]).abs() / out["iouN"]).max()) < 1e-5
    assert float(((out["grad32"] - out["grad"]).abs() / out["gradN"]).max()) < 1e-4
    assert out["kinks"] == 0 and float(out["allow"].abs().max()) == 0.0


@pytest.mark.parametrize("H,W,scale", GRID)
@pytest.mark.parametrize("P", [3, 5, 7])
def test_forward_and_gradients_vs_oracle_and_finite_differences(H, W, scale, P):
    """Forward and feature backward against the oracle to 1e-12; the coordinate gradient against the oracle and against central
    differences (h = 1e-6 px) of the float64 forward to 1e-7 of its magnitude term, on every RoI of the geometry grid."""
    from oracle import prroi_oracle as O
    g = torch.Generator().manual_seed(P)
    rois = R.geometry_rois(H, W, P, P, scale, 2, seed=P)
    feat = torch.randn(2, 6, H, W, generator=g, dtype=torch.float64)
    og = torch.randn(rois.shape[0], 6, P, P, generator=g, dtype=torch.float64)
    out, N, _ = R.forward(feat, rois, P, P, scale)
    assert float((out - torch.from_numpy(O.forward(feat.numpy(), rois.numpy(), P, P, scale))).abs().max()) < 1e-12
    fg, _, _ = R.backward(feat, rois, og, P, P, scale)
    assert float((fg - torch.from_numpy(O.backward(feat.numpy(), rois.numpy(), og.numpy(), P, P, scale))).abs().max()) < 1e-12
    rg, rN, _ = R.coor_backward(feat, rois, out, og, P, P, scale)
    ref = torch.from_numpy(O.coor_backward(feat.numpy(), rois.numpy(), out.numpy(), og.numpy(), P, P, scale))[:, 1:]
    assert float(((rg - ref).abs() / rN.clamp(min=1e-300)).max()) < 1e-12
    h = 1e-6
    r64 = rois.double()
    fd = torch.zeros_like(rg)
    for q in range(4):
        rp, rm = r64.clone(), r64.clone()
        rp[:, 1 + q] += h
        rm[:, 1 + q] -= h
        fp = (R.forward(feat, rp, P, P, scale)[0] * og).sum((1, 2, 3))
        fm = (R.forward(feat, rm, P, P, scale)[0] * og).sum((1, 2, 3))
        fd[:, q] = (fp - fm) / (2 * h)
    # skip the coordinates a difference step would move across w = 0 (the clamp of the extent: a kink of the forward itself)
    x0, y0, x1, y1 = r64[:, 1], r64[:, 2], r64[:, 3], r64[:, 4]
    smooth = ((x1 - x0).abs() > 2 * h) & ((y1 - y0).abs() > 2 * h)
    e = (rg - fd).abs() / rN.clamp(min=1e-300)
    assert bool((rN[smooth] > 0).any())
    assert float(e[smooth].max()) < 1e-7, float(e[smooth].max())
    reached = set().union(*(R.classify(r, H, W, P, P, scale) for r in rois))
    assert reached == set(R.CLASSES), set(R.CLASSES) - reached


def test_known_answer_avg_pool():
    """The reference's own test (PreciseRoIPooling/pytorch/tests/test_prroi_pooling2d.py:21-35): on integer-aligned RoIs with
    spatial_scale 0.5, PrRoIPool 7x7 equals avg_pool2d(k=2, s=1) slices -- in float64 and in the float32 formulation."""
    feat = torch.rand(4, 16, 24, 32, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    rois = torch.tensor([[0, 0, 0, 14, 14], [1, 14, 14, 28, 28]], dtype=torch.float32)
    ref = F.avg_pool2d(feat, kernel_size=2, stride=1)
    for out, tol in ((R.forward(feat, rois, 7, 7, 0.5)[0], 1e-14), (R.forward_f32(feat, rois, 7, 7, 0.5).double(), 1e-6)):
        assert float((out[0] - ref[0, :, :7, :7]).abs().max()) < tol and float((out[1] - ref[1, :, 7:14, 7:14]).abs().max()) < tol


@pytest.mark.parametrize("H,W,scale", GRID)
@pytest.mark.parametrize("P", [3, 5, 7])
def test_float32_yardsticks_within_the_float32_bound(H, W, scale, P):
    """The three float32 yardsticks (the reference's cell-by-cell formulation) are float32 computations of the same functions: every
    entry within the float32 bound B of its float64 value (what the kernels' e_32 side of the bar rests on), exact zeros where the
    magnitude term is 0, on every RoI of the geometry grid."""
    g = torch.Generator().manual_seed(10 + P)
    rois = R.geometry_rois(H, W, P, P, scale, 2, seed=10 + P)
    feat = torch.randn(2, 6, H, W, generator=g)
    og = torch.randn(rois.shape[0], 6, P, P, generator=g)
    o64, oN, oB = R.forward(feat, rois, P, P, scale)
    top = o64.float()
    f64, fN, fB = R.backward(feat, rois, og, P, P, scale)
    r64, rN, rB = R.coor_backward(feat, rois, top, og, P, P, scale)
    for name, y, ref, N, B in (("forward", R.forward_f32(feat, rois, P, P, scale), o64, oN, oB),
                               ("backward", R.backward_f32(feat, rois, og, P, P, scale), f64, fN, fB),
                               ("coor_backward", R.coor_backward_f32(feat, rois, top, og, P, P, scale), r64, rN, rB)):
        err = (y.double() - ref).abs()
        assert bool((err <= B).all()), (name, float((err / B.clamp(min=1e-300)).max()))
        assert float(y[N == 0].abs().max()) == 0 if bool((N == 0).any()) else True, name
