"""-m gpu: PrRoIPool, predict_iou and every IoUNet refinement step checked against float64, entry by entry (tests/iou_step_ref.py).

Every error is normalised by its own magnitude term (a pooled value by sum |f| Wy Wx / |bin|, a gradient entry by the sum of the
absolute terms that make it up, an IoU by sum_j |wp_j a_j| + |bp|), never by a global maximum, and must satisfy
e <= max(4 e_32, B / N): e_32 is the error of the reference's own float32 formulation of the same entry and B the bound on the float32
error of the kernel's summation order and weight arithmetic (iou_step_ref.Bins._sum_bound and the comments beside each step).

  a. the three PrRoIPool kernels through the C ABI on the geometry grid: maps 36 / 44 at 1/8, 18 / 22 at 1/16 (and 62 at 1/8, where
     a bin covers PR_MAXW - 2 cells: every case asserts a bin covering all n cells of a row or column), pooled 5x5, 3x3 and 7x7, B = 1 and 3, C = 160; every class of iou_step_ref.CLASSES reached.
     Boxes wholly outside the map, of zero width or height, or of negative width give exactly 0.  The feature backward adds with
     atomicAdd in any order and is held to its bound, not to bits.
  b. IoUPredictor.predict_iou and its box gradient at R = 1, 2, 10, 15, 16 on the DiMP (36 / 18) and PrDiMP (44 / 22) maps, boxes of
     every class; the gradient with the kink allowance.  The first R rows of a 16-box call equal an R-box call, a permutation of the
     boxes permutes every output and a repeat gives the same bits.
  c. IoUPredictor.refine in default space (5 iterations, step 1) and relative space (10, 2.5e-3), each with decay 1 and 0.8: iterate
     b_k is refine(num_iter=k); each step b_{k+1} - b_k against the float64 step from b_k; the IoUs refine returns equal predict_iou
     on b_{N-1} bit for bit.
Parts b and c are also held, case by case, to the yardstick itself: the worst e of a case within 20 x its worst e_32 plus 64 ulp
(iou_step_ref.yardstick_ratio; steps less the boxes' own rounding), which catches defects far below the worst-case bound of these
cancelling sums.

One line per case reports the worst e / bar, e / e_32 and kink units; test_zz_report the worst per kernel and geometry class.  The
file takes 80 s of test time (90 s with start-up) on an NVIDIA H100 80GB HBM3 at its 700 W power limit; most of it is the
reference's cell-by-cell float32 yardstick on the bins that span a whole map."""
import collections

import numpy as np
import pytest
import torch

import iou_step_ref as R
from pytracking_b200 import ops
from ref_weights import GOLDEN, iou_state_dict

pytestmark = pytest.mark.gpu
REPORT = collections.defaultdict(lambda: [0.0, 0.0, 0.0])      # (kernel, class) -> worst e / bar, e, e_32
KINKS = collections.Counter()
REACHED = set()
GRID_RUN = []
YARDS = collections.defaultdict(float)     # worst e_max / (YARD e32_max + FLOOR) per part


@pytest.fixture(scope="module")
def sd():
    return iou_state_dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def net(sd):
    return R.IoUNet64(sd, device="cuda")


@pytest.fixture(scope="module")
def pred(sd):
    from pytracking_b200.iou import IoUPredictor
    p = IoUPredictor(sd)
    yield p
    p.close()


def _merge(key, q):
    REPORT[key] = [max(a, b) for a, b in zip(REPORT[key], q)]


def _fwd(feat, rois, P, scale):
    return ops.prroi_pool_forward(feat, rois, P, P, scale)


def _bwd(feat, rois, out, og, P, scale):
    return ops.prroi_pool_backward(feat, rois, out, og, P, P, scale)


def _coor(feat, rois, out, og, P, scale):
    return ops.prroi_pool_coor_backward(feat, rois, out, og, P, P, scale)


@pytest.mark.parametrize("n,scale,P,B", R.PRROI_CASES)
def test_prroi_geometry_grid_vs_float64(n, scale, P, B):
    res, reached, cells = R.check_prroi(_fwd, _bwd, _coor, n, scale, P, B, 160, n + P + B, "cuda")
    REACHED.update(reached)
    GRID_RUN.append((n, scale, P, B))
    for k, q in res.items():
        _merge(k, q)
    print("prroi %dx%d 1/%d %dx%d B=%d: worst e/bar %.3f; widest bin %d cells" % (n, n, round(1 / scale), P, P, B,
                                                                             max(v[0] for v in res.values()), cells))


def _predict(pred, mod, feat):
    def run(boxes):
        i, g = pred.predict_iou(mod, feat, boxes.float().contiguous(), return_grad=True)
        return i.reshape(-1), g.reshape(-1, 4)
    return run


def _case_boxes(maps, R_, seed):
    boxes = R.class_boxes(R.IOU_MAPS[maps], seed, "cuda")
    perm = torch.randperm(boxes.shape[0], generator=torch.Generator().manual_seed(R_))
    return boxes, perm


@pytest.mark.parametrize("maps", sorted(R.IOU_MAPS))
@pytest.mark.parametrize("R_", [1, 2, 10, 15, 16])
def test_predict_iou_vs_float64(pred, net, maps, R_):
    mod, feat = R.iou_inputs_on(R.IOU_MAPS[maps], 256, R_, "cuda")
    boxes, perm = _case_boxes(maps, R_, R_)
    run = _predict(pred, mod, feat)
    for part in ((perm[:R_],) if R_ < 16 else (perm[:16], perm[12:28])):
        q = R.check_predict(run, net, R.IOU_MAPS[maps], R_, mod, feat, boxes[part])
        _merge(("predict_iou iou", maps), q[:3])
        _merge(("predict_iou grad", maps), q[3:6])
        KINKS[("predict_iou", maps)] += q[6]
        for b in boxes[part]:
            REACHED.update(R.classify(torch.cat([torch.zeros(1), b.cpu()[:2], b.cpu()[:2] + b.cpu()[2:]]), R.IOU_MAPS[maps][0],
                                      R.IOU_MAPS[maps][0], 5, 5, 1.0 / 8))
        YARDS["predict_iou iou"] = max(YARDS["predict_iou iou"], q[7])
        YARDS["predict_iou grad"] = max(YARDS["predict_iou grad"], q[8])
        print("predict_iou %s R=%d: iou e/bar %.3f e/e32 %.2f; grad e/bar %.3f e/e32 %.2f; yardstick %.3f / %.3f; kink units %d"
              % (maps, R_, q[0], q[1] / max(q[2], 1e-300), q[3], q[4] / max(q[5], 1e-300), q[7], q[8], q[6]))


@pytest.mark.parametrize("maps", sorted(R.IOU_MAPS))
def test_predict_iou_rows_permutation_repeat_bitwise(pred, maps):
    mod, feat = R.iou_inputs_on(R.IOU_MAPS[maps], 256, 3, "cuda")
    boxes, perm = _case_boxes(maps, 16, 5)
    b16 = boxes[perm[:16]].contiguous()
    i16, g16 = pred.predict_iou(mod, feat, b16, return_grad=True)
    for r in (1, 2, 10, 15):
        i, g = pred.predict_iou(mod, feat, b16[:r].contiguous(), return_grad=True)
        assert torch.equal(i[0], i16[0, :r]) and torch.equal(g[0], g16[0, :r]), r
    p = torch.randperm(16, generator=torch.Generator().manual_seed(1)).cuda()
    ip, gp = pred.predict_iou(mod, feat, b16[p].contiguous(), return_grad=True)
    assert torch.equal(ip[0], i16[0, p]) and torch.equal(gp[0], g16[0, p])
    i2, g2 = pred.predict_iou(mod, feat, b16, return_grad=True)
    assert torch.equal(i2, i16) and torch.equal(g2, g16)


@pytest.mark.parametrize("cfg", R.refine_configs(), ids=[c[0] for c in R.refine_configs()])
def test_every_refinement_step_vs_float64(pred, net, cfg):
    name, relative, iters, step, decay = cfg
    maps = "prdimp 352" if relative else "dimp 288"
    mod, feat = R.iou_inputs_on(R.IOU_MAPS[maps], 256, 40 + iters, "cuda")
    boxes = R.class_boxes(R.IOU_MAPS[maps], 41, "cuda", positive=True)
    keep = [i for i in range(boxes.shape[0]) if not (R.classify(torch.cat([torch.zeros(1), boxes[i].cpu()[:2], boxes[i].cpu()[:2] + boxes[i].cpu()[2:]]),
                                                                   R.IOU_MAPS[maps][0], R.IOU_MAPS[maps][0], 5, 5, 1.0 / 8) & {"wholly outside"})]
    boxes = boxes[keep][:16].contiguous()

    def refine(b, k):
        return pred.refine(mod, feat, b, k, step, decay, relative)
    q, bs = R.check_refine(refine, net, mod, feat, boxes, relative, iters, step, decay)
    _, iou = refine(boxes, iters)
    i_last = pred.predict_iou(mod, feat, bs[iters - 1].contiguous())
    assert torch.equal(iou, i_last.reshape(-1))
    moved = float((bs[-1] - bs[0]).abs().max())
    assert moved > 0.1, moved
    _merge(("refine step", name), q[:3])
    KINKS[("refine", name)] += q[3]
    YARDS["refine step"] = max(YARDS["refine step"], q[4])
    print("refine %s: %d boxes, %d steps: worst e/bar %.3f e/e32 %.2f; yardstick %.3f; kink units %d; moved %.2f px"
          % (name, boxes.shape[0], iters, q[0], q[1] / max(q[2], 1e-300), q[4], q[3], moved))


def test_zz_report():
    if not REPORT:
        pytest.skip("no case ran")
    for (k, c), (q, e, e32) in sorted(REPORT.items()):
        print("iou f64 worst %-18s %-20s e/bar %.3f  e %.2e  e_32 %.2e  e/e_32 %.2f" % (k, c, q, e, e32, e / max(e32, 1e-300)))
    print("iou f64 kink units: %s" % dict(KINKS))
    print("iou f64 worst yardstick ratio e / (%d e_32 + 64 ulp): %s" % (R.YARD, {k: round(v, 3) for k, v in YARDS.items()}))
    if len(GRID_RUN) == len(R.PRROI_CASES):
        assert REACHED >= set(R.CLASSES), set(R.CLASSES) - REACHED
