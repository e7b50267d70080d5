"""The float64 checks of tests/test_iou_steps_f64_gpu.py in the CPU tier: the PrRoIPool geometry grid and the predict_iou cases run the
kernel sources of csrc/prroi_kernels.cuh and csrc/iou_refine_kernels.cuh on the CPU under tests/cpu_emul/cuda_shim.h (prroi_emul.cpp,
iou_emul.cpp), held to the same bars (tests/iou_step_ref.py).  The shim is built with -ffp-contract=off and the device may contract
differently, so the two tiers share bars, not bits."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import iou_step_ref as R
from ref_weights import GOLDEN, iou_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REACHED = set()


def _build(tmp_path_factory, name):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp(name)), "lib%s.so" % name)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", name + ".cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def prroi(tmp_path_factory):
    return _build(tmp_path_factory, "prroi_emul")


@pytest.fixture(scope="module")
def iou(tmp_path_factory):
    return _build(tmp_path_factory, "iou_emul")


@pytest.fixture(scope="module")
def sd():
    return iou_state_dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def net(sd):
    return R.IoUNet64(sd)


def _p(t):
    return C.c_void_p(t.data_ptr())


def _kernels(lib):
    def fwd(feat, rois, P, scale):
        out = torch.full((rois.shape[0], feat.shape[1], P, P), float("nan"))
        assert lib.prroi_emul_forward(_p(feat), _p(rois), _p(out), *feat.shape, rois.shape[0], P, P, C.c_float(scale)) == 0
        return out

    def bwd(feat, rois, out, og, P, scale):
        fg = torch.full_like(feat, float("nan"))
        assert lib.prroi_emul_backward(_p(rois), _p(og), _p(fg), *feat.shape, rois.shape[0], P, P, C.c_float(scale)) == 0
        return fg

    def coor(feat, rois, out, og, P, scale):
        rg = torch.full((rois.shape[0], 5), float("nan"))
        assert lib.prroi_emul_coor_backward(_p(feat), _p(rois), _p(out), _p(og), _p(rg), *feat.shape, rois.shape[0], P, P, C.c_float(scale)) == 0
        return rg
    return fwd, bwd, coor


@pytest.mark.parametrize("n,scale,P,B", R.PRROI_CASES)
def test_prroi_geometry_grid_vs_float64(prroi, n, scale, P, B):
    res, reached, cells = R.check_prroi(*_kernels(prroi), n, scale, P, B, 40, n + P + B, "cpu")
    REACHED.update(reached)
    print("prroi cpu %dx%d 1/%d %dx%d B=%d: worst e/bar %.3f; widest bin %d cells" % (n, n, round(1 / scale), P, P, B,
                                                                             max(v[0] for v in res.values()), cells))


def test_prroi_grid_reached_every_class():
    if len(REACHED) == 0:
        pytest.skip("the grid did not run")
    assert REACHED == set(R.CLASSES), set(R.CLASSES) - REACHED


def _emul_predict(lib, sd, mod, feat):
    keep = []
    from pytracking_b200 import _lib

    def hp(key):
        t = sd["bb_regressor." + key].detach().float().contiguous()
        keep.append(t)
        return t

    def block(name):
        return _lib.LinearBlock(hp(name + ".linear.weight").data_ptr(), hp(name + ".linear.bias").data_ptr(), hp(name + ".bn.weight").data_ptr(),
                                hp(name + ".bn.bias").data_ptr(), hp(name + ".bn.running_mean").data_ptr(), hp(name + ".bn.running_var").data_ptr())
    b3, b4 = block("fc3_rt"), block("fc4_rt")
    wp, bp = hp("iou_predictor.weight"), hp("iou_predictor.bias")
    D3, D4 = sd["bb_regressor.fc3_rt.linear.weight"].shape[0], sd["bb_regressor.fc4_rt.linear.weight"].shape[0]
    m3, m4 = mod[0].contiguous(), mod[1].contiguous()
    f3, f4 = feat[0].contiguous(), feat[1].contiguous()

    def run(boxes):
        bx = boxes.float().contiguous().clone()
        r = bx.shape[0]
        iou, grad = torch.full((r,), float("nan")), torch.full((r, 4), float("nan"))
        assert lib.iou_emul_run(C.byref(b3), C.byref(b4), _p(wp), _p(bp), 256, 5, 256, 3, D3, D4, _p(m3), _p(m4), _p(f3), f3.shape[2], f3.shape[3],
                                _p(f4), f4.shape[2], f4.shape[3], _p(bx), r, 0, C.c_float(1.0), C.c_float(1.0), 0, _p(iou), _p(grad)) == 0
        keep.append(bx)
        return iou, grad
    return run


@pytest.mark.parametrize("maps", sorted(R.IOU_MAPS))
@pytest.mark.parametrize("R_", [1, 2, 10, 15, 16])
def test_predict_iou_vs_float64(iou, sd, net, maps, R_):
    """The predict_iou cases of tests/test_iou_steps_f64_gpu.py part b: the same boxes, and both 16-box slices at R = 16."""
    mod, feat = R.iou_inputs_on(R.IOU_MAPS[maps], 256, R_, "cpu")
    boxes = R.class_boxes(R.IOU_MAPS[maps], R_, "cpu")
    perm = torch.randperm(boxes.shape[0], generator=torch.Generator().manual_seed(R_))
    run = _emul_predict(iou, sd, mod, feat)
    for part in ((perm[:R_],) if R_ < 16 else (perm[:16], perm[12:28])):
        q = R.check_predict(run, net, R.IOU_MAPS[maps], R_, mod, feat, boxes[part])
        print("predict_iou cpu %s R=%d: iou e/bar %.3f e/e32 %.2f; grad e/bar %.3f e/e32 %.2f; yardstick %.3f / %.3f; kink units %d"
              % (maps, R_, q[0], q[1] / max(q[2], 1e-300), q[3], q[4] / max(q[5], 1e-300), q[7], q[8], q[6]))
