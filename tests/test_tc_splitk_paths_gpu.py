"""-m gpu: the two split-K reductions of conv_tc.cu give bitwise the same layer outputs.

A split-K layer reduces its partial tiles either through distributed shared memory (the split CTAs of a tile form a cluster) or
through the L2 workspace. `tc_configure` picks the workspace for cluster grids the device cannot hold at once (clusters of 3 and 5
on a 132-SM H100), so which path a layer takes depends on the device. Both add the same staged partials in split order, so the
forward pass must not change with the choice. The check runs the bench plan twice on one crop: once with the default choice and
once with B200TRK_TC_CLUSTER=0 (every split-K layer on the workspace). Every layer up to the first one whose launch geometry
differs between the two runs (without clusters the split count may exceed 8) must be bitwise equal."""
import ctypes as C

import pytest
import torch

from pytracking_b200 import _lib, synth
from pytracking_b200.engine import BackboneEngine

pytestmark = pytest.mark.gpu

OP_CONV = 3


def _run(sd, im):
    """{plan index: (grid, NHWC output)} of every tensor-core step after one forward pass of batch 1."""
    L = _lib.lib()
    eng = BackboneEngine(sd, arch="resnet50", max_batch=1, crop_size=288, precision=0)
    try:
        eng.forward(im, want=("layer2", "layer3", "classification"))
        torch.cuda.synchronize()
        out = {}
        for i in range(L.b200trk_net_num_ops(eng.handle)):
            info = (C.c_int * 8)()
            _lib.check(L.b200trk_net_op_info(eng.handle, i, C.byref(info)), "net_op_info")
            if info[0] != OP_CONV or not info[7]:
                continue
            g = (C.c_int * 4)()
            _lib.check(L.b200trk_net_op_grid(eng.handle, i, C.byref(g)), "net_op_grid")
            t = torch.empty(1, info[5], info[6], info[2], device="cuda")
            _lib.check(L.b200trk_net_op_output(eng.handle, i, 1, C.c_void_p(t.data_ptr()), None), "net_op_output")
            out[i] = (list(g), t)
        torch.cuda.synchronize()
        return out
    finally:
        eng.close()


def test_splitk_reductions_bitwise_equal(monkeypatch):
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    im = synth.make_crop(41, 1, 288).cuda()
    default = _run(sd, im)
    monkeypatch.setenv("B200TRK_TC_CLUSTER", "0")
    workspace = _run(sd, im)
    assert default.keys() == workspace.keys()
    compared_splits = set()
    for i in sorted(default):
        (g, y), (g0, y0) = default[i], workspace[i]
        if g != g0:
            break
        assert torch.equal(y, y0), "step %d (grid %s): the two split-K reductions differ" % (i, g)
        compared_splits.add(g[2])
    # the compared prefix must cover split-K layers on both sides of the choice: 2 and 4 splits fit as clusters, 3 and 5 do not
    assert {2, 3, 4, 5} <= compared_splits, compared_splits
