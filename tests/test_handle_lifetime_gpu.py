"""-m gpu tests of how the library's handles hold device memory:
  * a refused b200trk_net_attach_iou_head leaves the plan as it was (steps, IoU geometry, forward outputs bit for bit), and a
    corrected call then attaches the head;
  * ten create / destroy cycles of every handle type give back the device memory they took."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib, synth

pytestmark = pytest.mark.gpu

# as in test_tomp_steps_f64_gpu.py: other work on the device moves its free memory a little.  A DiMP-50 plan holds one weight copy of
# 52 MB at precision 1 and three at precision 0, so one plan leaked per cycle is far outside this after ten cycles.
SLACK = 64 << 20
CYCLES = 10
WANT = ("layer2", "layer3", "classification")


def _iou_sd():
    from ref_weights import GOLDEN, iou_state_dict
    return iou_state_dict(np.load(GOLDEN))


def _plan(eng):
    d = (C.c_int * 6)()
    _lib.check(_lib.lib().b200trk_net_iou_dims(eng.handle, C.byref(d)), "net_iou_dims")
    return _lib.lib().b200trk_net_num_ops(eng.handle), list(d)


def _same_outputs(a, b, im, want):
    for _ in range(3):                 # two eager passes, then the captured graph
        oa, ob = a.forward(im, want), b.forward(im, want)
        torch.cuda.synchronize()
        for k in want:
            assert torch.equal(oa[k], ob[k]), k


def test_refused_iou_head_leaves_the_plan_as_it_was():
    from pytracking_b200.engine import BackboneEngine
    sd = _iou_sd()
    bad = dict(sd)
    w = sd["bb_regressor.conv4_1t.0.weight"]
    bad["bb_regressor.conv4_1t.0.weight"] = w[:, :w.shape[1] // 2]      # layer3 has twice the channels conv4_1t now reads
    im = synth.make_crop(3, 1, 288).cuda()
    eng, fresh = BackboneEngine(sd), BackboneEngine(sd)
    try:
        before = _plan(eng)
        with pytest.raises(RuntimeError, match="conv4_1t"):
            eng.attach_iou_head(bad)
        assert _plan(eng) == before, "a refused attach changed the plan"
        _same_outputs(eng, fresh, im, WANT)
        eng.attach_iou_head(sd)
        fresh.attach_iou_head(sd)
        assert _plan(eng) == _plan(fresh) and _plan(eng)[1][0] > 0
        _same_outputs(eng, fresh, im, WANT + ("iou3", "iou4"))
    finally:
        eng.close()
        fresh.close()


# ---- create / destroy cycles: each builds the handle, runs it where that is cheap, and closes it --------------------------------------
def _net(precision):
    def cycle():
        from pytracking_b200.engine import BackboneEngine
        eng = BackboneEngine(synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3), precision=precision)
        im = synth.make_crop(1, 1, 288).cuda()
        for _ in range(3):             # up to the captured graph and its capture stream
            eng.forward(im)
        torch.cuda.synchronize()
        eng.close()
    return cycle


def _tower():
    from ref_weights import GOLDEN, tower_state_dict
    from pytracking_b200.transformer_engine import BoxTower
    tw = BoxTower(tower_state_dict(np.load(GOLDEN)), 18, 18, max_batch=4)
    tw.forward(torch.rand(4, 256, 18, 18, device="cuda"), torch.rand(4, 18, 18, device="cuda"))
    torch.cuda.synchronize()
    tw.close()


def _transformer():
    from pytracking_b200.transformer_engine import TransformerEngine
    L, B, d = 324, 2, 256
    eng = TransformerEngine(synth.make_transformer_state_dict(98, d, 8, 2048, 1, 1), L, B, d, 8, 2048, 1, 1)
    g = torch.Generator().manual_seed(0)
    src, pos, qe = torch.randn(L, B, d, generator=g), torch.randn(L, 1, d, generator=g), torch.randn(1, d, generator=g)
    eng.forward(src.cuda(), None, qe.cuda(), pos.cuda())
    torch.cuda.synchronize()
    eng.close()


def _iou_predictor():
    from pytracking_b200.iou import IoUPredictor
    IoUPredictor(_iou_sd()).close()


def _iou_modulation():
    from pytracking_b200.iou import IoUModulation
    IoUModulation(_iou_sd()).close()


def _state(newton):
    def cycle():
        from pytracking_b200.frame_engine import DiMPFrameEngine
        DiMPFrameEngine(synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3), newton=newton).close()
    return cycle


def _tracker():
    from test_augment_cpu import STOCK
    from tracker_cases import DIMP50
    from pytracking_b200.tracker import DiMPTracker, make_params
    sd = _iou_sd()
    trk = DiMPTracker(sd, make_params(**dict(DIMP50, use_iou_net=True)), filter_init="network", augmentation=STOCK,
                      random_shift_factor=1 / 3)
    trk.attach_iounet(sd)              # native modulation: initialize computes the vectors
    frames, bb = synth.make_sequence(0, num_frames=2)
    trk.initialize(frames[0], {"init_bbox": bb})
    trk.track(frames[1])
    torch.cuda.synchronize()
    trk.close()


def _batch():
    from tracker_cases import DIMP50
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import make_params
    bt = DiMPBatchTracker(synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3), make_params(**DIMP50), 4)
    seqs = [synth.make_sequence(q, num_frames=2) for q in range(4)]
    bt.step({s: (seqs[s][0][0], {"init_bbox": seqs[s][1]}) for s in range(4)})
    bt.step({s: (seqs[s][0][1], None) for s in range(4)})
    torch.cuda.synchronize()
    bt.close()


CYCLE = {"net_p0": _net(0), "net_p1": _net(1), "net_p2": _net(2), "tower": _tower, "transformer": _transformer,
         "iou_predictor": _iou_predictor, "iou_modulation": _iou_modulation, "gn_state": _state(None), "newton_state": _state({}),
         "tracker_iounet_augmented": _tracker, "batch": _batch}


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize("kind", sorted(CYCLE))
def test_create_destroy_cycles_give_back_device_memory(kind):
    CYCLE[kind]()                      # process-lifetime state (modules, kernel attributes, the scratch workspace) settles first
    free0 = _free()
    for _ in range(CYCLES):
        CYCLE[kind]()
    free1 = _free()
    assert free1 >= free0 - SLACK, "%s: %d create / destroy cycles kept %.1f MB of device memory" % (kind, CYCLES, (free0 - free1) / 2**20)
