"""-m gpu tests of the native IoUNet modulation (AtomIoUNet.get_modulation: b200trk_net_attach_iou_ref, b200trk_iou_modulation_*, and
DiMPTracker.attach_iounet(state_dict) without vectors), against the PrDiMP-50 reference run recorded with its seeded bb_regressor
(tests/golden/prdimp_host_iou.npz, oracle/gen_prdimp_golden.py) and float64:
  * the vectors initialize computes from the first frame are within 1e-4 of the modulation3 / modulation4 the reference computed;
  * with them, the native tracker replays the recorded IoUNet run: flags identical, boxes within 1e-2 px;
  * conv3_1r / conv4_1r on the operands they read (criteria of tests/test_tc_conv_layers_gpu.py), PrRoIPool + the three blocks within
    1e-5 of float64 on those outputs; repeats bitwise, a box's vectors independent of the other boxes and of the image order;
  * attaching the native modulation after initialize is refused."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytracking_b200 import _lib, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "prdimp_host_iou.npz")


def _setup():
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    import ref_weights
    from test_prdimp_host_logic_cpu import prdimp_params
    from test_prdimp_tracker_gpu import newton_from_golden, prdimp_state_dict
    d = np.load(GOLDEN)
    sd = prdimp_state_dict()
    sd.update(ref_weights.seeded_state_dict(d["iou_keys"], d["iou_shapes"], 5, prefix="bb_regressor."))
    sd["bb_regressor.iou_predictor.weight"] = sd["bb_regressor.iou_predictor.weight"] * 20.0
    params = prdimp_params("noaug", use_iou_net=True, iounet_k=3, num_init_random_boxes=9, box_jitter_pos=0.1, box_jitter_sz=0.5,
                           maximal_aspect_ratio=6, box_refinement_iter=10, box_refinement_step_length=2.5e-3,
                           box_refinement_step_decay=1, box_refinement_space="relative")
    return d, sd, params, newton_from_golden(d)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("precision", [0, 1])
def test_native_modulation_replays_recorded_prdimp_iounet_run(precision):
    from pytracking_b200.tracker import DiMPTracker, FLAGS
    d, sd, params, newton = _setup()
    trk = DiMPTracker(sd, params, newton=newton, precision=precision)
    trk.attach_iounet(sd)                                   # no vectors: initialize computes them
    frames, bb = synth.make_sequence(2, num_frames=len(d["flag"]))
    trk.initialize(frames[0], {"init_bbox": bb})
    assert np.array_equal(trk.state(), d["init_state"])
    m3, m4 = trk.modulation()
    e3, e4 = _rel(m3, d["modulation3"]), _rel(m4, d["modulation4"])
    assert e3 <= 1e-4 and e4 <= 1e-4, (e3, e4)
    with pytest.raises(RuntimeError, match="after initialize"):
        trk.attach_iounet(sd)
    L = _lib.lib()
    err = []
    for t in range(len(d["flag"])):
        u = np.ascontiguousarray(d["noise"][t], dtype=np.float32)
        _lib.check(L.b200trk_dimp_tracker_set_proposal_noise(trk.handle, u.ctypes.data_as(C.c_void_p), u.size), "set_proposal_noise")
        out = trk.track(frames[t + 1])
        assert trk.info.flag == d["flag"][t], (t, FLAGS[trk.info.flag], int(d["flag"][t]))
        err.append(float(np.abs(np.array(out["target_bbox"], np.float64) - d["bbox"][t].astype(np.float64)).max()))
        assert err[-1] < 1e-2, (t, out["target_bbox"], d["bbox"][t])
    print("native PrDiMP modulation (precision %d) vs reference: mod3 %.2e, mod4 %.2e; %d frames with it, box error median %.1e px, "
          "max %.1e px" % (precision, e3, e4, len(err), float(np.median(err)), max(err)))
    trk.close()


def test_native_modulation_refused_after_initialize():
    from pytracking_b200.tracker import DiMPTracker
    d, sd, params, newton = _setup()
    trk = DiMPTracker(sd, params, newton=newton)
    frames, bb = synth.make_sequence(2, num_frames=1)
    trk.initialize(frames[0], {"init_bbox": bb})
    with pytest.raises(RuntimeError, match="after initialize"):
        trk.attach_iounet(sd)
    trk.close()


def test_modulation_layers_against_float64_and_deterministic():
    from test_tc_conv_layers_gpu import _output, _reference, _weights
    from oracle import prroi_oracle
    from pytracking_b200.engine import BackboneEngine
    from pytracking_b200.iou import IoUModulation
    d, sd, params, newton = _setup()
    S = 3
    eng = BackboneEngine(sd, "resnet50", 4, S, 352, 0)
    eng.attach_iou_ref(sd)
    head = IoUModulation(sd)
    crops = synth.make_crop(11, S, 352).cuda()
    eng.forward(crops, want=("classification",))
    boxes = np.array([[100, 120, 90, 70], [-20, 150, 80, 60], [300, 10, 40, 110]], np.float32)
    m3, m4 = head.get(eng, S, boxes)
    torch.cuda.synchronize()
    L = _lib.lib()
    n = L.b200trk_net_num_ops(eng.handle)
    ys = []
    for i in (n - 2, n - 1):                                 # conv3_1r, conv4_1r: the last two plan steps
        info, io = (C.c_int * 8)(), (C.c_int * 4)()
        _lib.check(L.b200trk_net_op_info(eng.handle, i, C.byref(info)), "net_op_info")
        _lib.check(L.b200trk_net_op_io(eng.handle, i, C.byref(io)), "net_op_io")
        info = list(info)
        assert info[0] == 3 and info[7] == 1 and io[2] == 1
        pinfo = (C.c_int * 8)()
        _lib.check(L.b200trk_net_op_info(eng.handle, io[0], C.byref(pinfo)), "net_op_info")
        x = _output(eng, io[0], list(pinfo), S)
        y = _output(eng, i, info, S)
        w, b = _weights(eng, i, info)
        z64, m, zt = _reference(x, w, b, None, 1, 1, True)
        e = float(((y.double() - z64).abs() / m.clamp(min=1e-30)).max())
        et = float(((zt - z64).abs() / m.clamp(min=1e-30)).max())
        K = 9 * info[1]
        assert e <= et / 16 and e <= (K + 2) * 2.0 ** -23 + 2.0 ** -20, (i, e, et)
        ys.append(y.permute(0, 3, 1, 2).double().cpu().numpy())
    # PrRoIPool + fc3_1r + cat + fc34_*r in float64 on the convolutions' own outputs
    rois = np.stack([np.arange(S), boxes[:, 0], boxes[:, 1], boxes[:, 0] + boxes[:, 2], boxes[:, 1] + boxes[:, 3]], 1).astype(np.float64)
    p3 = prroi_oracle.forward(ys[0], rois, 3, 3, 1.0 / 8).reshape(S, -1)
    p4 = prroi_oracle.forward(ys[1], rois, 1, 1, 1.0 / 16).reshape(S, -1)

    def block(name, x):
        q = "bb_regressor." + name
        W = sd[q + ".0.weight"].double().reshape(sd[q + ".0.weight"].shape[0], -1).numpy()
        sc = (sd[q + ".1.weight"].double() / torch.sqrt(sd[q + ".1.running_var"].double() + 1e-5)).numpy()
        z = (x @ W.T + sd[q + ".0.bias"].double().numpy() - sd[q + ".1.running_mean"].double().numpy()) * sc + sd[q + ".1.bias"].double().numpy()
        return np.maximum(z, 0)
    cat = np.concatenate([block("fc3_1r", p3), p4], 1)
    r3, r4 = _rel(m3.cpu().numpy(), block("fc34_3r", cat)), _rel(m4.cpu().numpy(), block("fc34_4r", cat))
    assert r3 <= 1e-5 and r4 <= 1e-5, (r3, r4)
    # repeats bitwise; one box alone, on a permuted batch, gives the same bits
    for _ in range(2):
        a3, a4 = head.get(eng, S, boxes)
        assert torch.equal(a3, m3) and torch.equal(a4, m4)
    perm = [2, 0, 1]
    eng.forward(crops[perm].contiguous(), want=("classification",))
    for r in range(S):
        b3, b4 = head.get(eng, S, boxes[r:r + 1], images=[perm.index(r)])
        assert torch.equal(b3[0], m3[r]) and torch.equal(b4[0], m4[r]), r
    head.close()
    eng.close()
