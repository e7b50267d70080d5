"""-m gpu tests of the learnt filter initialiser (FilterInitializerLinear: b200trk_net_attach_filter_init / b200trk_net_filter_init, and
the trackers' filter_init="network"), against tests/golden/filter_init.npz (oracle/gen_filter_init_golden.py, the unmodified reference on
the CPU) and float64:
  * goldens: the filter from the golden's classification features within 1e-4 relative of the reference, at precision 0 and 1;
  * float64: filter_conv on the operands it read (criteria of tests/test_tc_conv_layers_gpu.py), the import step an exact transpose, and
    PrRoIPool + mean within 1e-5 of float64 on the convolution's output;
  * determinism: repeats bitwise; permuting the images (with the boxes' image indices) leaves every per-box filter bitwise the same;
  * trackers: DiMPTracker(filter_init="network") replays the reference DiMP run without filter_init_zero; the batch at capacity 1
    equals the solo tracker bit for bit, and at capacity 4 batch-mates change no bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytracking_b200 import _lib, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "filter_init.npz")
OP_CONV, OP_NCHW_IMPORT = 3, 6


def _sd():
    return synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)


def _engine(sd, crop, norm=0, square=0, precision=0, max_batch=3):
    from pytracking_b200.engine import BackboneEngine
    eng = BackboneEngine(sd, "resnet50", 4, max_batch, crop, precision)
    eng.attach_filter_init(sd, 4, norm, square)
    return eng


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("precision", [0, 1])
def test_filter_matches_reference_golden(precision):
    from test_filter_init_cpu import golden_cases
    sd = _sd()
    engines, worst = {}, 0.0
    for seed, S, H, norm, square, boxes, ref in golden_cases():
        key = (H, norm, square)
        if key not in engines:
            engines[key] = _engine(sd, 16 * H, norm, square, precision)
        feat = synth.make_clf_features(seed, S, 512, H, H).cuda()
        w = engines[key].filter_init(feat, boxes).cpu().numpy()
        e = _rel(w, ref)
        assert e <= 1e-4, (precision, seed, S, H, norm, square, e)
        worst = max(worst, e)
    for eng in engines.values():
        eng.close()
    print("filter initialiser vs reference, precision %d: worst relative difference %.2e" % (precision, worst))


def _step(eng, kind):
    L = _lib.lib()
    for i in range(L.b200trk_net_num_ops(eng.handle)):
        info = (C.c_int * 8)()
        _lib.check(L.b200trk_net_op_info(eng.handle, i, C.byref(info)), "net_op_info")
        if info[0] == kind and (kind != OP_CONV or i == L.b200trk_net_num_ops(eng.handle) - 1):
            return i, list(info)
    raise AssertionError("no plan step of kind %d" % kind)


@pytest.mark.parametrize("precision,H,S", [(0, 18, 1), (0, 22, 3), (1, 18, 3)])
def test_layers_against_float64(precision, H, S):
    from test_tc_conv_layers_gpu import _output, _reference, _weights, _grid
    from oracle import filter_init_oracle as O, prroi_oracle
    sd = _sd()
    eng = _engine(sd, 16 * H, precision=precision)
    L = _lib.lib()
    feat = synth.make_clf_features(7 + S, S, 512, H, H).cuda()
    boxes = np.array([[0.3, 0.35, 0.25, 0.2], [-0.08, 0.4, 0.2, 0.15], [0.9, 0.2, 0.2, 0.3]][:S], np.float32) * 16 * H
    w = eng.filter_init(feat, boxes)
    torch.cuda.synchronize()
    ii, iinfo = _step(eng, OP_NCHW_IMPORT)
    ci, cinfo = _step(eng, OP_CONV)
    io = (C.c_int * 4)()
    _lib.check(L.b200trk_net_op_io(eng.handle, ci, C.byref(io)), "net_op_io")
    assert io[0] == ii and io[1] == -1 and io[2] == 0 and io[3] == 1
    assert cinfo[7] == (1 if precision == 0 else 0)
    x = _output(eng, ii, iinfo, S)
    assert torch.equal(x, feat.permute(0, 2, 3, 1)), "the import step is not an exact NCHW -> NHWC copy"
    y = _output(eng, ci, cinfo, S)
    wt, b = _weights(eng, ci, cinfo)
    z64, m, zt = _reference(x, wt, b, None, 1, 1, False)
    e = float(((y.double() - z64).abs() / m.clamp(min=1e-30)).max())
    e_tf32 = float(((zt - z64).abs() / m.clamp(min=1e-30)).max())
    K = 9 * 512
    assert e <= (K + 2) * 2.0 ** -23 + 2.0 ** -20, (e, K)
    if precision == 0:
        assert e <= e_tf32 / 16, (e, e_tf32)
        assert _grid(eng, ci)[0] >= 1
    # PrRoIPool + mean on the convolution's own output, against float64
    conv = y.permute(0, 3, 1, 2).double().cpu().numpy()
    w64 = prroi_oracle.forward(conv, O.rois(boxes), 4, 4, 1.0 / 16).mean(0, keepdims=True)
    assert _rel(w.cpu().numpy(), w64) <= 1e-5, _rel(w.cpu().numpy(), w64)
    eng.close()


def test_deterministic_and_independent_of_image_order():
    sd = _sd()
    eng = _engine(sd, 352, max_batch=4)
    feat = synth.make_clf_features(5, 4, 512, 22, 22).cuda()
    boxes = np.array([[100, 120, 80, 60], [-20, 150, 70, 50], [300, 10, 60, 100], [40, 330, 120, 30]], np.float32)
    a = eng.filter_init(feat, boxes).clone()
    for _ in range(3):
        assert torch.equal(eng.filter_init(feat, boxes), a)
    perm = [2, 0, 3, 1]
    fp = feat[perm].contiguous()
    inv = [perm.index(i) for i in range(4)]           # image i now sits at position inv[i]
    for r in range(4):
        solo = eng.filter_init(feat, boxes[r:r + 1], images=[r]).clone()
        moved = eng.filter_init(fp, boxes[r:r + 1], images=[inv[r]])
        assert torch.equal(solo, moved), r
    eng.close()


def _dimp_params():
    from tracker_cases import DIMP50, OVERRIDES
    from pytracking_b200.tracker import make_params
    return make_params(**dict(DIMP50, **OVERRIDES["noaug"]))


def test_native_tracker_with_learnt_initialiser_replays_reference_run():
    from pytracking_b200.tracker import DiMPTracker, FLAGS
    d = np.load(GOLDEN)
    trk = DiMPTracker(_sd(), _dimp_params(), filter_init="network")
    frames, bb = synth.make_sequence(2, num_frames=20)
    assert len(frames) - 1 == len(d["track_flag"])
    trk.initialize(frames[0], {"init_bbox": bb})
    assert np.array_equal(trk.state(), d["track_init_state"])
    e_init = _rel(trk.engine.filter.cpu().numpy(), d["track_init_filter"])
    assert e_init <= 1e-4, e_init
    err = []
    for t in range(len(d["track_flag"])):
        out = trk.track(frames[t + 1])
        assert trk.info.flag == d["track_flag"][t], (t, FLAGS[trk.info.flag], int(d["track_flag"][t]))
        err.append(float(np.abs(np.array(out["target_bbox"], np.float64) - d["track_bbox"][t].astype(np.float64)).max()))
        assert err[-1] < 1e-2, (t, out["target_bbox"], d["track_bbox"][t])
    print("native DiMP-50 with the learnt initialiser vs recorded CPU reference: init filter %.2e, %d frames, box error median %.1e px, "
          "max %.1e px" % (e_init, len(err), float(np.median(err)), max(err)))
    trk.close()


def _batch_run(capacity, slot, frames, bb, mates=None):
    """Boxes and the filter after initialize of the sequence in `slot`; `mates` {slot: (frames, bb)} run alongside."""
    from pytracking_b200.batch import DiMPBatchTracker
    b = DiMPBatchTracker(_sd(), _dimp_params(), capacity, filter_init="network")
    mates = mates or {}
    boxes, f0 = [], None
    for t in range(len(frames)):
        step = {slot: (frames[t], {"init_bbox": bb} if t == 0 else None)}
        for s, (mf, mb) in mates.items():
            step[s] = (mf[t], {"init_bbox": mb} if t == 0 else None)
        out = b.step(step)
        if t == 0:
            torch.cuda.synchronize()
            f0 = b.filter(slot).clone()
        boxes.append(out[slot]["target_bbox"])
    torch.cuda.synchronize()
    b.close()
    return np.array(boxes, np.float32), f0


def test_batch_with_learnt_initialiser_is_bitwise_solo_and_independent_of_mates():
    from pytracking_b200.tracker import DiMPTracker
    frames, bb = synth.make_sequence(2, num_frames=8)
    trk = DiMPTracker(_sd(), _dimp_params(), filter_init="network")
    trk.initialize(frames[0], {"init_bbox": bb})
    torch.cuda.synchronize()
    f_solo = trk.engine.filter.clone()
    solo = [list(bb)] + [trk.track(f)["target_bbox"] for f in frames[1:]]
    trk.close()
    b1, f1 = _batch_run(1, 0, frames, bb)
    assert torch.equal(f1, f_solo)
    assert np.array_equal(b1[1:], np.array(solo, np.float32)[1:])
    alone, fa = _batch_run(4, 2, frames, bb)
    mates = {s: synth.make_sequence(s + 3, num_frames=8) for s in (0, 1, 3)}
    together, ft = _batch_run(4, 2, frames, bb, mates)
    assert torch.equal(fa, ft)
    assert np.array_equal(alone, together)
