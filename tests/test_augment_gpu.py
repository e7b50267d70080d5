"""-m gpu tests of the augmented initialisation (b200trk_augment_crops, b200trk_dimp_tracker_initialize_augmented_host,
DiMPTracker(augmentation=...)), against tests/golden/augment.npz (oracle/gen_augment_golden.py, the unmodified reference with cv2 on
the CPU) and oracle/augmentation_ref.py:
  * crops: the expanded patch from the crop kernel and the 13 crops through the C ABI -- identity, translation, flip and rotate equal
    the reference's crops (SHA-256) on the recorded first frames; every crop equals the oracle (the blur its tap-order sums) and the
    blur lies within the float64 bound, for targets at every image border at 288^2 and 352^2; repeats are bitwise;
  * replays: native DiMP-50 with the stock augmentation, with the learnt initialiser and with the zero one, and PrDiMP-50 with the
    learnt initialiser, against the recorded reference runs: initial filter within 1e-4 relative, flags identical and boxes
    bit-identical over 20 frames;
  * refusals: the batch tracker, 'scale' and a network built for too small a batch raise and leave the tracker as it was."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import augmentation_ref as A
from pytracking_b200 import _lib, synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment.npz")


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def device_crops(prefix, frame, bb, seed=0):
    """(patch, crops, transform list) from the crop kernel and b200trk_augment_crops for a first frame and box."""
    from test_augment_cpu import STOCK, params
    from pytracking_b200.tracker import HostLogic, draw_augmentation
    p = params(prefix)
    iss = p.image_sample_size
    torch.manual_seed(seed)
    desc, _ = draw_augmentation(STOCK, iss, 1 / 3, 512)
    hl = HostLogic(p)
    g, _ = hl.init_state_augmented(frame.shape[0], frame.shape[1], bb, desc)
    hl.close()
    g.win_r = g.win_c = 0
    L = _lib.lib()
    im = torch.from_numpy(frame).cuda()
    patch = torch.empty(3, g.out_h, g.out_w, device="cuda")
    T = desc.num_transforms
    crops = torch.empty(T, 3, iss, iss, device="cuda")
    _lib.check(L.b200trk_sample_patch(C.c_void_p(im.data_ptr()), frame.shape[0], frame.shape[1], C.byref(g), g.out_h, g.out_w,
                                      C.c_void_p(patch.data_ptr()), None), "sample_patch")
    _lib.check(L.b200trk_augment_crops(C.c_void_p(patch.data_ptr()), g.out_h, g.out_w, iss, iss, desc.transform, T,
                                       C.c_void_p(crops.data_ptr()), None), "augment_crops")
    torch.cuda.synchronize()
    xf = []
    for k in range(T):
        t = desc.transform[k]
        par = (t.param[0], t.param[1]) if t.kind == 3 else (t.param[0] if t.kind == 4 else None)
        xf.append((t.kind, (t.shift[0], t.shift[1]), par))
    return patch.cpu().numpy(), crops.cpu().numpy(), xf, iss


@pytest.mark.parametrize("prefix", ["dimp_", "prdimp_"])
def test_crops_are_the_reference_crops_on_the_recorded_first_frames(prefix):
    from test_augment_cpu import PARAMS, digest
    d = np.load(GOLDEN)
    frames, bb = synth.make_sequence(PARAMS[prefix], num_frames=1)
    patch, crops, xf, iss = device_crops(prefix, frames[0], bb)
    for k, (kind, shift, par) in enumerate(xf):
        if kind != 3:
            assert digest(crops[k]) == str(d[prefix + "crop_digest"][k]), (prefix, k, kind)
        assert np.array_equal(crops[k], A.transform(patch, kind, shift, par, (iss, iss))), (prefix, k)
        if kind == 3:
            e = np.abs(crops[k].astype(np.float64) - A.crop(A.blur64(patch, par), (iss, iss), shift)).max()
            assert e <= A.blur_bound(patch, par), (prefix, k, e)


BORDER_BOXES = [[0, 0, 60, 40], [600, 10, 40, 50], [5, 440, 70, 40], [590, 430, 50, 50], [300, 0, 30, 20], [0, 220, 25, 90]]


@pytest.mark.parametrize("prefix", ["dimp_", "prdimp_"])
def test_crops_match_oracle_at_every_image_border_and_repeat_bitwise(prefix):
    frames, _ = synth.make_sequence(3, num_frames=1)
    for i, bb in enumerate(BORDER_BOXES):
        patch, crops, xf, iss = device_crops(prefix, frames[0], bb, seed=i)
        for k, (kind, shift, par) in enumerate(xf):
            assert np.array_equal(crops[k], A.transform(patch, kind, shift, par, (iss, iss))), (prefix, bb, k)
        again = device_crops(prefix, frames[0], bb, seed=i)[1]
        assert np.array_equal(again, crops), (prefix, bb)


def _replay(name, make_tracker):
    from pytracking_b200.tracker import FLAGS
    d = np.load(GOLDEN)
    frames, bb = synth.make_sequence(2, num_frames=20)
    trk = make_tracker(d)
    torch.manual_seed(0)
    trk.initialize(frames[0], {"init_bbox": bb})
    torch.cuda.synchronize()
    e_init = _rel(trk.engine.filter.cpu().numpy(), d["track_%s_init_filter" % name])
    assert e_init <= 1e-4, (name, e_init)
    err = []
    for t in range(len(d["track_%s_flag" % name])):
        out = trk.track(frames[t + 1])
        assert trk.info.flag == d["track_%s_flag" % name][t], (name, t, FLAGS[trk.info.flag])
        err.append(float(np.abs(np.array(out["target_bbox"], np.float64) - d["track_%s_bbox" % name][t].astype(np.float64)).max()))
        assert err[-1] == 0.0, (name, t, out["target_bbox"], d["track_%s_bbox" % name][t])
    print("%s with the stock augmentation vs recorded CPU reference: init filter %.2e, %d frames, boxes bit-identical in %d, max "
          "error %.1e px" % (name, e_init, len(err), sum(e == 0.0 for e in err), max(err)))
    trk.close()


def _dimp_tracker(filter_init):
    from test_augment_cpu import STOCK
    from tracker_cases import DIMP50
    from pytracking_b200.tracker import DiMPTracker, make_params
    p = make_params(**dict(DIMP50, target_not_found_threshold=-1e9, train_skipping=20, net_opt_update_iter=2))
    return lambda d: DiMPTracker(synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3), p, filter_init=filter_init,
                                 augmentation=STOCK, random_shift_factor=1 / 3)


def test_native_dimp50_with_stock_augmentation_replays_reference_run():
    _replay("dimp", _dimp_tracker("network"))


def test_native_dimp50_with_stock_augmentation_and_zero_initialiser_replays_reference_run():
    _replay("dimp_zero", _dimp_tracker("zero"))


def test_native_prdimp50_with_stock_augmentation_replays_reference_run():
    from test_augment_cpu import STOCK
    from test_prdimp_host_logic_cpu import prdimp_params
    from pytracking_b200.tracker import DiMPTracker

    def make(d):
        v = dict(zip([str(k) for k in d["prdimp_newton_keys"]], [float(x) for x in d["prdimp_newton_vals"]]))
        newton = dict(feat_stride=v["feat_stride"], gauss_sigma=v["gauss_sigma"], min_filter_reg=v["min_filter_reg"],
                      alpha_eps=v["alpha_eps"], init_uni_weight=v["uni_weight"], normalize_label=bool(v["normalize_label"]),
                      label_shrink=v["label_shrink"], softmax_reg=None if math.isnan(v["softmax_reg"]) else v["softmax_reg"],
                      label_threshold=v["label_threshold"], init_step_length=float(np.exp(d["prdimp_log_step_length"].astype(np.float32))[0]),
                      init_filter_reg=float(d["prdimp_filter_reg"][0]))
        sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
        sd = {k: v for k, v in sd.items() if not k.startswith("classifier.filter_optimizer.")}
        p = prdimp_params(target_not_found_threshold=-1e9, train_skipping=20, net_opt_update_iter=2)
        return DiMPTracker(sd, p, newton=newton, filter_init="network", augmentation=STOCK, random_shift_factor=1 / 3)
    _replay("prdimp", make)


def test_refusals_leave_the_tracker_unchanged():
    from test_augment_cpu import STOCK
    from tracker_cases import DIMP50
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import DiMPTracker, draw_augmentation, make_params
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    p = make_params(**DIMP50)
    with pytest.raises(NotImplementedError):
        DiMPBatchTracker(sd, p, 2, augmentation=STOCK)
    with pytest.raises(NotImplementedError):
        DiMPTracker(sd, p, augmentation=dict(STOCK, scale=[1.1]))
    frames, bb = synth.make_sequence(0, num_frames=2)
    trk = DiMPTracker(sd, p)                      # un-augmented: a network built for batches of 1
    trk.initialize(frames[0], {"init_bbox": bb})
    torch.cuda.synchronize()
    state, filt = trk.state().copy(), trk.engine.filter.clone()
    torch.manual_seed(0)
    desc, mult = draw_augmentation(STOCK, 288, 1 / 3, 512)
    im = torch.from_numpy(frames[1]).contiguous()
    bb2 = (C.c_double * 4)(10, 20, 30, 40)
    L = _lib.lib()
    for mutate in (lambda d: None, lambda d: setattr(d.transform[5], "kind", _lib.AUG_KINDS["scale"])):
        mutate(desc)
        assert L.b200trk_dimp_tracker_initialize_augmented_host(trk.handle, C.c_void_p(im.data_ptr()), 480, 640, C.byref(bb2),
                                                                C.byref(desc), None) != 0
        torch.cuda.synchronize()
        assert np.array_equal(trk.state(), state) and torch.equal(trk.engine.filter, filt)
    trk.close()
