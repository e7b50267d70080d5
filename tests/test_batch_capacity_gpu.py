"""-m gpu: the lock-step batch (pytracking_b200/batch.py, b200trk_dimp_batch_*) where test_batch_tracker_gpu does not take it:
  * capacity 16 with frames of six sizes in one step -- among them 241x323, 199x257 and 97x131, whose H*W*3 bytes are not a
    multiple of 256, so the frame uploader packs every later frame at a rounded-up offset -- given as numpy arrays, pinned tensors and
    pageable tensors in the same step, then as CUDA tensors (the device entry): every item's crop, the init step's windowed 576^2
    crop included, equals `b200trk_sample_patch` on that frame with the crop geometry the step reports, and torch-CPU bilinear
    resampling of the reference's sample_patch, bit for bit;
  * scores at capacity 16 (DiMP-50, 288^2) and at capacity 4 and 16 (PrDiMP-50, 352^2, softmax localisation) within 1e-4 relative of
    a solo engine given the same crop and filter, with the same arg-max cell (test_batch_tracker_gpu's method; 1e-4 is DESIGN 2's
    score-map tolerance);
  * at capacity 16 each tracked slot's localisation result equals, byte for byte, `b200trk_dimp_localize` on the slot's score map
    with neigh / prev_vec derived from the slot's state before the step and the step's crop geometry;
  * PrDiMP-50 at capacity 4: a sequence's bits do not depend on its batch-mates, and closed-loop boxes stay within 0.5 px of solo
    trackers on the stock schedule (DESIGN 4.10's bar for DiMP-50; test_batch_tracker_gpu's helpers, run on the PrDiMP configuration)."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib, synth
from test_batch_tracker_gpu import (BENCH, PRDIMP, STOCK, _batch, _solo, check_batch_mates_do_not_change_a_sequence,
                                    check_closed_loop_within_half_a_pixel_of_solo)
from test_tracker_gpu import _run_localize

pytestmark = pytest.mark.gpu

PRDIMP_STOCK = dict(PRDIMP, train_skipping=20, net_opt_update_iter=2)
# 16 slots; the odd sizes come first so that every later frame of the step sits behind a rounded-up offset
SIZES = [(241, 323), (480, 640), (97, 131), (720, 1280), (1080, 1920), (199, 257), (240, 320), (480, 640), (97, 131), (241, 323),
         (720, 1280), (240, 320), (1080, 1920), (199, 257), (480, 640), (97, 131)]
HOST_KINDS = ("numpy", "pinned", "pageable")


def _sequence(q, n, hw):
    """(uint8 frames, init box) of synthetic sequence q at frame size hw (the init box is the target's, inside the frame)."""
    frames, _ = synth.make_sequence(q, n, *hw)
    return frames, synth.sequence_ground_truth(q, n, *hw)[0]


def _as(frame, kind):
    if kind == "numpy":
        return frame
    t = torch.from_numpy(frame)
    return {"pinned": lambda: t.pin_memory(), "pageable": lambda: t, "cuda": lambda: t.cuda()}[kind]()


def _info(bt, slot):
    """A copy of the slot's FrameInfo (bt.last_info holds views of the batch's result array, which the next step overwrites)."""
    return _lib.FrameInfo.from_buffer_copy(bytes(bt.last_info[slot]))


def _check_crop(bt, slot, frame, info, st, init):
    """The slot's crop of this step against b200trk_sample_patch and torch-CPU bilinear, bitwise. st: the slot's state the crop was
    planned from (after init_state for an init item, before the step for a tracked one)."""
    from oracle import preprocessing_ref as R
    iss = bt.params.image_sample_size
    H, W = frame.shape[:2]
    g = info.crop
    mine = bt.crop(slot).clone()
    dev = torch.from_numpy(frame).cuda()
    one = torch.empty(3, iss, iss, device="cuda")
    _lib.check(_lib.lib().b200trk_sample_patch(C.c_void_p(dev.data_ptr()), H, W, C.byref(g), iss, iss, C.c_void_p(one.data_ptr()),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream)), "sample_patch")
    torch.cuda.synchronize()
    assert torch.equal(mine, one), "slot %d (%dx%d, init %d): batch crop differs from sample_patch on the same geometry" % (slot, H, W, init)
    im = R.numpy_to_torch(frame)
    sz = torch.tensor([float(iss), float(iss)])
    if init:
        ef = bt.params.augmentation_expansion_factor
        assert g.out_h == 2 * iss and g.win_r == iss // 2, "the init crop is not the windowed expanded patch"
        ref = R.sample_init_patch(im, torch.tensor([st[0], st[1]]).round(), torch.tensor(st[4]), sz, ef)
    else:
        ref, coord = R.sample_patch(im, torch.tensor([st[0], st[1]]), torch.tensor(st[4]) * sz, sz)
        assert np.array_equal(np.array(g.coord, dtype=np.float32), coord.numpy().reshape(4)), slot
    assert torch.equal(mine.cpu(), ref[0]), "slot %d (%dx%d, init %d): batch crop differs from torch-CPU bilinear" % (slot, H, W, init)


def _run_mixed(bt, q0, kinds, n):
    """Starts one sequence per slot (sizes SIZES, frame container per slot from `kinds`) and tracks n frames, checking every crop."""
    seqs = {s: _sequence(q0 + s, n, SIZES[s]) for s in range(bt.capacity)}
    for t in range(n + 1):
        before = {s: bt.state(s) for s in seqs} if t else None
        bt.step({s: (_as(seqs[s][0][t], kinds[s]), {"init_bbox": seqs[s][1]} if t == 0 else None) for s in seqs})
        for s in seqs:
            st = bt.state(s) if t == 0 else before[s]
            _check_crop(bt, s, seqs[s][0][t], _info(bt, s), st, t == 0)


def test_capacity_16_mixed_frame_sizes_and_containers():
    bt = _batch(16, BENCH)
    try:
        _run_mixed(bt, 0, [HOST_KINDS[s % 3] for s in range(16)], 2)      # host entry: pinned and pageable frames in one step
        for s in range(16):
            bt.release(s)
        _run_mixed(bt, 100, ["cuda"] * 16, 2)                             # device entry
    finally:
        bt.close()


def _loc_inputs(bt, st, g):
    """neigh / prev_vec of localize_target for a slot whose state before the step was st and whose crop geometry is g, in the float32
    order of the host (loc_inputs, dimp_tracker.cu; test_batch_kernels_cpu._trajectory_problems)."""
    fs, iss = bt.feat_dims[1], bt.params.image_sample_size
    neigh = [np.float32(np.float32(bt.params.target_neighborhood_scale) * (st[2 + i] / np.float32(g.sample_scale))) * np.float32(fs / iss)
             for i in range(2)]
    pv = [(st[i] - np.float32(g.sample_pos[i])) / (np.float32(iss // fs) * np.float32(g.sample_scale)) for i in range(2)]
    return neigh, pv


@pytest.mark.parametrize("kind,capacity", [("dimp", 16), ("prdimp", 4), ("prdimp", 16)])
def test_scores_match_solo_and_localisation_matches_single_kernel(kind, capacity):
    cfg, newton = (STOCK, None) if kind == "dimp" else (PRDIMP_STOCK, {})
    n = 8
    bt = _batch(capacity, cfg, newton)
    solo = _solo(cfg, newton)
    eng = solo.engine
    try:
        seqs = [synth.make_sequence(q, n) for q in range(capacity)]
        bt.step({s: (seqs[s][0][0], {"init_bbox": seqs[s][1]}) for s in range(capacity)})
        worst, flags = 0.0, set()
        for t in range(1, n + 1):
            filters = [bt.filter(s).clone() for s in range(capacity)]
            states = [bt.state(s) for s in range(capacity)]
            bt.step({s: (seqs[s][0][t], None) for s in range(capacity)})
            for s in range(capacity):
                info = _info(bt, s)
                if capacity == 16:
                    neigh, pv = _loc_inputs(bt, states[s], info.crop)
                    one = _run_localize(bt.scores(s)[None], bt.params, [neigh], [pv])
                    assert bytes(one) == bytes(info.loc), (kind, t, s, one.flag, info.loc.flag)
                    flags.add(int(info.loc.flag))
                eng.filter.copy_(filters[s])
                eng.localize_device(bt.crop(s)[None].contiguous())
                ref, mine = eng.scores[0].float().cpu(), bt.scores(s).float().cpu()
                err = float((mine - ref).abs().max() / ref.abs().max())
                worst = max(worst, err)
                assert err <= 1e-4, (kind, capacity, t, s, err)
                assert int(mine.argmax()) == int(ref.argmax()), (kind, capacity, t, s)
        print("%s capacity %d: worst relative score difference vs solo %.3g; localisation flags %s" % (kind, capacity, worst, sorted(flags)))
    finally:
        solo.close()
        bt.close()


def test_prdimp_batch_mates_do_not_change_a_sequence():
    check_batch_mates_do_not_change_a_sequence(PRDIMP, {})


def test_prdimp_closed_loop_stock_schedule_within_half_a_pixel_of_solo():
    d = check_closed_loop_within_half_a_pixel_of_solo(PRDIMP_STOCK, {})
    print("PrDiMP capacity 4, stock schedule: largest box difference vs solo %.3g px" % d)
