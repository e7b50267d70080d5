"""-m gpu tests of PrDiMP-50 (BASELINE configs[2]) in the native tracker.  They read only committed goldens
(tests/golden/prdimp_host_noaug.npz, recorded by oracle/gen_prdimp_golden.py from the unmodified reference PrDiMP tracker):

  * native initialisation + closed-loop frames from uint8 frames: scalar state bit-identical after initialize, boxes bit-identical (until a
    documented near-tie) and flags identical on every frame up to there, first-frame score map within 1e-4;
  * the same with PrDiMP's IoUNet refinement on a seeded bb_regressor (tests/golden/prdimp_host_iou.npz): flags identical, boxes
    within 1e-2 px;
  * the Newton update on the state's pitched sample memory (NaN padding) at n = 1, 31, 32, 50: padding untouched, filter bitwise equal
    to b200trk_prdimp_sd_newton on a dense copy, the CUDA-core kernel below 32 samples and the tensor-core kernel from 32;
  * 'inside' / 'inside_major' crops from the crop kernel against oracle/preprocessing_modes_ref.py, bit-exact.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PO = "classifier.filter_optimizer."


def prdimp_state_dict():
    """The seeded weights baseline/ref_tracker.build_prdimp loads into klcedimpnet50 (its optimiser keeps the constructor's values)."""
    from pytracking_b200 import synth
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    return {k: v for k, v in sd.items() if not k.startswith((PO, "classifier.filter_initializer."))}


def newton_from_golden(d):
    """PrDiMPSteepestDescentNewton arguments from the hyper-parameters and learnt scalars stored in the golden."""
    v = dict(zip([str(k) for k in d["newton_keys"]], [float(x) for x in d["newton_vals"]]))
    return dict(feat_stride=v["feat_stride"], gauss_sigma=v["gauss_sigma"], min_filter_reg=v["min_filter_reg"], alpha_eps=v["alpha_eps"],
                init_uni_weight=v["uni_weight"], normalize_label=bool(v["normalize_label"]), label_shrink=v["label_shrink"],
                softmax_reg=None if math.isnan(v["softmax_reg"]) else v["softmax_reg"], label_threshold=v["label_threshold"],
                init_step_length=float(np.exp(d["log_step_length"].astype(np.float32))[0]), init_filter_reg=float(d["filter_reg"][0]))


def test_native_prdimp_tracker_reproduces_recorded_reference_run():
    from test_prdimp_host_logic_cpu import prdimp_params, softmax_reg
    from pytracking_b200 import synth
    from pytracking_b200.tracker import DiMPTracker, FLAGS
    d = np.load(os.path.join(GOLDEN, "prdimp_host_noaug.npz"))
    trk = DiMPTracker(prdimp_state_dict(), prdimp_params("noaug"), newton=newton_from_golden(d))
    assert _lib().b200trk_dimp_state_optimizer_kind(trk.engine.state) == 1
    frames, bb = synth.make_sequence(2, num_frames=len(d["flag"]))
    trk.initialize(frames[0], {"init_bbox": bb})
    assert np.array_equal(trk.state(), d["init_state"])
    f_init = trk.engine.filter.cpu().numpy()
    e_init = float(np.abs(f_init - d["init_filter"]).max() / np.abs(d["init_filter"]).max())
    drift, horizon = [], len(d["flag"])
    for t in range(len(d["flag"])):
        out = trk.track(frames[t + 1])
        s = trk.engine.scores[0].cpu().numpy()
        ref_s = d["scores"][t]
        p, p_ref = softmax_reg(s[None], None)[0], softmax_reg(ref_s[None], None)[0]
        if not np.array_equal(np.array(out["target_bbox"], dtype=np.float32), d["bbox"][t]):
            # The acceptance rule of the DiMP closed-loop test (tests/test_tracker_gpu.py), in probabilities: the loop may part only
            # where the recorded run's two best cells are closer than twice the probability-map drift of the preceding frames, and
            # not before frame 10.
            mine, theirs = np.unravel_index(np.argmax(p), p.shape), np.unravel_index(np.argmax(p_ref), p_ref.shape)
            gap = abs(float(p_ref[mine]) - float(p_ref[theirs])) / float(p_ref.max())
            recent = max(drift[-5:])
            print("native PrDiMP leaves the recorded trajectory at frame %d: cells %s / %s, gap %.2e, recent drift %.2e" % (t, mine, theirs, gap, recent))
            assert gap <= 2 * recent, (t, out["target_bbox"], d["bbox"][t], FLAGS[trk.info.flag], gap, recent)
            horizon = t
            break
        assert trk.info.flag == d["flag"][t], (t, FLAGS[trk.info.flag], int(d["flag"][t]))
        if t == 0:      # debug_info['max_score'] is the probability, as the reference reports it
            assert abs(trk.debug_info["max_score"] - d["max_score"][0]) <= 1e-4 * d["max_score"][0]
            assert float(np.abs(s - ref_s).max() / np.abs(ref_s).max()) <= 1e-4
        drift.append(float(np.abs(p - p_ref).max() / p_ref.max()))
    assert horizon >= 10, horizon
    print("native PrDiMP vs recorded CPU reference: init filter %.2e, probability-map rel. diff frame 1 %.2e, median %.2e, max %.2e, "
          "frames %d" % (e_init, drift[0], float(np.median(drift)), max(drift), horizon))
    trk.close()


def test_native_prdimp_tracker_with_iounet_matches_recorded_reference_run():
    """PrDiMP's IoUNet refinement (relative box space, 10 steps of 2.5e-3, top-3 mean of the classifier box and 9 jittered proposals) on
    the seeded bb_regressor, native initialisation, closed loop from uint8 frames, against the reference run recorded on the CPU
    (tests/golden/prdimp_host_iou.npz, with the proposal noise and the first-frame modulation vectors it used): flags identical, boxes
    within 1e-2 px."""
    import sys
    from test_prdimp_host_logic_cpu import prdimp_params
    from pytracking_b200 import synth
    from pytracking_b200.tracker import DiMPTracker, FLAGS
    sys.path.insert(0, os.path.dirname(__file__))
    import ref_weights
    d = np.load(os.path.join(GOLDEN, "prdimp_host_iou.npz"))
    iters, step, k, nrand, relative = [float(v) for v in d["refine_params"]]
    assert (iters, step, k, nrand, relative) == (10, 2.5e-3, 3, 9, 1)
    sd = prdimp_state_dict()
    sd.update(ref_weights.seeded_state_dict(d["iou_keys"], d["iou_shapes"], 5, prefix="bb_regressor."))
    sd["bb_regressor.iou_predictor.weight"] = sd["bb_regressor.iou_predictor.weight"] * 20.0
    params = prdimp_params("noaug", use_iou_net=True, iounet_k=3, num_init_random_boxes=9, box_jitter_pos=0.1, box_jitter_sz=0.5,
                           maximal_aspect_ratio=6, box_refinement_iter=10, box_refinement_step_length=2.5e-3,
                           box_refinement_step_decay=1, box_refinement_space="relative")
    trk = DiMPTracker(sd, params, newton=newton_from_golden(d))
    frames, bb = synth.make_sequence(2, num_frames=len(d["flag"]))
    trk.initialize(frames[0], {"init_bbox": bb})
    assert np.array_equal(trk.state(), d["init_state"])
    trk.attach_iounet(sd, [torch.from_numpy(d["modulation3"]), torch.from_numpy(d["modulation4"])])
    L = _lib()
    err = []
    for t in range(len(d["flag"])):
        u = np.ascontiguousarray(d["noise"][t], dtype=np.float32)
        from pytracking_b200 import _lib as Lmod
        Lmod.check(L.b200trk_dimp_tracker_set_proposal_noise(trk.handle, u.ctypes.data_as(C.c_void_p), u.size), "set_proposal_noise")
        out = trk.track(frames[t + 1])
        assert trk.info.flag == d["flag"][t], (t, FLAGS[trk.info.flag], int(d["flag"][t]))
        assert trk.info.refined == 1, t
        err.append(float(np.abs(np.array(out["target_bbox"], dtype=np.float64) - d["bbox"][t].astype(np.float64)).max()))
        assert err[-1] < 1e-2, (t, out["target_bbox"], d["bbox"][t])
    print("native PrDiMP + IoUNet vs recorded CPU reference: %d frames, box error median %.1e px, max %.1e px"
          % (len(err), float(np.median(err)), max(err)))
    trk.close()


def _lib():
    from pytracking_b200 import _lib as L
    return L.lib()


@pytest.fixture(scope="module")
def engine():
    from pytracking_b200.frame_engine import DiMPFrameEngine
    d = np.load(os.path.join(GOLDEN, "prdimp_host_noaug.npz"))
    eng = DiMPFrameEngine(prdimp_state_dict(), arch="resnet50", filter_size=4, memory_size=50, max_batch=1, crop_size=352,
                          newton=newton_from_golden(d))
    yield eng
    eng.close()


@pytest.mark.parametrize("n", [1, 31, 32, 50])
def test_newton_update_on_pitched_sample_memory(engine, monkeypatch, n):
    from pytracking_b200 import ops, synth
    from pytracking_b200.frame_engine import _view
    monkeypatch.delenv("B200TRK_SD_TC", raising=False)
    eng, L = engine, _lib()
    cc, hc, wc = eng.feat_dims
    assert (cc, hc, wc) == (512, 22, 22)
    pitch = L.b200trk_dimp_state_memory_pitch(eng.state)
    assert pitch == 512 and pitch > hc * wc
    raw = _view(L.b200trk_dimp_state_memory(eng.state), (eng.memory_size * cc * pitch,), eng, eng.device)
    pad = raw.view(eng.memory_size, cc, pitch)[:, :, hc * wc:]
    seed = 11 * n
    raw.fill_(float("nan"))
    eng.memory.copy_(synth.make_clf_features(seed, eng.memory_size, cc, hc, wc).cuda())
    eng.boxes.copy_(synth.make_boxes(seed + 1, eng.memory_size, center=(hc * 16) / 2 - 25).cuda())
    g = torch.Generator().manual_seed(seed + 2)
    w0 = (0.01 * torch.randn(1, cc, 4, 4, generator=g)).cuda()
    sw = (torch.rand(n, generator=g) + 0.5).numpy().astype(np.float32)
    sw /= sw.sum(dtype=np.float32)
    crop = synth.make_crop(seed + 3, 1, 352).pin_memory()
    target_box = synth.make_boxes(seed + 4, 1, center=(hc * 16) / 2 - 25)[0].numpy()
    eng.localize(crop)
    eng.filter.copy_(w0)
    eng.update(0, n // 2, target_box, sw, n, 10)           # the crop's feature into slot n // 2 (pitched rows), then 10 Newton steps
    torch.cuda.synchronize()
    expect_tc = 1 if n >= 32 else 0
    assert L.b200trk_sd_last_kernel() == expect_tc
    w = eng.filter.clone()
    assert bool(torch.isnan(pad).all()), "the padding of the sample memory was written"
    assert bool(torch.isfinite(w).all()), "non-finite filter (the pitch padding was read)"
    nw = eng.newton
    feat = eng.memory[:n].contiguous()
    w_dense, _, _ = ops.prdimp_sd_newton(w0, feat, eng.boxes[:n].clone(), eng.sample_weights[:n].clone(), 10, nw["gauss_sigma"],
                                         eng.step_length, eng.reg_weight, nw["alpha_eps"], nw["softmax_reg"], nw["label_threshold"],
                                         nw["normalize_label"], nw["label_shrink"], nw["init_uni_weight"] or 0.0, nw["feat_stride"])
    torch.cuda.synchronize()
    assert L.b200trk_sd_last_kernel() == expect_tc
    assert torch.equal(w, w_dense), "pitched and dense sample memory give different filters (n=%d)" % n


def test_inside_crops_from_the_crop_kernel_bit_exact():
    from test_prdimp_host_logic_cpu import crop_cases
    from oracle import preprocessing_modes_ref as PM
    from pytracking_b200 import _lib as Lmod
    L = _lib()
    rng = np.random.RandomState(3)
    torch.set_num_threads(8)
    n = 0
    for H, W, bb, mode, msc, hl, g, st in crop_cases():
        img = np.ascontiguousarray(rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
        sz = torch.tensor([352.0, 352.0])
        ref, _ = PM.sample_patch(PM.R.numpy_to_torch(img), torch.tensor([st[0], st[1]]), torch.tensor(st[4]) * sz, sz, mode, msc)
        im_dev = torch.from_numpy(img).cuda()
        out = torch.empty(3, 352, 352, device="cuda")
        Lmod.check(L.b200trk_sample_patch(C.c_void_p(im_dev.data_ptr()), H, W, C.byref(g), 352, 352, C.c_void_p(out.data_ptr()),
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)), "sample_patch")
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), ref[0]), (H, W, bb, mode, msc, int((out.cpu() != ref[0]).sum()))
        hl.close()
        n += 1
    assert n == 48
