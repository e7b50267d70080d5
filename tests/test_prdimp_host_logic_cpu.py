"""PrDiMP-50 (BASELINE configs[2]) in the native tracker, on the CPU: the host half (csrc/dimp_tracker.cu) with border_mode 'inside' /
'inside_major' and the localisation kernel (csrc/dimp_tracker_kernels.cuh) with the softmax score pre-processing, against the
UNMODIFIED reference PrDiMP tracker recorded by oracle/gen_prdimp_golden.py and against oracle/preprocessing_modes_ref.py.

Torch's CPU exp is not bit-equal to expf, so probabilities are compared to a relative 2e-6 and decisions (cells, flags, use_second) exactly,
except at a near-tie: two cells, or a maximum and a threshold, closer than that tolerance, where either answer is admissible."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib
from pytracking_b200.tracker import HostLogic, make_params

from tracker_cases import GOLDEN, _loc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROB_RTOL = 2e-6
# pytracking/parameter/dimp/prdimp50.py (use_iou_net off) + the BASELINE configs[2] overrides of baseline/ref_tracker.build_prdimp
PRDIMP50 = dict(image_sample_size=352, search_area_scale=6, border_mode="inside_major", patch_max_scale_change=1.5, sample_memory_size=50,
                learning_rate=0.01, init_samples_minimum_weight=0.25, train_skipping=1, update_classifier=True, net_opt_iter=10,
                net_opt_update_iter=10, net_opt_hn_iter=1, advanced_localization=True, score_preprocess="softmax",
                target_not_found_threshold=-1e9, distractor_threshold=0.8, hard_negative_threshold=0.5, target_neighborhood_scale=2.2,
                dispalcement_scale=0.8, hard_negative_learning_rate=0.02, update_scale_when_uncertain=True,
                augmentation_expansion_factor=2, use_iou_net=False)
PRDIMP_OVERRIDES = {
    "noaug": dict(net_opt_update_iter=2),
    "stress": dict(target_not_found_threshold=0.0052, uncertain_threshold=0.00535, hard_sample_threshold=0.0055, distractor_threshold=0.3,
                   hard_negative_threshold=0.2, train_skipping=3, sample_memory_size=12, net_opt_update_iter=2, dispalcement_scale=0.25,
                   search_area_scale=12),
}


def prdimp_params(name=None, **kw):
    return make_params(**dict(PRDIMP50, **(PRDIMP_OVERRIDES[name] if name else {}), **kw))


@pytest.mark.parametrize("name", ["noaug", "stress"])
def test_prdimp_host_logic_replays_reference_trajectory(name):
    d = np.load(os.path.join(GOLDEN, "prdimp_host_%s.npz" % name))
    hl = HostLogic(prdimp_params(name))
    H, W = [int(v) for v in d["image_hw"]]
    if name == "noaug":
        g, box = hl.init_state(H, W, d["init_bbox"])        # 'inside_major' leaves the initial sample alone (dimp.py:332-350)
        assert np.array_equal(hl.state(), d["init_state"])
        assert np.array_equal(box, d["init_target_box"])
        assert (g.out_h, g.win_r, g.win_c) == (704, 176, 176)
        assert np.array_equal(np.array(g.sample_pos), d["init_sample_pos"]) and np.float32(g.sample_scale) == d["init_sample_scale"]
    else:
        hl.adopt(H, W, d["init_state"], d["init_sw"], d["init_counts"][0], d["init_counts"][1])
    max_sw_err = 0.0
    for t in range(len(d["flag"])):
        g = hl.plan_crop()
        assert np.array_equal(np.array(g.coord, dtype=np.float32), d["coord"][t]), (name, t, list(g.coord), d["coord"][t])
        info, sw = hl.commit(g, _loc(d, t))
        assert np.array_equal(np.array(info.bbox, dtype=np.float32), d["bbox"][t]), (name, t)
        assert np.array_equal(hl.state()[:5], d["state"][t]), (name, t)
        assert info.updated == d["updated"][t], (name, t)
        if info.updated:
            assert info.replace_ind == d["replace_ind"][t], (name, t)
            assert np.array_equal(np.array(info.target_box, dtype=np.float32), d["target_box"][t]), (name, t)
            assert np.float32(info.learning_rate) == np.float32(d["lr"][t])
            max_sw_err = max(max_sw_err, float(np.abs(sw - d["sw"][t]).max() / d["sw"][t].max()))
        assert info.num_iter == d["num_iter"][t], (name, t, info.num_iter, d["num_iter"][t])
        if info.num_iter:
            assert info.n_stored == d["n_stored"][t]
    assert max_sw_err < 2e-6, max_sw_err
    if name == "stress":       # the memory wraps around and train_skipping > 1 skips optimiser runs
        assert (d["replace_ind"][d["updated"] == 1] < d["replace_ind"].max()).sum() > 12 and (d["num_iter"][d["updated"] == 1] == 0).any()
    hl.close()


# (H, W, init_bbox, search_area_scale): shifts off each border, shrink below / clamped at 1.5, df > 1, a sample larger than a 240x320 frame
CROP_CASES = [
    (480, 640, [2, 200, 60, 50], 6), (480, 640, [600, 200, 60, 50], 6), (480, 640, [300, 3, 60, 50], 6), (480, 640, [300, 440, 60, 50], 6),
    (480, 640, [300, 200, 80, 70], 8.5), (480, 640, [300, 200, 120, 100], 9), (480, 640, [250, 150, 150, 130], 12),
    (1080, 1920, [900, 500, 300, 200], 6), (1080, 1920, [20, 1000, 600, 500], 6), (240, 320, [150, 100, 50, 40], 6),
    (240, 320, [5, 5, 80, 60], 10), (240, 320, [300, 200, 30, 30], 20),
]


def crop_cases():
    """-> (H, W, bb, mode, max_scale_change, HostLogic after init, crop request, tracker state) for both inside modes on every case,
    with patch_max_scale_change 1.5 (PrDiMP) and None (no upper clamp on the shrink factor)."""
    for msc in (1.5, None):
        for mode in ("inside_major", "inside"):
            for (H, W, bb, sas) in CROP_CASES:
                kw = dict(search_area_scale=sas, augmentation_expansion_factor=None, patch_max_scale_change=msc)
                hl = HostLogic(prdimp_params(border_mode=mode, **kw))
                if mode == "inside":              # the native initialisation refuses 'inside'; set the scalars of an inside_major init
                    ini = HostLogic(prdimp_params(**kw))
                    ini.init_state(H, W, bb)
                    hl.adopt(H, W, ini.state(), np.ones(50, np.float32), 1, 1)
                    ini.close()
                else:
                    hl.init_state(H, W, bb)
                yield H, W, bb, mode, msc, hl, hl.plan_crop(), hl.state()


def test_inside_crop_geometry_edge_cases():
    from oracle import preprocessing_modes_ref as PM
    seen = set()
    for H, W, bb, mode, msc, hl, g, st in crop_cases():
        im = torch.zeros(1, 3, H, W)
        sz = torch.tensor([352.0, 352.0])
        pos, scale = torch.tensor([st[0], st[1]]), torch.tensor(st[4])
        ref = PM.sample_patch_geometry(im, pos, scale * sz, sz, mode, msc)
        assert (g.df, g.os_r, g.os_c, g.tl_r, g.tl_c, g.in_h, g.in_w) == ref[:7], ((H, W, bb, mode, msc), ref)
        assert np.array_equal(np.array(g.coord, dtype=np.float32), ref[7].numpy().reshape(4)), (H, W, bb, mode, msc)
        # what the case exercised: shift off a border, shrink (clamped or not), decimation, centring of an oversized sample
        full = float(st[4]) * 352
        shrink = max(full / H, full / W) if mode == "inside" else min(full / H, full / W)
        seen.add(("shrink_clamped" if msc else "shrink_unclamped") if shrink > 1.5 else "shrink" if shrink > 1 else "no_shrink")
        if g.df > 1:
            seen.add("df")
        if g.tl_r < 0 or g.tl_c < 0:
            seen.add("centred")
        hl.close()
    assert {"shrink_clamped", "shrink_unclamped", "shrink", "no_shrink", "df", "centred"} <= seen, seen


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("prdimp_emul")), "libprdimp_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", "prdimp_emul.cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


def test_inside_crops_from_the_kernel_source_bit_exact(emul):
    from oracle import preprocessing_modes_ref as PM
    rng = np.random.RandomState(3)
    for H, W, bb, mode, msc, hl, g, st in crop_cases():
        img = np.ascontiguousarray(rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
        sz = torch.tensor([352.0, 352.0])
        ref, _ = PM.sample_patch(PM.R.numpy_to_torch(img), torch.tensor([st[0], st[1]]), torch.tensor(st[4]) * sz, sz, mode, msc)
        out = np.empty((3, 352, 352), np.float32)
        assert emul.prdimp_emul_sample_patch(img.ctypes.data_as(C.c_void_p), H, W, C.byref(g), 352, 352, out.ctypes.data_as(C.c_void_p)) == 0
        assert torch.equal(torch.from_numpy(out), ref[0]), (H, W, bb, mode)
        hl.close()


def _localize(emul, scores, params, neigh, pv):
    s = np.ascontiguousarray(scores, dtype=np.float32)
    n, p = np.ascontiguousarray(neigh, dtype=np.float32), np.ascontiguousarray(pv, dtype=np.float32)
    res = _lib.LocResult()
    assert emul.prdimp_emul_localize(s.ctypes.data_as(C.c_void_p), s.shape[0], s.shape[1], s.shape[2], C.byref(params),
                                     n.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p), C.byref(res)) == 0
    return res


def softmax_reg(scores, reg):
    """activation.softmax_reg over the whole map of each scale (float64, for the tie analysis only)."""
    x = scores.reshape(scores.shape[0], -1).astype(np.float64)
    m = x.max(axis=1, keepdims=True) if reg is None else np.maximum(x.max(axis=1, keepdims=True), reg)
    e = np.exp(x - m)
    den = e.sum(axis=1, keepdims=True) + (0.0 if reg is None else np.exp(reg - m))
    return (e / den).reshape(scores.shape)


def near_tie(p, thresholds, m1):
    """True when the second-largest probability of the map, or a threshold, is within PROB_RTOL of the maximum."""
    flat = np.sort(p.reshape(-1))
    return flat[-1] - flat[-2] <= PROB_RTOL * flat[-1] or any(abs(m1 - t) <= PROB_RTOL * m1 for t in thresholds if np.isfinite(t))


def test_localize_kernel_softmax_on_recorded_trajectories(emul):
    flags, parted = set(), []
    for name in ("noaug", "stress"):
        d = np.load(os.path.join(GOLDEN, "prdimp_host_%s.npz" % name))
        params = prdimp_params(name)
        hl = HostLogic(params)
        H, W = [int(v) for v in d["image_hw"]]
        hl.adopt(H, W, d["init_state"], d["init_sw"], d["init_counts"][0], d["init_counts"][1])
        for t in range(len(d["flag"])):
            g = hl.plan_crop()
            st = hl.state()
            neigh = [np.float32(np.float32(params.target_neighborhood_scale) * (st[2 + i] / np.float32(g.sample_scale))) * np.float32(22.0 / 352.0)
                     for i in range(2)]
            pv = [(st[i] - np.float32(g.sample_pos[i])) / (np.float32(16.0) * np.float32(g.sample_scale)) for i in range(2)]
            out = _localize(emul, d["scores"][t][None], params, [neigh], [pv])
            assert abs(out.max_score - d["max_score"][t]) <= PROB_RTOL * d["max_score"][t], (name, t)
            assert abs(out.score1 - d["m1"][t, 0]) <= PROB_RTOL * d["m1"][t, 0], (name, t)
            same = out.flag == d["flag"][t] and (out.r1, out.c1) == (int(d["m1"][t, 1]), int(d["m1"][t, 2])) and out.use_second == d["use2"][t]
            if d["m2"][t, 1] >= 0:
                same = same and (out.r2, out.c2) == (int(d["m2"][t, 1]), int(d["m2"][t, 2]))
                assert abs(out.score2 - d["m2"][t, 0]) <= PROB_RTOL * d["m1"][t, 0], (name, t)
            if not same:
                p = softmax_reg(d["scores"][t][None], None)
                assert near_tie(p, (params.target_not_found_threshold, params.uncertain_threshold, params.hard_sample_threshold),
                                float(d["m1"][t, 0])), (name, t, out.flag, d["flag"][t])
                parted.append((name, t))
            flags.add(int(out.flag))
            hl.commit(g, _loc(d, t))
        hl.close()
    assert len(parted) <= 2, parted
    assert flags >= {1, 2, 3}, flags


def test_localize_kernel_softmax_matches_reference_code_on_random_maps(emul):
    """The kernel against the reference's own localize_target with score_preprocess='softmax' (tests/golden/prdimp_localize_random.npz):
    flag, scale index, translation and debug_info['max_score'], with and without softmax_reg."""
    from oracle.gen_prdimp_golden import localize_cases
    from pytracking_b200.tracker import FLAGS
    gold = np.load(os.path.join(GOLDEN, "prdimp_localize_random.npz"))
    code = {None: 0, "normal": 1, "hard_negative": 2, "uncertain": 3, "not_found": 4}
    img_support_sz, out_sz = torch.Tensor([352, 352]), torch.Tensor([22, 22])
    seen, parted = set(), []
    for trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos in localize_cases():
        S = scores.shape[0]
        neigh = [(2.2 * (target_sz / sample_scales[s]) * (out_sz / img_support_sz)).numpy() for s in range(S)]
        pv = [((pos - sample_pos[s]) / ((img_support_sz / out_sz) * sample_scales[s])).numpy() for s in range(S)]
        out = _localize(emul, scores.numpy(), make_params(**dict(kw, softmax_reg=reg)), neigh, pv)
        assert abs(out.max_score - gold["max_score"][trial]) <= PROB_RTOL * gold["max_score"][trial], trial
        scale_ind = int(gold["scale_ind"][trial])
        cell = (out.r2, out.c2) if out.use_second else (out.r1, out.c1)
        mine = (torch.Tensor(cell) - 11) * (img_support_sz / out_sz) * sample_scales[out.scale_ind]
        if code[FLAGS[out.flag]] != int(gold["flag"][trial]) or out.scale_ind != scale_ind or \
                not torch.equal(mine, torch.from_numpy(gold["translation"][trial])):
            p = softmax_reg(scores.numpy(), reg)
            assert near_tie(p[scale_ind], (kw["target_not_found_threshold"], kw["uncertain_threshold"], kw["hard_sample_threshold"]),
                            float(gold["max_score"][trial])), (trial, FLAGS[out.flag], int(gold["flag"][trial]))
            parted.append(trial)
        seen.add((FLAGS[out.flag], out.use_second, reg is None))
    assert len(parted) <= 2, parted
    for r in (True, False):
        assert {("normal", 0, r), ("hard_negative", 0, r), ("uncertain", 0, r), ("not_found", 0, r)} <= seen, seen
    assert any(k[0] is None for k in seen), seen            # plain localisation (advanced_localization off)
    assert any(k[0] == "hard_negative" and k[1] == 1 for k in seen), seen


def test_localize_kernel_exp_matches_reference_code_on_random_maps(emul):
    """score_preprocess='exp' on the same seeded maps against the reference's localize_target (the _exp arrays of
    tests/golden/prdimp_localize_random.npz): flag, scale index, translation, max_score."""
    from oracle.gen_prdimp_golden import localize_cases
    from pytracking_b200.tracker import FLAGS
    gold = np.load(os.path.join(GOLDEN, "prdimp_localize_random.npz"))
    code = {None: 0, "normal": 1, "hard_negative": 2, "uncertain": 3, "not_found": 4}
    img_support_sz, out_sz = torch.Tensor([352, 352]), torch.Tensor([22, 22])
    seen, parted = set(), []
    for trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos in localize_cases():
        S = scores.shape[0]
        neigh = [(2.2 * (target_sz / sample_scales[s]) * (out_sz / img_support_sz)).numpy() for s in range(S)]
        pv = [((pos - sample_pos[s]) / ((img_support_sz / out_sz) * sample_scales[s])).numpy() for s in range(S)]
        out = _localize(emul, scores.numpy(), make_params(**dict(kw, score_preprocess="exp", softmax_reg=reg)), neigh, pv)
        assert abs(out.max_score - gold["max_score_exp"][trial]) <= PROB_RTOL * gold["max_score_exp"][trial], trial
        scale_ind = int(gold["scale_ind_exp"][trial])
        cell = (out.r2, out.c2) if out.use_second else (out.r1, out.c1)
        mine = (torch.Tensor(cell) - 11) * (img_support_sz / out_sz) * sample_scales[out.scale_ind]
        if code[FLAGS[out.flag]] != int(gold["flag_exp"][trial]) or out.scale_ind != scale_ind or \
                not torch.equal(mine, torch.from_numpy(gold["translation_exp"][trial])):
            e = np.exp(scores.numpy().astype(np.float64))[scale_ind]
            assert near_tie(e, (), float(gold["max_score_exp"][trial])), (trial, FLAGS[out.flag], int(gold["flag_exp"][trial]))
            parted.append(trial)
        seen.add(FLAGS[out.flag])
    assert len(parted) <= 2, parted
    assert {None, "normal", "hard_negative", "uncertain"} <= seen, seen


def test_newton_filter_reg_override_replaces_the_learnt_value():
    """params.filter_reg sets the optimiser's filter_reg and min_filter_reg (dimp.py:598-600), also over a learnt filter_reg in the
    state_dict: reg_weight = filter_reg^2 in float32."""
    from pytracking_b200.frame_engine import newton_scalars
    from pytracking_b200.tracker import newton_hparams
    sd = {"classifier.filter_optimizer.filter_reg": torch.tensor([0.2]), "classifier.filter_optimizer.log_step_length": torch.tensor([0.1])}
    base = dict(min_filter_reg=0.05)
    step, reg = newton_scalars(sd, newton_hparams(base))
    assert step == float(torch.exp(torch.tensor([0.1])).item()) and reg == float((torch.tensor([0.2]) ** 2).item())
    for p in (0.01, 0.5):
        step, reg = newton_scalars(sd, newton_hparams(base, filter_reg=p))
        f = torch.tensor([p])
        assert reg == float((f * f).item()), (p, reg)
    # without learnt values in the state_dict: the constructor's, then the override
    step, reg = newton_scalars({}, newton_hparams(dict(init_step_length=1.0, init_filter_reg=0.05, min_filter_reg=0.05)))
    assert step == 1.0 and reg == float((torch.tensor([0.05]) * torch.tensor([0.05])).clamp(min=0.05 ** 2).item())
    h = newton_hparams(base, filter_reg=0.3, softmax_reg=2.0, label_threshold=0.1, label_shrink=0.05)
    assert (h["init_filter_reg"], h["min_filter_reg"], h["softmax_reg"], h["label_threshold"], h["label_shrink"]) == (0.3, 0.3, 2.0, 0.1, 0.05)


def test_make_params_rejects_what_is_not_implemented():
    for kw in (dict(border_mode="constant"), dict(score_filter_ksz=3), dict(low_score_opt_threshold=0.1), dict(score_preprocess="sigmoid")):
        with pytest.raises(NotImplementedError):
            prdimp_params(**kw)
    p = prdimp_params()
    assert (p.border_mode, p.patch_max_scale_change, p.score_preprocess, p.has_softmax_reg) == (2, 1.5, 2, 0)
    assert (make_params().border_mode, make_params().score_preprocess) == (0, 0)


def test_native_init_refuses_border_mode_inside():
    hl = HostLogic(prdimp_params(border_mode="inside"))
    with pytest.raises(RuntimeError, match="inside"):
        hl.init_state(480, 640, [300, 200, 60, 50])
    hl.close()
