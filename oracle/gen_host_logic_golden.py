"""TEST INFRASTRUCTURE ONLY -- records what the host half of the native whole-frame tracker (csrc/dimp_tracker.cu: plan_crop / commit)
and its two small kernels (sample_patch, localize) must reproduce, from the UNMODIFIED reference DiMP tracker run on the CPU.

    python -m oracle.gen_host_logic_golden [cfg2|stress|noaug|localize|localize_nan]      (needs a reference checkout: baseline/_ref or PYTRACKING_REFERENCE)

Per configuration (`tests/golden/dimp_host_<name>.npz`): the scalar state after DiMP.initialize, and per frame the crop request
(sample_patch's patch_coord), the score map, both dcf.max2d results and the flag of localize_advanced, the output box, the memory
update (slot, target box, learning rate, sample weights) and the optimiser iterations.  Configurations:
  cfg2    -- parameter/dimp/dimp50.py + the BASELINE configs[1] overrides (default augmentation: 15 init samples)
  stress  -- thresholds moved into the range random-init scores live in, so every branch of the decision tree
             (not_found / uncertain / hard_negative by either maximum / normal), memory wrap-around and train_skipping > 1 occur
  noaug   -- use_augmentation=False, filter_init_zero=True: the configuration the native initialisation implements
and `tests/golden/dimp_localize_random.npz`: the reference's `DiMP.localize_target` (translation, scale index, flag) on the 400 seeded
problems of tests/tracker_cases.py:random_localize_cases, and `tests/golden/dimp_localize_nan.npz` (target localize_nan): the same on
the NaN maps of tests/tracker_cases.py:nan_localize_cases.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
FLAG = {None: 0, "normal": 1, "hard_negative": 2, "uncertain": 3, "not_found": 4}

CONFIGS = {
    "cfg2": dict(frames=200, seq=0, aug=True, overrides={}),
    "stress": dict(frames=120, seq=1, aug=True, overrides=dict(target_not_found_threshold=0.052, uncertain_threshold=0.0555,
                                                               hard_sample_threshold=0.058, distractor_threshold=0.3,
                                                               hard_negative_threshold=0.07, train_skipping=3, sample_memory_size=24,
                                                               net_opt_update_iter=2, dispalcement_scale=0.25)),
    "noaug": dict(frames=40, seq=2, aug=False, overrides=dict(filter_init_zero=True, net_opt_update_iter=2)),
}


def record(name, cfg):
    from oracle import ref_shims
    ref_shims.install()
    from baseline import ref_tracker
    from pytracking_b200 import synth
    import pytracking.libs.dcf as dcf
    import pytracking.features.preprocessing as pre
    torch.set_num_threads(8)
    frames, bb = synth.make_sequence(cfg["seq"], num_frames=cfg["frames"])
    trk = ref_tracker.build_dimp("cpu", overrides=cfg["overrides"], use_augmentation=cfg["aug"])
    cur, rec = {}, {}
    orig_max2d, orig_sample = dcf.max2d, pre.sample_patch
    orig_classify, orig_memory, orig_update = trk.classify_target, trk.update_memory, trk.update_classifier
    orig_opt = trk.params.net.net.classifier.filter_optimizer.forward

    def max2d_hook(a):
        v, i = orig_max2d(a)
        cur.setdefault("max2d", []).append((v.reshape(-1)[0].item(), i.reshape(-1, 2)[0].tolist()))
        return v, i

    def classify_hook(x):
        s = orig_classify(x)
        cur["scores"] = s.detach().clone().numpy().reshape(s.shape[-2], s.shape[-1])
        cur["max2d"] = []
        return s

    def memory_hook(sample_x, target_box, learning_rate=None):
        orig_memory(sample_x, target_box, learning_rate)
        cur["replace_ind"] = int(trk.previous_replace_ind[0])
        cur["target_box"] = target_box.clone().numpy()
        cur["lr"] = float(learning_rate)
        cur["sw"] = trk.sample_weights[0].clone().numpy()

    def opt_hook(weights, feat=None, bb=None, sample_weight=None, num_iter=None, compute_losses=True):
        cur["num_iter"] = int(num_iter)
        cur["n_stored"] = int(feat.shape[0])
        return orig_opt(weights, feat=feat, bb=bb, sample_weight=sample_weight, num_iter=num_iter, compute_losses=compute_losses)

    dcf.max2d = max2d_hook
    trk.classify_target, trk.update_memory = classify_hook, memory_hook
    trk.params.net.net.classifier.filter_optimizer.forward = opt_hook
    try:
        torch.manual_seed(0)
        np.random.seed(0)
        trk.initialize(frames[0], {"init_bbox": list(bb)})
        rec["init_bbox"] = np.array(bb, dtype=np.float64)
        rec["image_hw"] = np.array(frames[0].shape[:2])
        rec["params"] = np.array([trk.params.sample_memory_size, trk.params.train_skipping, trk.params.net_opt_iter,
                                  trk.params.net_opt_update_iter, trk.params.net_opt_hn_iter])
        rec["params_f"] = np.array([trk.params.target_not_found_threshold, trk.params.distractor_threshold,
                                    trk.params.hard_negative_threshold, trk.params.dispalcement_scale], dtype=np.float64)
        rec["init_state"] = np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale),
                                      trk.base_target_sz[0], trk.base_target_sz[1], float(trk.min_scale_factor),
                                      float(trk.max_scale_factor)], dtype=np.float32)
        rec["init_sw"] = trk.sample_weights[0].clone().numpy()
        rec["init_counts"] = np.array([int(trk.num_stored_samples[0]), int(trk.num_init_samples[0])])
        rec["init_sample_pos"] = trk.init_sample_pos.clone().numpy()
        rec["init_sample_scale"] = np.array(float(trk.init_sample_scale), dtype=np.float32)
        rec["init_target_box"] = trk.target_boxes[0].clone().numpy()
        keys = ("coord", "scores", "m1", "m2", "flag", "use2", "bbox", "updated", "replace_ind", "target_box", "lr", "sw", "num_iter",
                "n_stored", "state")
        per = {k: [] for k in keys}
        mem = trk.params.sample_memory_size
        for t in range(1, len(frames)):
            cur.clear()
            coords = {}
            orig_extract = trk.extract_backbone_features

            def extract_hook(im, pos, scales, sz):
                out = orig_extract(im, pos, scales, sz)
                coords["c"] = out[1].clone().float().numpy().reshape(4)
                return out
            trk.extract_backbone_features = extract_hook
            orig_loc = trk.localize_target

            def loc_hook(scores, sample_pos, sample_scales):
                out = orig_loc(scores, sample_pos, sample_scales)
                cell = out[0] / (16.0 * sample_scales[out[1]]) + 9.0          # translation -> score-map cell it came from
                cur["cell"] = [int(round(float(cell[0]))), int(round(float(cell[1])))]
                return out
            trk.localize_target = loc_hook
            o = trk.track(frames[t], {})
            trk.extract_backbone_features = orig_extract
            trk.localize_target = orig_loc
            m = cur["max2d"]
            per["coord"].append(coords["c"])
            per["scores"].append(cur["scores"])
            per["m1"].append([m[0][0], m[0][1][0], m[0][1][1]])
            per["m2"].append([m[1][0], m[1][1][0], m[1][1][1]] if len(m) > 1 else [0.0, -1, -1])
            flag = trk.debug_info["flag"]
            per["flag"].append(FLAG[flag])
            per["bbox"].append(np.array(o["target_bbox"], dtype=np.float32))
            upd = "replace_ind" in cur
            per["updated"].append(int(upd))
            per["replace_ind"].append(cur.get("replace_ind", -1))
            per["target_box"].append(cur.get("target_box", np.zeros(4, dtype=np.float32)))
            per["lr"].append(cur.get("lr", 0.0))
            per["sw"].append(cur.get("sw", np.zeros(mem, dtype=np.float32)))
            per["num_iter"].append(cur.get("num_iter", 0))
            per["n_stored"].append(cur.get("n_stored", 0))
            per["state"].append(np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale)],
                                         dtype=np.float32))
            # which maximum gave the translation (dimp.py:289-292)
            per["use2"].append(int(len(m) > 1 and cur["cell"] == m[1][1] and cur["cell"] != m[0][1]))
        for k in keys:
            rec[k] = np.array(per[k])
    finally:
        dcf.max2d = orig_max2d
    flags = rec["flag"]
    print(name, "flags:", {k: int((flags == v).sum()) for k, v in FLAG.items()}, "updates:", int(rec["updated"].sum()),
          "iters:", np.unique(rec["num_iter"]).tolist(), "wraps:", int((rec["replace_ind"][rec["updated"] == 1] < rec["n_stored"].max() - 1).sum()))
    np.savez_compressed(os.path.join(GOLDEN, "dimp_host_%s.npz" % name), **rec)


def record_localize():
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking.tracker.dimp.dimp import DiMP
    from pytracking.utils import TrackerParams
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from tracker_cases import random_localize_cases
    tv, scale_ind, flag = [], [], []
    for trial, kw, scores, target_sz, sample_scales, sample_pos, pos in random_localize_cases():
        trk = DiMP.__new__(DiMP)
        p = TrackerParams()
        for k, v in kw.items():
            setattr(p, k, v)
        p.target_neighborhood_scale = 2.2
        trk.params = p
        trk.output_window = None
        trk.kernel_size = torch.Tensor([4, 4])
        trk.img_support_sz = torch.Tensor([288, 288])
        trk.target_sz = target_sz
        trk.pos = pos
        t, si, _, f = trk.localize_target(scores.clone().unsqueeze(1), sample_pos, sample_scales)
        assert t.dtype == torch.float32
        tv.append(t.numpy())
        scale_ind.append(int(si))
        flag.append(FLAG[f])
    np.savez_compressed(os.path.join(GOLDEN, "dimp_localize_random.npz"), translation=np.array(tv, dtype=np.float32),
                        scale_ind=np.array(scale_ind), flag=np.array(flag))


def record_localize_nan():
    import types
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking.tracker.dimp.dimp import DiMP
    from pytracking.utils import TrackerParams
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from tracker_cases import nan_localize_cases
    tv, scale_ind, flag = [], [], []
    for trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos in nan_localize_cases():
        trk = DiMP.__new__(DiMP)
        p = TrackerParams()
        for k, v in kw.items():
            setattr(p, k, v)
        p.target_neighborhood_scale = 2.2
        trk.params = p
        trk.net = types.SimpleNamespace(classifier=types.SimpleNamespace(filter_optimizer=types.SimpleNamespace(softmax_reg=reg)))
        trk.output_window = None
        trk.kernel_size = torch.Tensor([4, 4])
        trk.img_support_sz = torch.Tensor([288, 288])
        trk.target_sz = target_sz
        trk.pos = pos
        t, si, _, f = trk.localize_target(scores.clone().unsqueeze(1), sample_pos, sample_scales)
        tv.append(t.numpy())
        scale_ind.append(int(si))
        flag.append(FLAG[f])
    np.savez_compressed(os.path.join(GOLDEN, "dimp_localize_nan.npz"), translation=np.array(tv, dtype=np.float32),
                        scale_ind=np.array(scale_ind), flag=np.array(flag))


if __name__ == "__main__":
    targets = {"localize": record_localize, "localize_nan": record_localize_nan}
    for name in (sys.argv[1:] or list(CONFIGS) + list(targets)):
        targets[name]() if name in targets else record(name, CONFIGS[name])
