"""TEST INFRASTRUCTURE ONLY -- records what the native tracker must reproduce for PrDiMP-50 (BASELINE configs[2]), from the UNMODIFIED
reference PrDiMP tracker (baseline.ref_tracker.build_prdimp) run on the CPU.

    python -m oracle.gen_prdimp_golden [noaug|stress|localize]      (needs a reference checkout: baseline/_ref or PYTRACKING_REFERENCE)

Per configuration (`tests/golden/prdimp_host_<name>.npz`), as oracle/gen_host_logic_golden.py records DiMP: the scalar state after
initialize, and per frame the crop request (patch_coord, 'inside_major' crops), the raw score map, both dcf.max2d results and the flag of
localize_advanced on the softmax probabilities, debug_info['max_score'], the output box, the memory update and the optimiser iterations;
plus the Newton optimiser's scalars and hyper-parameters, so that a GPU test can rebuild the network without the reference.
  noaug   -- use_augmentation=False, filter_init_zero=True, 40 frames: the configuration the native initialisation implements
  stress  -- search_area_scale 12 (the sample is taller than the 480-row frame and is centred on it) and thresholds moved into the
             range the softmax probabilities of the random-init net live in: normal, hard_negative (by threshold and by distractor) and
             uncertain occur, with memory wrap-around (sample_memory_size 12) and train_skipping 3.  not_found ends the trajectory's
             updates for good at these scores, and use_second does not occur; both are covered by prdimp_localize_random.npz
Every frame's crop is also checked here: oracle.preprocessing_modes_ref.sample_patch must be bit-equal to the reference's sample_patch.
`tests/golden/prdimp_localize_random.npz`: the reference's localize_target with score_preprocess='softmax' (with and without the
optimiser's softmax_reg), and with 'exp', on seeded 23x23 maps.
`tests/golden/prdimp_host_iou.npz`: PrDiMP-50 with IoUNet refinement on a seeded bb_regressor (record_iou).
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
    "noaug": dict(frames=40, seq=2, overrides=dict(net_opt_update_iter=2)),
    "stress": dict(frames=60, seq=1, overrides=dict(target_not_found_threshold=0.0052, uncertain_threshold=0.00535,
                                                    hard_sample_threshold=0.0055, distractor_threshold=0.3,
                                                    hard_negative_threshold=0.2, train_skipping=3, sample_memory_size=12,
                                                    net_opt_update_iter=2, dispalcement_scale=0.25, search_area_scale=12)),
}
NEWTON_KEYS = ("feat_stride", "gauss_sigma", "min_filter_reg", "alpha_eps", "uni_weight", "normalize_label", "label_shrink",
               "softmax_reg", "label_threshold")


def newton_record(fo):
    """The optimiser's hyper-parameters and learnt scalars (softmax_reg None -> nan)."""
    vals = [float("nan") if getattr(fo, k) is None else float(getattr(fo, k)) for k in NEWTON_KEYS]
    return dict(newton_keys=np.array(NEWTON_KEYS), newton_vals=np.array(vals, dtype=np.float64),
                log_step_length=fo.log_step_length.detach().float().numpy().copy(), filter_reg=fo.filter_reg.detach().float().numpy().copy())


def record(name, cfg):
    from oracle import ref_shims
    ref_shims.install()
    from baseline import ref_tracker
    from pytracking_b200 import synth
    from oracle import preprocessing_modes_ref as PM
    import pytracking.libs.dcf as dcf
    import pytracking.features.preprocessing as pre
    torch.set_num_threads(8)
    frames, bb = synth.make_sequence(cfg["seq"], num_frames=cfg["frames"])
    trk = ref_tracker.build_prdimp("cpu", overrides=cfg["overrides"], use_augmentation=False)
    cur, rec = {}, {}
    orig_max2d, orig_sample = dcf.max2d, pre.sample_patch
    orig_classify, orig_memory = trk.classify_target, trk.update_memory
    fo = trk.params.net.net.classifier.filter_optimizer
    orig_opt = fo.forward
    checked = [0]

    def max2d_hook(a):
        v, i = orig_max2d(a)
        cur.setdefault("max2d", []).append((v.reshape(-1)[0].item(), i.reshape(-1, 2)[0].tolist()))
        return v, i

    def sample_hook(im, pos, sample_sz, output_sz=None, mode="replicate", max_scale_change=None, is_mask=False):
        out = orig_sample(im, pos, sample_sz, output_sz, mode, max_scale_change, is_mask)
        if mode in PM.MODES and not is_mask:
            mine = PM.sample_patch(im, pos, sample_sz, output_sz, mode, max_scale_change)
            assert torch.equal(mine[0], out[0]) and torch.equal(mine[1], out[1]), "preprocessing_modes_ref differs from sample_patch"
            checked[0] += 1
        return out

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

    dcf.max2d, pre.sample_patch = max2d_hook, sample_hook
    trk.classify_target, trk.update_memory = classify_hook, memory_hook
    fo.forward = opt_hook
    try:
        torch.manual_seed(0)
        np.random.seed(0)
        trk.initialize(frames[0], {"init_bbox": list(bb)})
        rec.update(newton_record(fo))
        rec["init_bbox"] = np.array(bb, dtype=np.float64)
        rec["image_hw"] = np.array(frames[0].shape[:2])
        rec["init_state"] = np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale),
                                      trk.base_target_sz[0], trk.base_target_sz[1], float(trk.min_scale_factor),
                                      float(trk.max_scale_factor)], dtype=np.float32)
        rec["init_sw"] = trk.sample_weights[0].clone().numpy()
        rec["init_counts"] = np.array([int(trk.num_stored_samples[0]), int(trk.num_init_samples[0])])
        rec["init_sample_pos"] = trk.init_sample_pos.clone().numpy()
        rec["init_sample_scale"] = np.array(float(trk.init_sample_scale), dtype=np.float32)
        rec["init_target_box"] = trk.target_boxes[0].clone().numpy()
        rec["init_filter"] = trk.target_filter.detach().clone().numpy()
        keys = ("coord", "scores", "m1", "m2", "flag", "use2", "max_score", "bbox", "updated", "replace_ind", "target_box", "lr", "sw",
                "num_iter", "n_stored", "state")
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
                centre = (scores.shape[-1] - 1) / 2
                cell = out[0] / (16.0 * sample_scales[out[1]]) + centre      # translation -> score-map cell it came from
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
            per["flag"].append(FLAG[trk.debug_info["flag"]])
            per["max_score"].append(trk.debug_info["max_score"])
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
            per["use2"].append(int(len(m) > 1 and cur["cell"] == m[1][1] and cur["cell"] != m[0][1]))
        for k in keys:
            rec[k] = np.array(per[k])
    finally:
        dcf.max2d, pre.sample_patch = orig_max2d, orig_sample
    assert checked[0] >= len(frames) - 1, checked[0]
    flags = rec["flag"]
    print(name, "flags:", {k: int((flags == v).sum()) for k, v in FLAG.items()}, "use2:", int(rec["use2"].sum()),
          "updates:", int(rec["updated"].sum()), "iters:", np.unique(rec["num_iter"]).tolist(),
          "max_score range:", float(rec["max_score"].min()), float(rec["max_score"].max()),
          "shrunk crops:", int(((rec["coord"][:, 2] - rec["coord"][:, 0]) < (rec["coord"][:, 3] - rec["coord"][:, 1]) - 0.5).sum()))
    np.savez_compressed(os.path.join(GOLDEN, "prdimp_host_%s.npz" % name), **rec)


def localize_cases(n=240):
    """Seeded 23x23 localisation problems for the softmax path: yields (trial, params overrides, reg, raw scores [S,23,23], target_sz,
    sample_scales, sample_pos, pos).  Raw scores are logits of a few peaks over noise, so the probabilities span the flag thresholds."""
    g = torch.Generator().manual_seed(1)
    for trial in range(n):
        S = 1 + trial % 2
        reg = None if trial % 2 == 0 else float(0.5 + 2 * torch.rand(1, generator=g))
        kw = dict(advanced_localization=trial % 10 != 9, target_not_found_threshold=0.04,
                  uncertain_threshold=0.05 if trial % 4 == 0 else -float("inf"),
                  hard_sample_threshold=0.06 if trial % 5 == 0 else -float("inf"), distractor_threshold=0.8, hard_negative_threshold=0.5,
                  dispalcement_scale=0.3 + 0.5 * (trial % 2), score_preprocess="softmax")
        scores = 2.0 * torch.rand(S, 23, 23, generator=g) - 1.0
        for s in range(S):
            for _ in range(1 + trial % 3):
                r, c = [int(v) for v in torch.randint(0, 23, (2,), generator=g)]
                scores[s, r, c] = 2.0 + 4.0 * float(torch.rand(1, generator=g))
        if trial % 7 == 0:
            scores[0, 3, 11] = scores[0, 12, 4] = scores.max() + 0.5
        target_sz = torch.Tensor([60, 80]) * (0.5 + float(torch.rand(1, generator=g)))
        sample_scales = 1.0 + 0.5 * torch.rand(S, generator=g)
        sample_pos = torch.Tensor([[240, 320]]).repeat(S, 1) + torch.rand(S, 2, generator=g)
        pos = sample_pos[0] + 40 * (torch.rand(2, generator=g) - 0.5)
        yield trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos


def record_localize():
    """The reference's localize_target on localize_cases() with score_preprocess='softmax' (the cases' own setting) and, on the same
    maps, with 'exp' (arrays suffixed _exp)."""
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking.tracker.dimp.dimp import DiMP
    from pytracking.utils import TrackerParams
    import types
    out = {}
    for sfx, pre in (("", "softmax"), ("_exp", "exp")):
        tv, scale_ind, flag, maxs, regs = [], [], [], [], []
        for trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos in localize_cases():
            trk = DiMP.__new__(DiMP)
            p = TrackerParams()
            for k, v in dict(kw, score_preprocess=pre).items():
                setattr(p, k, v)
            p.target_neighborhood_scale = 2.2
            trk.params = p
            trk.net = types.SimpleNamespace(classifier=types.SimpleNamespace(filter_optimizer=types.SimpleNamespace(softmax_reg=reg)))
            trk.output_window = None
            trk.kernel_size = torch.Tensor([4, 4])
            trk.img_support_sz = torch.Tensor([352, 352])
            trk.target_sz = target_sz
            trk.pos = pos
            t, si, s, f = trk.localize_target(scores.clone().unsqueeze(1), sample_pos, sample_scales)
            tv.append(t.numpy())
            scale_ind.append(int(si))
            flag.append(FLAG[f])
            maxs.append(float(torch.max(s[si])))
            regs.append(float("nan") if reg is None else reg)
        out.update({"translation" + sfx: np.array(tv, dtype=np.float32), "scale_ind" + sfx: np.array(scale_ind),
                    "flag" + sfx: np.array(flag), "max_score" + sfx: np.array(maxs, dtype=np.float32)})
        out["reg"] = np.array(regs, dtype=np.float64)
    np.savez_compressed(os.path.join(GOLDEN, "prdimp_localize_random.npz"), **out)


IOU_FRAMES, IOU_SEQ = 20, 2


def seeded_iou_net_state(keys, shapes):
    """The seeded bb_regressor of tests/ref_weights.iou_state_dict (same seed and predictor scale) for a stored layout."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ref_weights
    sd = ref_weights.seeded_state_dict(keys, shapes, 5, prefix="bb_regressor.")
    sd["bb_regressor.iou_predictor.weight"] = sd["bb_regressor.iou_predictor.weight"] * 20.0
    return sd


def record_iou():
    """PrDiMP-50 with IoUNet refinement (prdimp50.py: relative box space, 10 ascent steps of 2.5e-3, top-3 mean, 9 random boxes),
    un-augmented, on the seeded bb_regressor.  The proposal noise is drawn from torch's global generator seeded with 1000 + t before frame
    t, and stored, so that a test can hand the native tracker the same numbers.  -> tests/golden/prdimp_host_iou.npz"""
    from oracle import ref_shims
    ref_shims.install()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ref_weights
    from baseline import ref_tracker
    from pytracking_b200 import synth
    torch.set_num_threads(8)
    frames, bb = synth.make_sequence(IOU_SEQ, num_frames=IOU_FRAMES)
    trk = ref_tracker.build_prdimp("cpu", use_iou_net=True, use_augmentation=False, overrides=dict(net_opt_update_iter=2))
    net = trk.params.net.net
    rec = {}
    rec["iou_keys"], rec["iou_shapes"] = ref_weights.layout_arrays(net.bb_regressor.state_dict())
    missing, unexpected = net.load_state_dict(seeded_iou_net_state(rec["iou_keys"], rec["iou_shapes"]), strict=False)
    assert not unexpected and not any(k.startswith("bb_regressor.") for k in missing), unexpected
    rec.update(newton_record(net.classifier.filter_optimizer))
    torch.manual_seed(0)
    trk.initialize(frames[0], {"init_bbox": list(bb)})
    rec["init_bbox"] = np.array(bb, dtype=np.float64)
    rec["init_state"] = np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale),
                                  trk.base_target_sz[0], trk.base_target_sz[1], float(trk.min_scale_factor),
                                  float(trk.max_scale_factor)], dtype=np.float32)
    rec["modulation3"] = trk.iou_modulation[0].detach().reshape(-1).numpy().copy()
    rec["modulation4"] = trk.iou_modulation[1].detach().reshape(-1).numpy().copy()
    n = trk.params.num_init_random_boxes
    noise, bbox, flag = [], [], []
    for t in range(1, len(frames)):
        torch.manual_seed(1000 + t)
        noise.append(torch.rand(n, 4, generator=torch.Generator().manual_seed(1000 + t)).numpy())
        o = trk.track(frames[t], {})
        bbox.append(np.array(o["target_bbox"], dtype=np.float32))
        flag.append(FLAG[trk.debug_info["flag"]])
    rec.update(noise=np.array(noise), bbox=np.array(bbox), flag=np.array(flag))
    rec["refine_params"] = np.array([trk.params.box_refinement_iter, trk.params.box_refinement_step_length, trk.params.iounet_k,
                                     n, float(trk.params.box_refinement_space == "relative")], dtype=np.float64)
    print("iou flags:", {k: int((rec["flag"] == v).sum()) for k, v in FLAG.items()}, "refine params:", rec["refine_params"].tolist())
    np.savez_compressed(os.path.join(GOLDEN, "prdimp_host_iou.npz"), **rec)


if __name__ == "__main__":
    for name in (sys.argv[1:] or list(CONFIGS) + ["localize", "iou"]):
        if name == "localize":
            record_localize()
        elif name == "iou":
            record_iou()
        else:
            record(name, CONFIGS[name])
