"""Native PrDiMP-50 (BASELINE configs[2]) frames/s, timed the way bench.py times DiMP-50's `value`, and native DiMP-50 in the same
process, the two alternating three times.

    python tools/prdimp_bench.py [--steps K] [--warmup W] [--rounds 3]

Per arm: initialise on frame 0 of the synthetic sequence of bench.py, PREROLL untimed frames (the memory fills up), W untimed warm-up
frames, then K frames with the uint8 frames already resident in HBM, L2 flushed (256 MB written) right before the timed region, CUDA
events around the K calls of `track_device`.  PrDiMP-50 runs parameter/dimp/prdimp50.py with the bench overrides
(target_not_found_threshold=-1e9, train_skipping=1, net_opt_update_iter=10; use_iou_net=False, un-augmented initialisation with the
zero filter), 352x352 crops, 'inside_major' crops, softmax localisation and the Newton optimiser; DiMP-50 runs bench.py's parameters.
Prints one JSON line with the device name and power limit.  Uses neither baseline/_ref nor the reference tree.
"""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (constants, the frame sequence and device_info; bench.py runs nothing on import)

PO = "classifier.filter_optimizer."
# pytracking/parameter/dimp/prdimp50.py + the bench overrides of baseline/ref_tracker.build_prdimp
PRDIMP_PARAMS = dict(image_sample_size=352, search_area_scale=6, border_mode="inside_major", patch_max_scale_change=1.5,
                     sample_memory_size=bench.MEMORY, learning_rate=0.01, init_samples_minimum_weight=0.25, train_skipping=1,
                     update_classifier=True, net_opt_iter=10, net_opt_update_iter=bench.SD_ITERS, net_opt_hn_iter=1,
                     advanced_localization=True, score_preprocess="softmax", target_not_found_threshold=-1e9, distractor_threshold=0.8,
                     hard_negative_threshold=0.5, target_neighborhood_scale=2.2, dispalcement_scale=0.8, hard_negative_learning_rate=0.02,
                     augmentation_expansion_factor=2, use_iou_net=False)
# klcedimpnet50 with the ltr/train_settings/dimp/prdimp50.py optimiser arguments (baseline/ref_tracker.build_prdimp)
PRDIMP_NEWTON = dict(feat_stride=16, init_step_length=1.0, init_filter_reg=0.05, min_filter_reg=0.05, gauss_sigma=1 / 4 / 6.0 * 22,
                     alpha_eps=0.05, normalize_label=True)


def build(kind, dev):
    from pytracking_b200 import synth
    from pytracking_b200.tracker import DiMPTracker, make_params
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    if kind == "dimp50":
        return DiMPTracker(sd, make_params(**bench.TRACKER_PARAMS), device=dev)
    sd = {k: v for k, v in sd.items() if not k.startswith((PO, "classifier.filter_initializer."))}
    return DiMPTracker(sd, make_params(**PRDIMP_PARAMS), device=dev, newton=PRDIMP_NEWTON)


def time_arm(kind, dev, steps, warmup):
    trk = build(kind, dev)
    n_frames = bench.PREROLL + warmup + steps
    frames, bb, _ = bench.make_frames(0, n_frames)
    H, W = frames[0].shape[:2]
    pinned = torch.empty(n_frames + 1, H, W, 3, dtype=torch.uint8).pin_memory()
    for i, f in enumerate(frames):
        pinned[i] = torch.from_numpy(f)
    trk.initialize(pinned[0], {"init_bbox": bb})
    f = 1
    for _ in range(bench.PREROLL):
        trk.track(pinned[f]); f += 1
    assert trk.info.n_stored == bench.MEMORY, trk.info.n_stored
    dev_frames = pinned[f:f + warmup + steps].to(dev)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    for i in range(warmup):
        trk.track_device(dev_frames[i])
    torch.cuda.synchronize()
    flush.fill_(1.0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gc.collect(); gc.disable()
    torch.cuda.synchronize()
    e0.record()
    for i in range(steps):
        trk.track_device(dev_frames[warmup + i])
    e1.record()
    torch.cuda.synchronize()
    gc.enable()
    ms = e0.elapsed_time(e1)
    box = [float(v) for v in trk.info.bbox]
    trk.close()
    del dev_frames, flush
    torch.cuda.empty_cache()
    return steps / (ms * 1e-3), box


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"prdimp50": [], "dimp50": []}
    boxes = {}
    for _ in range(args.rounds):
        for kind in ("prdimp50", "dimp50"):
            fps, box = time_arm(kind, dev, args.steps, args.warmup)
            res[kind].append(fps)
            boxes[kind] = box
    med = {k: float(np.median(v)) for k, v in res.items()}
    print(json.dumps({
        "metric": "native tracked frames/s, uint8 frames resident in HBM, L2 flushed, CUDA events (bench.py `value` method)",
        "device": bench.device_info(0), "steps": args.steps, "warmup": args.warmup, "preroll": bench.PREROLL,
        "prdimp50_fps": res["prdimp50"], "dimp50_fps": res["dimp50"], "prdimp50_fps_median": med["prdimp50"],
        "dimp50_fps_median": med["dimp50"], "prdimp50_over_dimp50_frame_time": med["dimp50"] / med["prdimp50"],
        "last_box": boxes,
        "config": {"prdimp50": "parameter/dimp/prdimp50.py + target_not_found_threshold=-1e9, train_skipping=1, net_opt_update_iter=10, "
                               "use_iou_net=False, un-augmented init, 352x352 crops, inside_major, softmax, PrDiMPSteepestDescentNewton",
                   "dimp50": "bench.py TRACKER_PARAMS (BASELINE configs[1])"}}))


if __name__ == "__main__":
    main()
