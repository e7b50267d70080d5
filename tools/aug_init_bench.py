"""Time of a native DiMP-50 `initialize` with the stock first-frame augmentation (13 crops + 2 dropout copies, the learnt filter
initialiser, 10 steepest-descent iterations over 15 samples) against the un-augmented one, and of its parts on their own: the
augmentation kernels (torch.profiler, kernel time), the batch-13 forward pass and the 10 iterations at n = 15 (CUDA events).

    python tools/aug_init_bench.py [--reps 30]

Prints one JSON line: median, min, 10th / 90th percentile and max milliseconds per item, the GPU's name and its power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from filter_init_bench import _time      # noqa: E402

STOCK = {"fliplr": True, "rotate": [10, -10, 45, -45], "blur": [(3, 1), (1, 3), (2, 2)],
         "relativeshift": [(0.6, 0.6), (-0.6, 0.6), (0.6, -0.6), (-0.6, -0.6)], "dropout": (2, 0.2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    from pytracking_b200 import _lib, synth
    from pytracking_b200.tracker import DiMPTracker, make_params
    from tracker_cases import DIMP50
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    p = make_params(**dict(DIMP50, target_not_found_threshold=-1e9, net_opt_update_iter=2))
    frames, bb = synth.make_sequence(2, num_frames=1)
    out = {}
    plain = DiMPTracker(sd, p, filter_init="network")
    out["initialize_unaugmented"] = _time(lambda: plain.initialize(frames[0], {"init_bbox": bb}), a.reps)
    plain.close()
    trk = DiMPTracker(sd, p, filter_init="network", augmentation=STOCK, random_shift_factor=1 / 3)
    init = lambda: trk.initialize(frames[0], {"init_bbox": bb})
    out["initialize_augmented"] = _time(init, a.reps)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            init()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for tag in ("augment_crops_kernel", "feature_dropout_kernel", "sample_patch_kernel"):
            if tag in ev.key:
                out[tag + "_us"] = float(ev.device_time)
    L, e = _lib.lib(), trk.engine
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    crop = torch.zeros(13, 3, 288, 288, device="cuda")
    out["forward_batch13"] = _time(lambda: _lib.check(L.b200trk_net_forward(e.backbone.handle, C.c_void_p(crop.data_ptr()), 13, None, None,
                                                                            C.c_void_p(e.clf.data_ptr()), stream()), "net_forward"), a.reps)
    box = np.array([100, 100, 80, 60], np.float32)
    sw = np.full(15, 1 / 15, np.float32)
    out["optimizer_n15_10iter"] = _time(lambda: e.update(0, 14, box, sw, 15, 10), a.reps)
    trk.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out.update(gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(), reps=a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
