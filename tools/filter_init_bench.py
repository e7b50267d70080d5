"""Time of a native DiMP-50 `initialize` (crop, forward, initial filter, 10 steepest-descent iterations) with the zero filter and with
the network's learnt initialiser (FilterInitializerLinear), and of the initialiser alone, by CUDA events on the current GPU.

    python tools/filter_init_bench.py [--reps 50] [--precision 0]

Prints one JSON line: median, min, 10th / 90th percentile and max milliseconds per configuration, the GPU's name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = np.array([a.elapsed_time(b) for a, b in ev])
    return {"median_ms": float(np.median(t)), "min_ms": float(t.min()), "p10_ms": float(np.percentile(t, 10)),
            "p90_ms": float(np.percentile(t, 90)), "max_ms": float(t.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--precision", type=int, default=0)
    a = ap.parse_args()
    from pytracking_b200 import synth
    from pytracking_b200.tracker import DiMPTracker, make_params
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from tracker_cases import DIMP50, OVERRIDES
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    frames, bb = synth.make_sequence(2, num_frames=1)
    out = {}
    for mode in ("zero", "network"):
        trk = DiMPTracker(sd, make_params(**dict(DIMP50, **OVERRIDES["noaug"])), precision=a.precision, filter_init=mode)
        out["initialize_" + mode] = _time(lambda: trk.initialize(frames[0], {"init_bbox": bb}), a.reps)
        if mode == "network":
            eng = trk.engine
            out["initialiser_alone"] = _time(lambda: eng.backbone.filter_init(eng.clf[:1], np.array([[100, 100, 80, 60]], np.float32)), a.reps)
        trk.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out.update(gpu=q.splitlines()[0] if q else torch.cuda.get_device_name(), precision=a.precision, reps=a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
