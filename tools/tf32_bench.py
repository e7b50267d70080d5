"""Precision 0 (3xTF32) against precision 2 (single-pass TF32) on the wgmma convolutions, alternated in one process:

    python tools/tf32_bench.py [--rounds 3] [--steps 100] [--reps 30] [--out profiles/tf32_bench.json]

Per round, for each precision in turn:
  forward   the backbone + classification head forward alone (CUDA events around each call, warm), DiMP-50 at 288 and PrDiMP-50 at 352,
            batch S = 1, 4, 8, 16
  tracker   DiMPTracker tracked frames/s by bench.py's device-timed method: TRACKER_PARAMS, PREROLL untimed frames, uint8 frames
            resident in HBM, L2 flushed (256 MB write) before the timed region, CUDA events around `steps` frames
  batch     lock-step DiMPBatchTracker frames/s (all sequences) at S = 4 and 8, tools/batch_bench.py's method
Each number is reported as median [p10, p90] over every sample of every round, with the card's name and power limit read in this run.
Prints one JSON line and writes it to --out."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import PREROLL, TRACKER_PARAMS, device_info  # noqa: E402
from batch_bench import run_batch  # noqa: E402

PRECISIONS = (0, 2)
FORWARD = {"dimp50_288": 288, "prdimp50_352": 352}
FORWARD_S = (1, 4, 8, 16)
BATCH_S = (4, 8)


def stats(xs):
    return {"median": float(np.median(xs)), "p10": float(np.percentile(xs, 10)), "p90": float(np.percentile(xs, 90)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from pytracking_b200 import synth
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.engine import BackboneEngine
    from pytracking_b200.tracker import DiMPTracker, make_params
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    W, K = args.warmup, args.steps
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    n_frames = PREROLL + W + K
    seqs = [synth.make_sequence(q, num_frames=n_frames + 1) for q in range(max(BATCH_S))]
    frames = [torch.from_numpy(np.stack(f)).to(dev) for f, _ in seqs]
    bbs = [bb for _, bb in seqs]
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    engines = {(p, name): BackboneEngine(sd, "resnet50", 4, max(FORWARD_S), crop, p) for p in PRECISIONS for name, crop in FORWARD.items()}
    crops = {crop: synth.make_crop(5, max(FORWARD_S), crop).to(dev) for crop in FORWARD.values()}
    samples = {}

    def add(key, v):
        samples.setdefault(key, []).append(v)

    for _ in range(args.rounds):
        for p in PRECISIONS:
            # ---- forward alone ----
            for name, crop in FORWARD.items():
                eng = engines[(p, name)]
                for S in FORWARD_S:
                    im = crops[crop][:S].contiguous()
                    for _ in range(5):
                        eng.forward(im, want=("classification",))
                    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
                    for a, b in ev:
                        a.record(); eng.forward(im, want=("classification",)); b.record()
                    torch.cuda.synchronize()
                    for a, b in ev:
                        add("forward_us/%s/S%d/p%d" % (name, S, p), a.elapsed_time(b) * 1e3)
            # ---- solo tracker, bench.py's device-timed method ----
            trk = DiMPTracker(sd, make_params(**TRACKER_PARAMS), arch="resnet50", precision=p, device=dev)
            trk.initialize(frames[0][0].cpu(), {"init_bbox": bbs[0]})
            for t in range(1, 1 + PREROLL + W):
                trk.track_device(frames[0][t])
            flush.fill_(1.0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for t in range(1 + PREROLL + W, 1 + PREROLL + W + K):
                trk.track_device(frames[0][t])
            e1.record()
            torch.cuda.synchronize()
            add("tracker_fps/dimp50/p%d" % p, K / (e0.elapsed_time(e1) / 1e3))
            trk.close()
            # ---- lock-step batch ----
            for S in BATCH_S:
                bt = DiMPBatchTracker(sd, make_params(**TRACKER_PARAMS), S, device=dev, precision=p)
                ms, _ = run_batch(bt, frames[:S], bbs[:S], W, K, flush)
                add("batch_fps/dimp50/S%d/p%d" % (S, p), S * K / (ms / 1e3))
                bt.close()
    for eng in engines.values():
        eng.close()
    out = {"device": device_info(0), "rounds": args.rounds, "steps": K, "reps": args.reps,
           "method": "precisions alternated within each round; forward: CUDA events per call, warm; tracker / batch: CUDA events around "
                     "K frames, frames in HBM, L2 flushed before the timed region",
           "results": {k: stats(v) for k, v in samples.items()}}
    # speed-up of precision 2 over 0 on the medians: time ratio p0 / p2 for the forward, rate ratio p2 / p0 for frames/s
    out["speedup_p2"] = {}
    for key in sorted(out["results"]):
        if key.endswith("/p0"):
            a, b = out["results"][key]["median"], out["results"][key[:-3] + "/p2"]["median"]
            out["speedup_p2"][key[:-3]] = a / b if key.startswith("forward") else b / a
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
