"""Aggregate throughput of several DiMP-50 sequences tracked in lock-step on one GPU (pytracking_b200/batch.py) against the same
sequences tracked by solo DiMPTrackers one after another:

    python tools/batch_bench.py [--capacities 1,2,4,8] [--steps 100] [--warmup 5] [--rounds 3] [--out profiles/batch_bench.json]

Per capacity S and schedule, S synthetic sequences (synth.make_sequence(q)) with bench.py's TRACKER_PARAMS and PREROLL: initialised and
pre-rolled untimed, then `steps` frames per sequence timed with CUDA events, frames resident in HBM, L2 flushed before the timed region.
Rounds alternate batch and solo over the same sequences.  Schedules:
  bench  10 optimiser iterations every frame (bench.py's schedule)
  stock  train_skipping=20, net_opt_update_iter=2 (pytracking/parameter/dimp/dimp50.py): most frames are crop + forward + classify + localise
Also reported: the network forward alone at batch S vs batch 1, and the mean IoU of every sequence against its ground truth.
Prints one JSON line (device name and power limit included)."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import PREROLL, TRACKER_PARAMS, device_info, event_time_us  # noqa: E402

SCHEDULES = {"bench": {}, "stock": dict(train_skipping=20, net_opt_update_iter=2)}


def run_batch(bt, frames, bbs, W, K, flush):
    S = len(frames)
    bt.step({s: (frames[s][0], {"init_bbox": bbs[s]}) for s in range(S)})
    boxes = [[] for _ in range(S)]
    for t in range(1, 1 + PREROLL + W):
        out = bt.step({s: (frames[s][t], None) for s in range(S)})
        for s in range(S):
            boxes[s].append(out[s]["target_bbox"])
    flush.fill_(1.0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(1 + PREROLL + W, 1 + PREROLL + W + K):
        out = bt.step({s: (frames[s][t], None) for s in range(S)})
        for s in range(S):
            boxes[s].append(out[s]["target_bbox"])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), boxes


def run_solo(trks, frames, bbs, W, K, flush):
    S = len(frames)
    boxes = [[] for _ in range(S)]
    for s in range(S):
        trks[s].initialize(frames[s][0].cpu().numpy(), {"init_bbox": bbs[s]})
    for t in range(1, 1 + PREROLL + W):
        for s in range(S):
            boxes[s].append(list(trks[s].track_device(frames[s][t]).bbox))
    flush.fill_(1.0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(1 + PREROLL + W, 1 + PREROLL + W + K):
        for s in range(S):
            boxes[s].append(list(trks[s].track_device(frames[s][t]).bbox))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), boxes


def mean_ious(boxes, n_frames):
    from pytracking_b200 import shard, synth
    out = []
    for q, b in enumerate(boxes):
        gt = torch.tensor(synth.sequence_ground_truth(q, n_frames)[1:1 + len(b)], dtype=torch.float32)
        out.append(round(float(shard.iou_overlap(torch.tensor(b, dtype=torch.float32), gt).mean()), 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacities", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--schedules", default="bench,stock")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from pytracking_b200 import synth
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import DiMPTracker, make_params
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    W, K = args.warmup, args.steps
    n_frames = PREROLL + W + K
    caps = [int(c) for c in args.capacities.split(",")]
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    seqs = [synth.make_sequence(q, num_frames=n_frames) for q in range(max(caps))]
    frames = [torch.from_numpy(np.stack(f)).to(dev) for f, _ in seqs]
    bbs = [bb for _, bb in seqs]
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    rows = []
    for sched in args.schedules.split(","):
        params = dict(TRACKER_PARAMS, **SCHEDULES[sched])
        solo = [DiMPTracker(sd, make_params(**params), device=dev) for _ in range(max(caps))]
        for S in caps:
            bt = DiMPBatchTracker(sd, make_params(**params), S, device=dev)
            fb, fs, iou_b, iou_s = [], [], None, None
            for _ in range(args.rounds):
                ms, boxes = run_batch(bt, frames[:S], bbs[:S], W, K, flush)
                fb.append(S * K / ms * 1e3)
                iou_b = mean_ious(boxes, n_frames)
                ms, boxes = run_solo(solo[:S], frames[:S], bbs[:S], W, K, flush)
                fs.append(S * K / ms * 1e3)
                iou_s = mean_ious(boxes, n_frames)
            crop = synth.make_crop(5, S, params["image_sample_size"]).to(dev)
            fwd_s = event_time_us(lambda: bt.backbone.forward(crop, want=("classification",)), 20)
            crop1 = crop[:1].contiguous()
            fwd_1 = event_time_us(lambda: solo[0].engine.backbone.forward(crop1, want=("classification",)), 20)
            rows.append({"schedule": sched, "capacity": S, "batch_fps": [round(v, 1) for v in fb], "solo_fps": [round(v, 1) for v in fs],
                         "batch_fps_median": round(statistics.median(fb), 1), "solo_fps_median": round(statistics.median(fs), 1),
                         "speedup_median": round(statistics.median(fb) / statistics.median(fs), 3),
                         "forward_batch_S_us": round(fwd_s, 1), "forward_batch_1_us": round(fwd_1, 1),
                         "forward_per_sequence_ratio": round(fwd_s / S / fwd_1, 3),
                         "mean_iou_batch": iou_b, "mean_iou_solo": iou_s})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
            bt.close()
        for t in solo:
            t.close()
    res = {"metric": "aggregate tracked frames/s of S DiMP-50 sequences on one GPU: lock-step batch vs solo trackers in turn",
           "device": device_info(0), "steps": K, "warmup": W, "preroll": PREROLL, "rounds": args.rounds,
           "timing": "CUDA events around K steps of all S sequences; frames resident in HBM; L2 flushed (256 MB write) before each timed region",
           "rows": rows}
    line = json.dumps(res)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
