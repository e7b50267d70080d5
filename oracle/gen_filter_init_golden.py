"""TEST INFRASTRUCTURE ONLY -- records what the native learnt filter initialiser must reproduce, from the UNMODIFIED reference
FilterInitializerLinear (ltr/models/target_classifier/initializer.py:118-173) and DiMP tracker, run on the CPU with PrRoIPool from
the CPU restatement installed at the reference's `_prroi_pooling` seam (oracle/ref_shims.py).

    python -m oracle.gen_filter_init_golden        (needs a reference checkout: baseline/_ref or PYTRACKING_REFERENCE)

`tests/golden/filter_init.npz`:
  * heads -- FilterInitializerLinear.forward with DiMP-50's filter_conv (synth.make_dimp_state_dict('resnet50', seed=0, lut_seed=3),
    the weights every DiMP-50 / PrDiMP-50 test network carries) on seeded classification features (synth.make_clf_features) of 288^2
    and 352^2 crops (18^2 and 22^2 maps), S = 1 and 3 images, boxes that are interior, straddle each border of the crop, or are thin;
    plus filter_norm and pool_square once each.  Keys case_<i>_{meta,boxes,filter}; meta = (seed, S, H, filter_norm, pool_square).
  * track -- the reference DiMP tracker with use_augmentation=False, net_opt_update_iter=2 and WITHOUT filter_init_zero (so that
    initialize starts the optimiser from FilterInitializerLinear's filter), use_iou_net=False, 20 frames of synth.make_sequence(2):
    the scalar state and the filter after initialize, and per frame the output box and the localisation flag.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
FLAG = {None: 0, "normal": 1, "hard_negative": 2, "uncertain": 3, "not_found": 4}
PREFIX = "classifier.filter_initializer."


def cases():
    """(seed, S, H, filter_norm, pool_square, boxes [S,4] in crop pixels (x, y, w, h)) -- H the feature map side, 16 H the crop side."""
    out = []
    for H in (18, 22):
        ext = 16.0 * H
        interior = [0.3 * ext, 0.35 * ext, 0.25 * ext, 0.2 * ext]
        left, top = [-0.08 * ext, 0.4 * ext, 0.2 * ext, 0.15 * ext], [0.45 * ext, -0.1 * ext, 0.18 * ext, 0.22 * ext]
        right, bottom = [0.9 * ext, 0.2 * ext, 0.2 * ext, 0.3 * ext], [0.3 * ext, 0.93 * ext, 0.3 * ext, 0.12 * ext]
        thin_w, thin_h = [0.5 * ext, 0.2 * ext, 3.0, 0.4 * ext], [0.1 * ext, 0.6 * ext, 0.5 * ext, 2.5]
        out.append((1 + H, 1, H, 0, 0, [interior]))
        out.append((2 + H, 3, H, 0, 0, [left, top, right]))
        out.append((3 + H, 3, H, 0, 0, [bottom, thin_w, thin_h]))
    out.append((40, 3, 18, 1, 0, out[1][5]))
    out.append((41, 3, 22, 0, 1, out[4][5]))
    return out


def reference_filter_init(sd, feat, boxes, filter_norm, pool_square):
    """FilterInitializerLinear.forward of the reference on feat [S,C,H,W], boxes [S,4]: S images of one sequence -> [1,C,4,4]."""
    from ltr.models.target_classifier.initializer import FilterInitializerLinear
    m = FilterInitializerLinear(filter_size=4, feature_dim=feat.shape[1], feature_stride=16, pool_square=bool(pool_square),
                                filter_norm=bool(filter_norm))
    m.filter_conv.weight.data.copy_(sd[PREFIX + "filter_conv.weight"])
    m.filter_conv.bias.data.copy_(sd[PREFIX + "filter_conv.bias"])
    m.eval()
    with torch.no_grad():
        return m(feat.reshape(feat.shape[0], 1, *feat.shape[1:]), torch.as_tensor(boxes, dtype=torch.float32).reshape(-1, 1, 4))


def main():
    from oracle import ref_shims
    ref_shims.install()
    from baseline import ref_tracker
    from pytracking_b200 import synth
    torch.set_num_threads(8)
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    rec = {}
    for i, (seed, S, H, norm, square, boxes) in enumerate(cases()):
        feat = synth.make_clf_features(seed, S, 512, H, H)
        w = reference_filter_init(sd, feat, boxes, norm, square)
        rec["case_%d_meta" % i] = np.array([seed, S, H, norm, square], dtype=np.int64)
        rec["case_%d_boxes" % i] = np.array(boxes, dtype=np.float32)
        rec["case_%d_filter" % i] = w.reshape(1, 512, 4, 4).numpy().astype(np.float32)
    rec["num_cases"] = np.array(len(cases()))
    # the tracker run
    frames, bb = synth.make_sequence(2, num_frames=20)
    trk = ref_tracker.build_dimp("cpu", overrides=dict(net_opt_update_iter=2), use_augmentation=False)
    assert not getattr(trk.params, "filter_init_zero", False)
    torch.manual_seed(0)
    trk.initialize(frames[0], {"init_bbox": list(bb)})
    assert type(trk.net.classifier.filter_initializer).__name__ == "FilterInitializerLinear"
    rec["track_init_state"] = np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale),
                                        trk.base_target_sz[0], trk.base_target_sz[1], float(trk.min_scale_factor),
                                        float(trk.max_scale_factor)], dtype=np.float32)
    rec["track_init_filter"] = trk.target_filter.detach().reshape(1, 512, 4, 4).numpy().astype(np.float32)
    bbox, flags = [], []
    for t in range(1, len(frames)):
        o = trk.track(frames[t], {})
        bbox.append(np.array(o["target_bbox"], dtype=np.float32))
        flags.append(FLAG[trk.debug_info["flag"]])
    rec["track_bbox"], rec["track_flag"] = np.array(bbox), np.array(flags, dtype=np.int64)
    print("flags:", {k: int((rec["track_flag"] == v).sum()) for k, v in FLAG.items()})
    np.savez_compressed(os.path.join(GOLDEN, "filter_init.npz"), **rec)


if __name__ == "__main__":
    main()
