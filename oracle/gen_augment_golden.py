"""TEST INFRASTRUCTURE ONLY -- records what the native first-frame augmentation (csrc/augment_kernels.cuh,
b200trk_dimp_tracker_initialize_augmented_host) must reproduce, from the UNMODIFIED reference run on the CPU with cv2 present.

    python -m oracle.gen_augment_golden        (needs a reference checkout: baseline/_ref or PYTRACKING_REFERENCE; cv2)

`tests/golden/augment.npz`:
  * warp_<h>x<w>_<i>: augmentation.Rotate(angle i of WARP_ANGLES) on seeded float32 HWC images (warp_image) of even, odd and
    non-square sizes; warp576_digest: SHA-256 of the outputs at 576^2 for the four stock angles;
  * per first frame (prefix dimp_ = parameter/dimp/dimp50.py on synth.make_sequence(0), 288^2 crops from a 576^2 patch;
    prdimp_ = prdimp50.py on make_sequence(1), 352^2 from 704^2), after torch.manual_seed(0): the transforms' kinds and shifts,
    the 15 target boxes, the dropout multipliers, SHA-256 of each of the 13 crops, 32x32 windows of the three blurred crops,
    the sample weights and counts;
  * track_<name>: 20-frame runs with the stock augmentation and schedule (train_skipping 20, net_opt_update_iter 2; the not-found
    test disabled, as for every random-init run), use_iou_net False: dimp (the learnt FilterInitializerLinear), dimp_zero
    (filter_init_zero) and prdimp (the learnt initialiser loaded into klcedimpnet50): the filter after initialize, per frame the
    box, the flag and the maximum score.  prdimp also stores the Newton optimiser's hyper-parameters.
  * blur_order_*: dimp rerun with Blur.__call__ replaced by the oracle's tap-order float32 blur: whether the boxes and flags stay
    the same, and by how much the initial filter moves -- whether the summation order of the blur can reach the trajectory.
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
FLAG = {None: 0, "normal": 1, "hard_negative": 2, "uncertain": 3, "not_found": 4}
WARP_SIZES = [(24, 24), (23, 23), (17, 29)]
WARP_ANGLES = [10, -10, 45, -45, 30, -7.5]
STOCK_ANGLES = [10, -10, 45, -45]
TRACK_OVERRIDES = dict(train_skipping=20, net_opt_update_iter=2)
CROP_WINDOW = (slice(None), slice(128, 160), slice(128, 160))


def warp_image(h, w, seed):
    return (np.random.RandomState(seed).rand(h, w, 3) * 255).astype(np.float32)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def kind_of(T):
    return {"Identity": 0, "Translation": 1, "FlipHorizontal": 2, "Blur": 3, "Rotate": 4}[type(T).__name__]


def record_first_frame(prefix, trk, frame, bb, rec):
    """Runs trk.initialize on `frame` after torch.manual_seed(0), capturing the crops and the dropout masks."""
    import torch.nn.functional as F
    import pytracking.tracker.dimp.dimp as dimp_mod
    cap = {}
    orig_spt, orig_do = dimp_mod.sample_patch_transformed, F.dropout2d

    def spt(*a, **k):
        out = orig_spt(*a, **k)
        cap["crops"] = out.detach().clone()
        return out

    def do(x, p=0.5, training=True, inplace=False):
        before = torch.get_rng_state()
        out = orig_do(x, p, training, inplace)
        after = torch.get_rng_state()
        torch.set_rng_state(before)
        m = orig_do(torch.ones(x.shape[0], x.shape[1], 1, 1), p, training)
        torch.set_rng_state(after)
        assert torch.equal(x * m, out), "dropout2d on ones does not reproduce the reference's masks"
        cap["mask"] = m.reshape(x.shape[0], x.shape[1]).clone()
        return out

    dimp_mod.sample_patch_transformed, F.dropout2d = spt, do
    try:
        torch.manual_seed(0)
        trk.initialize(frame, {"init_bbox": list(bb)})
    finally:
        dimp_mod.sample_patch_transformed, F.dropout2d = orig_spt, orig_do
    n_t = cap["crops"].shape[0]
    rec[prefix + "kinds"] = np.array([kind_of(T) for T in trk.transforms[:n_t]], np.int64)
    rec[prefix + "shifts"] = np.array([list(T.shift) for T in trk.transforms[:n_t]], np.int64)
    rec[prefix + "boxes"] = trk.target_boxes[:int(trk.num_init_samples[0])].numpy().astype(np.float32)
    rec[prefix + "dropout"] = cap["mask"].numpy().astype(np.float32)
    rec[prefix + "crop_digest"] = np.array([digest(c.numpy()) for c in cap["crops"]])
    rec[prefix + "blur_window"] = np.stack([c.numpy()[CROP_WINDOW] for c, T in zip(cap["crops"], trk.transforms) if kind_of(T) == 3])
    rec[prefix + "sw"] = trk.sample_weights[0].numpy().copy()
    rec[prefix + "counts"] = np.array([int(trk.num_stored_samples[0]), int(trk.num_init_samples[0])])
    rec[prefix + "init_state"] = np.array([trk.pos[0], trk.pos[1], trk.target_sz[0], trk.target_sz[1], float(trk.target_scale),
                                           trk.base_target_sz[0], trk.base_target_sz[1], float(trk.min_scale_factor),
                                           float(trk.max_scale_factor)], dtype=np.float32)


def run_track(name, trk, frames, bb, rec):
    torch.manual_seed(0)
    trk.initialize(frames[0], {"init_bbox": list(bb)})
    rec["track_%s_init_filter" % name] = trk.target_filter.detach().reshape(1, -1, 4, 4).numpy().astype(np.float32)
    bbox, flags, scores = [], [], []
    for t in range(1, len(frames)):
        o = trk.track(frames[t], {})
        bbox.append(np.array(o["target_bbox"], dtype=np.float32))
        flags.append(FLAG[trk.debug_info["flag"]])
        scores.append(float(trk.debug_info["max_score"]))
    rec["track_%s_bbox" % name] = np.array(bbox)
    rec["track_%s_flag" % name] = np.array(flags, np.int64)
    rec["track_%s_max_score" % name] = np.array(scores, np.float32)
    print(name, "flags:", {k: int((rec["track_%s_flag" % name] == v).sum()) for k, v in FLAG.items()}, flush=True)


def build_prdimp_learnt(sd):
    from baseline import ref_tracker
    trk = ref_tracker.build_prdimp("cpu", overrides=dict(TRACK_OVERRIDES, filter_init_zero=False))
    fi = trk.params.net.net.classifier.filter_initializer
    with torch.no_grad():
        fi.filter_conv.weight.copy_(sd["classifier.filter_initializer.filter_conv.weight"])
        fi.filter_conv.bias.copy_(sd["classifier.filter_initializer.filter_conv.bias"])
    return trk


def ordered_blur_call(self, image, is_mask=False):
    """augmentation.Blur.__call__ with the oracle's tap-order float32 sums in place of torch's conv2d."""
    from oracle import augmentation_ref as A
    out = torch.from_numpy(A.blur(image[0].numpy(), tuple(self.sigma)))[None]
    return self.crop_to_output(out)


def main():
    from oracle import ref_shims
    ref_shims.install()
    from baseline import ref_tracker
    from pytracking_b200 import synth
    from oracle.gen_prdimp_golden import newton_record
    import cv2
    import pytracking.features.augmentation as aug
    torch.set_num_threads(8)
    rec = {"cv2_version": np.array(cv2.__version__)}
    for h, w in WARP_SIZES:
        for i, a in enumerate(WARP_ANGLES):
            rec["warp_%dx%d_%d" % (h, w, i)] = aug.Rotate(a)(warp_image(h, w, h * 100 + w))
    big = warp_image(576, 576, 576)
    rec["warp576_digest"] = np.array([digest(aug.Rotate(a)(big)) for a in STOCK_ANGLES])
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    frames0, bb0 = synth.make_sequence(0, num_frames=1)
    frames1, bb1 = synth.make_sequence(1, num_frames=1)
    record_first_frame("dimp_", ref_tracker.build_dimp("cpu", overrides=TRACK_OVERRIDES), frames0[0], bb0, rec)
    record_first_frame("prdimp_", build_prdimp_learnt(sd), frames1[0], bb1, rec)
    frames, bb = synth.make_sequence(2, num_frames=20)
    run_track("dimp", ref_tracker.build_dimp("cpu", overrides=TRACK_OVERRIDES), frames, bb, rec)
    run_track("dimp_zero", ref_tracker.build_dimp("cpu", overrides=dict(TRACK_OVERRIDES, filter_init_zero=True)), frames, bb, rec)
    trk = build_prdimp_learnt(sd)
    run_track("prdimp", trk, frames, bb, rec)
    rec.update({"prdimp_" + k: v for k, v in newton_record(trk.params.net.net.classifier.filter_optimizer).items()})
    # the blur's summation order against the recorded trajectory
    orig = aug.Blur.__call__
    aug.Blur.__call__ = ordered_blur_call
    try:
        alt = {}
        run_track("dimp", ref_tracker.build_dimp("cpu", overrides=TRACK_OVERRIDES), frames, bb, alt)
    finally:
        aug.Blur.__call__ = orig
    same = bool(np.array_equal(alt["track_dimp_bbox"], rec["track_dimp_bbox"]) and np.array_equal(alt["track_dimp_flag"], rec["track_dimp_flag"]))
    f, g = alt["track_dimp_init_filter"].astype(np.float64), rec["track_dimp_init_filter"].astype(np.float64)
    rec["blur_order_same_track"] = np.array(same)
    rec["blur_order_filter_rel"] = np.array(np.abs(f - g).max() / np.abs(g).max())
    rec["blur_order_box_max_px"] = np.array(np.abs(alt["track_dimp_bbox"].astype(np.float64) - rec["track_dimp_bbox"]).max())
    print("tap-order blur: boxes and flags %s; initial filter moves %.2e relative, boxes %.2e px" % (
        "identical" if same else "DIFFERENT", float(rec["blur_order_filter_rel"]), float(rec["blur_order_box_max_px"])))
    np.savez_compressed(os.path.join(GOLDEN, "augment.npz"), **rec)


if __name__ == "__main__":
    main()
