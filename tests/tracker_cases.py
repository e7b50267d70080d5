"""Tracker parameter sets and golden-trajectory helpers shared by the CPU host-logic test and the GPU tracker tests."""
import os

from pytracking_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
DIMP50 = dict(image_sample_size=288, search_area_scale=5, sample_memory_size=50, learning_rate=0.01, init_samples_minimum_weight=0.25,
              train_skipping=20, update_classifier=True, net_opt_iter=10, net_opt_update_iter=2, net_opt_hn_iter=1,
              advanced_localization=True, target_not_found_threshold=0.25, distractor_threshold=0.8, hard_negative_threshold=0.5,
              target_neighborhood_scale=2.2, dispalcement_scale=0.8, hard_negative_learning_rate=0.02, augmentation_expansion_factor=2,
              use_iou_net=False)
OVERRIDES = {
    "cfg2": dict(target_not_found_threshold=-1e9, train_skipping=1, net_opt_update_iter=10),
    "stress": dict(target_not_found_threshold=0.052, uncertain_threshold=0.0555, hard_sample_threshold=0.058, distractor_threshold=0.3,
                   hard_negative_threshold=0.07, train_skipping=3, sample_memory_size=24, net_opt_update_iter=2, dispalcement_scale=0.25),
    "noaug": dict(target_not_found_threshold=-1e9, train_skipping=1, net_opt_update_iter=2),
}


def random_localize_cases(n=400):
    """Seeded localisation problems for the localisation kernel (score maps with a few peaks and exact ties, thresholds, geometry):
    yields (trial, params overrides, scores [S,19,19], target_sz, sample_scales, sample_pos, pos).  The reference's answers to the
    same problems are tests/golden/dimp_localize_random.npz (oracle/gen_host_logic_golden.py)."""
    import torch
    g = torch.Generator().manual_seed(0)
    for trial in range(n):
        S = 1 + trial % 3
        kw = dict(advanced_localization=trial % 10 != 9, target_not_found_threshold=0.2,
                  uncertain_threshold=0.25 if trial % 4 == 0 else -float("inf"),
                  hard_sample_threshold=0.3 if trial % 5 == 0 else -float("inf"), distractor_threshold=0.8, hard_negative_threshold=0.5,
                  dispalcement_scale=0.3 + 0.5 * (trial % 2))
        scores = 0.1 * torch.rand(S, 19, 19, generator=g)
        for s in range(S):
            for _ in range(1 + trial % 3):               # a few peaks of comparable height
                r, c = [int(v) for v in torch.randint(0, 19, (2,), generator=g)]
                scores[s, r, c] = 0.15 + 0.6 * float(torch.rand(1, generator=g))
        if trial % 7 == 0:                               # exact ties: the arg-max order must follow dcf.max2d
            scores[0, 3, 11] = scores[0, 12, 4] = scores.max() + 0.1
        target_sz = torch.Tensor([60, 80]) * (0.5 + float(torch.rand(1, generator=g)))
        sample_scales = 1.0 + 0.5 * torch.rand(S, generator=g)
        sample_pos = torch.Tensor([[240, 320]]).repeat(S, 1) + torch.rand(S, 2, generator=g)
        pos = sample_pos[0] + 40 * (torch.rand(2, generator=g) - 0.5)
        yield trial, kw, scores, target_sz, sample_scales, sample_pos, pos


def nan_localize_cases():
    """Seeded localisation problems with NaN in the score maps: yields (trial, params overrides, softmax_reg, scores [S,19,19], target_sz,
    sample_scales, sample_pos, pos).  One NaN cell inside and outside the target neighbourhood, a NaN column, a NaN scale among finite
    ones, an all-NaN map, with and without advanced localisation and through the 'exp' and 'softmax' pre-processing.  The reference's
    answers are tests/golden/dimp_localize_nan.npz (oracle/gen_host_logic_golden.py localize_nan)."""
    import torch
    g = torch.Generator().manual_seed(3)
    nan = float("nan")
    kinds = ("inside", "outside", "column", "scale", "all", "two")
    pres = ((None, "none"), (None, "exp"), (None, "softmax"), (1.5, "softmax"))
    trial = 0
    for kind in kinds:
        for j in range(4):
            S = 1 + (trial % 3) if kind != "scale" else 2 + j % 2
            reg, pre = pres[j] if kind in ("inside", "all", "column") else pres[j % 2]
            kw = dict(advanced_localization=j != 3 or kind == "scale", target_not_found_threshold=0.2 if pre == "none" else 0.01,
                      uncertain_threshold=-float("inf"), hard_sample_threshold=-float("inf"), distractor_threshold=0.8,
                      hard_negative_threshold=0.5, dispalcement_scale=0.3 + 0.5 * (trial % 2), score_preprocess=pre)
            scores = 0.1 * torch.rand(S, 19, 19, generator=g)
            peaks = []
            for s in range(S):
                r, c = [int(v) for v in torch.randint(2, 17, (2,), generator=g)]
                scores[s, r, c] = 0.3 + 0.5 * float(torch.rand(1, generator=g))
                peaks.append((r, c))
            s0 = int(torch.randint(0, S, (1,), generator=g))
            r, c = peaks[s0]
            if kind == "inside":
                scores[s0, r + 1, c - 1] = nan
            elif kind == "outside":
                scores[s0, (r + 9) % 19, (c + 9) % 19] = nan
            elif kind == "column":
                scores[s0, :, (c + 7) % 19] = nan
            elif kind == "scale":
                scores[S - 1, 4 + j, 3] = nan
            elif kind == "all":
                scores[s0] = nan
            else:
                scores[s0, 2, 5] = scores[s0, 14, 5] = scores[s0, 9, 12] = nan
            target_sz = torch.Tensor([60, 80]) * (0.5 + float(torch.rand(1, generator=g)))
            sample_scales = 1.0 + 0.5 * torch.rand(S, generator=g)
            sample_pos = torch.Tensor([[240, 320]]).repeat(S, 1) + torch.rand(S, 2, generator=g)
            pos = sample_pos[0] + 40 * (torch.rand(2, generator=g) - 0.5)
            yield trial, kw, reg, scores, target_sz, sample_scales, sample_pos, pos
            trial += 1


def _loc(d, t):
    loc = _lib.LocResult()
    loc.flag, loc.scale_ind = int(d["flag"][t]), 0
    loc.score1, loc.r1, loc.c1 = float(d["m1"][t, 0]), int(d["m1"][t, 1]), int(d["m1"][t, 2])
    loc.score2, loc.r2, loc.c2 = float(d["m2"][t, 0]), int(d["m2"][t, 1]), int(d["m2"][t, 2])
    loc.use_second = int(d["use2"][t])
    loc.max_score = loc.score1
    return loc


