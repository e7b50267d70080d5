"""The float64 one-step reference of tests/sd_step_ref.py against the oracle's optimisers (oracle/dimp_oracle.py) run for one iteration on
float64 inputs, in all four modes, and the partition coverage of the GPU test's case list (tests/test_sd_steps_f64_gpu.py)."""
import math

import numpy as np
import pytest
import torch

import sd_step_ref as R
from oracle import dimp_oracle as O
from pytracking_b200 import synth


def _inputs(n, c, fs, seed):
    g = torch.Generator().manual_seed(seed)
    feat = synth.make_clf_features(seed, n, c, fs, fs).double()
    bb = synth.make_boxes(seed + 1, n, center=(fs * 16) / 2 - 25).double()
    sw = torch.rand(n, generator=g, dtype=torch.float64) + 0.5
    w = 0.01 * torch.randn(2, c, 4, 4, generator=g, dtype=torch.float64)
    lab = torch.rand(n, fs + 1, fs + 1, generator=g, dtype=torch.float64)
    return feat, bb, sw / sw.sum(), w, lab


def _oracle_and_problem(mode, feat, bb, sw, lab):
    """(oracle one-iteration call w -> (w1, loss0), Problem) for the same optimiser."""
    p = {k: v.double() for k, v in synth.make_dimp_optimizer_params(seed=3).items()}
    if mode == "gn":
        step, reg = math.exp(float(p["log_step_length"])), max(float(p["filter_reg"]) ** 2, 1e-3 ** 2)
        luts = [p[k] for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
        prob = R.Problem("gn", feat, sw, bb=bb, luts=luts, step_length=step, reg=reg, alpha_eps=0.02)
        run = lambda w: O.dimp_sd_gn(w, feat, bb, sw, p, 1, alpha_eps=0.02)
    elif mode == "newton":
        sigma = 0.25 * feat.shape[-1] / 5
        prob = R.Problem("newton", feat, sw, bb=bb, gauss_sigma=sigma, step_length=math.exp(-0.1), reg=0.05 ** 2, alpha_eps=0.05,
                         softmax_reg=-1.0, label_threshold=0.01, normalize_label=True, label_shrink=0.1, uni_weight=0.05)
        run = lambda w: O.prdimp_sd_newton(w, feat, bb, sw, -0.1, 0.05, 1, sigma, min_filter_reg=0.05, alpha_eps=0.05, softmax_reg_val=-1.0,
                                           label_threshold=0.01, normalize_label=True, label_shrink=0.1, uni_weight=0.05)
    elif mode == "l2":
        prob = R.Problem("l2", feat, sw, bb=bb, gauss_sigma=1.3, hinge_threshold=0.05, step_length=0.9, reg=0.1 ** 2, alpha_eps=0.01)
        run = lambda w: O.dimp_l2_sd_gn(w, feat, bb, sw, math.log(0.9), 0.1, 1, 1.3, 0.05, alpha_eps=0.01)
    else:
        act = mode.split("_")[1]
        prob = R.Problem("hinge", feat, sw, label=lab, filter_reg=0.1, hinge_threshold=0.3, activation_leak=0.1, score_act=act,
                         act_param=0.7, steplength_reg=0.02)
        run = lambda w: O.gn_sd_hinge(w, feat, lab, sw, 0.1, 1, 0.3, 0.1, act, 0.7, 0.02)
    return run, prob


@pytest.mark.parametrize("mode", ["gn", "newton", "l2", "hinge_relu", "hinge_bentpar"])
@pytest.mark.parametrize("fs,use_sw", [(18, True), (22, False)])
def test_step_matches_oracle_one_iteration(mode, fs, use_sw):
    """d = w - w_1 and the loss at w equal the oracle's num_iter = 1 run to 1e-12 relative, for each filter of a stack of two."""
    feat, bb, sw, w, lab = _inputs(3, 32, fs, 11 + fs)
    if mode == "newton":
        w = w * 20          # scores of O(1): a softmax far from uniform
    run, prob = _oracle_and_problem(mode, feat, bb, sw if use_sw else None, lab)
    out = R.step(prob, w)
    assert out["d"].dtype == torch.float64 and out["d"].shape == w.shape
    for k in range(w.shape[0]):
        w1, _, losses = run(w[k:k + 1])
        d_or = w[k:k + 1] - w1
        e = float((out["d"][k] - d_or[0]).abs().max() / d_or.abs().max())
        el = abs(float(out["loss"][k]) - float(losses[0])) / abs(float(losses[0]))
        assert e < 1e-12 and el < 1e-12, (mode, k, e, el)
    # the other side of a kink: the one-cell updates of kink_steps / ghg_steps equal a full evaluation with the override, and differ
    # from the plain step (the override reaches the arithmetic)
    ref = R.step(prob, w, detail=True)
    if R.has_kinks(prob):
        cells = torch.tensor([[0, 0, 0], [2, 7, fs], [1, fs // 2, 3]])
        dk = R.kink_steps(prob, ref, 1, cells)
        for f, (i, y, x) in enumerate(cells.tolist()):
            da = ref["da"][1].clone()
            da[i, y, x] = R.flipped_dact(prob, ref["s"][1])[i, y, x]
            full = R.step(prob, w[1:2], dact=da.unsqueeze(0))["d"][0]
            assert float((dk[f] - full).abs().max() / full.abs().max()) < 1e-12
        flip = R.step(prob, w, dact=R.flipped_dact(prob, out["s"]))
        assert float((flip["d"] - out["d"]).abs().max()) > 1e-3 * float(out["d"].abs().max())
    if mode == "newton":
        dk = R.ghg_steps(prob, ref, 0, torch.tensor([0, 2]))
        for f, i in enumerate((0, 2)):
            fl = torch.zeros(1, 3, dtype=torch.bool)
            fl[0, i] = True
            full = R.step(prob, w[0:1], ghg_flip=fl)["d"][0]
            assert float((dk[f] - full).abs().max() / full.abs().max()) < 1e-12
            assert not torch.equal(full, out["d"][0])
    bound = R.fp32_bound(prob, ref, 8, 8, 40)
    assert bound.shape == (2,) and bool((bound > 0).all()) and bool((bound < 1e-2).all()), bound


def test_tf32_rounding_is_round_to_nearest_ties_away():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 2 ** -11 - 2 ** -20, 3.0e38,
                      float("inf"), float("-inf")], dtype=torch.float32)
    want = [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -(1.0 + 2 ** -10), 1.0, None, float("inf"), float("-inf")]
    r = R.tf32_round(x)
    for a, b in zip(r.tolist(), want):
        if b is not None:
            assert a == b
    assert (r.view(torch.int32) & 0x1fff).eq(0).all()
    assert torch.isnan(R.tf32_round(torch.tensor([float("nan")]))).all()
    y = torch.randn(10000, generator=torch.Generator().manual_seed(1))
    e = (R.tf32_round(y) - y).abs() / y.abs()
    assert float(e.max()) <= 2.0 ** -11


def test_case_list_reaches_every_partition_feature_at_132_sms():
    """The tensor-core cases of the GPU test reach every feature of the unit partition that exists on 132 SMs (H100 SXM).  A range that
    crosses a 128-channel chunk boundary does not exist there: 132 is a multiple of every chunk count (C / 128 = 1..4), so lo(b) lands
    exactly on each chunk boundary; it exists on 114 (H100 PCIe) and 148 SMs, where the same cases reach it."""
    reached, smax = set(), 0
    tc = [c for c in R.cases() if R.kernel_for(c[0], c[4]) == "tc"]
    for kernel, mode, fs, C, n, _ in tc:
        p = R.tc_partition(n, C, fs, 132)
        reached |= p["features"]
        smax = max(smax, p["smax"])
    assert reached == set(R.FEATURES) - {"range crosses a chunk boundary"}, set(R.FEATURES) - reached
    for C in (128, 256, 384, 512):
        for n in range(1, 51):
            for fs in (18, 22):
                assert "range crosses a chunk boundary" not in R.tc_partition(n, C, fs, 132)["features"]
    for G in (114, 148):
        assert any("range crosses a chunk boundary" in R.tc_partition(n, C, fs, G)["features"] for _, _, fs, C, n, _ in tc), G
    assert smax == 3
    # the default dispatch runs the tensor-core kernel at every n = 32..50 and the CUDA-core kernel below, for both tracker modes;
    # the forced kernels cover the other side of the switch
    for mode in ("gn", "newton"):
        ns = {k: sorted(c[4] for c in R.cases() if c[1] == mode and c[0] == k) for k in ("default", "cuda", "tc")}
        assert ns["default"] == list(range(1, 51)) and ns["cuda"] == list(range(32, 51)) and ns["tc"] == [1, 2, 5, 9, 16, 31]


def test_partition_mirror_smax_matches_launcher_rule():
    """smax of the mirror = the launcher's rule (most distinct samples any adjoint range touches), checked by brute force."""
    for n, C, fs, G in ((50, 512, 18, 132), (9, 512, 22, 132), (33, 384, 18, 114), (45, 128, 22, 148)):
        kbt = (fs * fs + 31) // 32
        UT = C // 128 * n * kbt
        want = max([len({(u // kbt) % n for u in range(UT * b // G, UT * (b + 1) // G)}) for b in range(G)] + [1])
        assert R.tc_partition(n, C, fs, G)["smax"] == want
    assert np.isfinite(R.Problem("l2", torch.zeros(2, 4, 18, 18), None, bb=torch.tensor([[100.0, 100, 50, 50]] * 2), gauss_sigma=1.0,
                                 hinge_threshold=0.05, step_length=1.0, reg=0.01).label_margin())
