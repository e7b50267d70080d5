"""-m gpu: the tensor-core steepest-descent kernel (sd_tc.cu) gives the same filter, bit for bit, as recorded from an earlier build.

The kernel's sweeps are scheduled and laid out for speed (the apply tile's pixels in a bank-conflict-free row order, the two
warpgroups taking turns at the MMA issue), but every accumulator receives the same products in the same order, so a change of
schedule or layout must not move a single bit. The DiMP update is non-smooth, so a last-bit change can move a tracker's closed loop; this test
pins the filter to `tests/golden/sd_tc_sweeps.npz`, recorded on an H100 by `tests/golden/record_sd_tc_sweeps.py`, on seeded
inputs at the sizes the trackers run: n = 32, 33 and 50 samples of C = 512 channels, DiMP-50 (18x18, 10 Gauss-Newton iterations)
and PrDiMP-50 (22x22, 10 Newton iterations). The filter must also be bitwise equal from run to run and close to the CUDA-core
kernel's (sd_optimizer.cu, B200TRK_SD_TC=0), which sums in another order."""
import os

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu

CASES = [(kind, n) for kind in ("dimp18", "prdimp22") for n in (32, 33, 50)]
LUTS = ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")


def case_key(kind, n):
    return "%s_n%d" % (kind, n)


def run_case(kind, n):
    """The optimiser call of case (kind, n) on seeded inputs; returns the filter."""
    h = 18 if kind == "dimp18" else 22
    seed = 300 + 7 * n + h
    feat = synth.make_clf_features(seed, n, 512, h, h).cuda()
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda()
    g = torch.Generator().manual_seed(seed + 2)
    sw = torch.rand(n, generator=g) + 0.5
    sw = (sw / sw.sum()).cuda()
    w0 = (0.01 * torch.randn(1, 512, 4, 4, generator=g)).cuda()
    if kind == "dimp18":
        p = synth.make_dimp_optimizer_params(seed=3)
        w, _, _ = ops.dimp_sd_gn(w0, feat, bb, sw, *[p[k].cuda() for k in LUTS], 10, 0.9, 0.01)
    else:
        sigma = 0.25 * h / 5        # output_sigma_factor * feature_sz / search_area_scale (PrDiMP-50)
        w, _, _ = ops.prdimp_sd_newton(w0, feat, bb, sw, 10, sigma, 1.0, 0.05 ** 2, alpha_eps=0.05, softmax_reg=None,
                                       label_threshold=0.0, normalize_label=True, label_shrink=0.0)
    torch.cuda.synchronize()
    return w.cpu().numpy()


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sd_tc_sweeps.npz"))


@pytest.mark.parametrize("kind,n", CASES)
def test_sd_tc_filter_is_bitwise_the_recorded_one(golden, monkeypatch, kind, n):
    monkeypatch.delenv("B200TRK_SD_TC", raising=False)
    w = run_case(kind, n)
    assert _lib.lib().b200trk_sd_last_kernel() == 1
    ref = golden[case_key(kind, n)]
    diff = np.flatnonzero(w.view(np.uint32) != ref.view(np.uint32))
    assert diff.size == 0, "%d of %d filter entries differ from the recording (max abs %.3e)" % (
        diff.size, w.size, float(np.abs(w - ref).max()))
    assert np.array_equal(run_case(kind, n).view(np.uint32), w.view(np.uint32)), "not deterministic"

    monkeypatch.setenv("B200TRK_SD_TC", "0")
    w_cc = run_case(kind, n)
    assert _lib.lib().b200trk_sd_last_kernel() == 0
    rel = float(np.abs(w.astype(np.float64) - w_cc).max() / np.abs(w_cc).max())
    print("sd_tc %s: filter vs CUDA-core kernel %.2e" % (case_key(kind, n), rel))
    assert rel < 1e-4, rel
