"""-m gpu: the steepest-descent optimiser on the memory layout the frame engine runs it on.

The engine keeps its sample memory at a channel-plane pitch of H*W rounded up to 32 floats (352 for 18x18, 512 for 22x22) and calls
the optimiser on it in `update`. Here every padding float of that buffer is NaN, so a single read of the padding turns the filter
into NaN. The filter `update` leaves must be finite, bitwise equal to the dense entry point run with the same kernel on a contiguous
copy of the same samples (both kernels read each plane through the same per-plane addressing and sum in an order that does not depend
on the pitch), and close to the float64 solution of the oracle (oracle/dimp_oracle.py run on float64 inputs).

With the crop's own classification feature among the samples, Gauss-Newton steepest descent is not monotone on this problem: the
float64 oracle takes rising steps (e.g. 1.27 -> 3.23 at step 6 for 288 / n = 32), so the losses are compared with the oracle's
(rtol 1e-3) instead of asserted to decrease. The same steps amplify rounding, most at n = 50: there the float32 oracle, which sums
every correlation in float64 and rounds once per operation, is 1.1e-6 (288) and 2.1e-3 (352) from the float64 solution, and the
tensor-core kernel, whose 3xTF32 sweeps round after every MMA, 8.2e-5 and 1.9e-3 (element-wise 5.2e-2 and 0.78; H100, 700 W). The
filter must therefore be within the bars of the full-size optimiser tests (1e-4 global, 1e-3 element-wise) or within 100x the
float32 oracle's own distance to float64, whichever is larger; at n = 32 and 33 both kernels stay within 3x of the float32 oracle's
distance (worst: tensor-core kernel 3.8e-6, element-wise 1.7e-3; float32 oracle 1.8e-6 and 7.8e-4). A wrong, stale or NaN-poisoned sample moves the filter
by orders of magnitude more."""
import numpy as np
import pytest
import torch

from pytracking_b200 import _lib, ops, synth
from pytracking_b200.frame_engine import DiMPFrameEngine, _view

pytestmark = pytest.mark.gpu

PO = "classifier.filter_optimizer."
LUTS = ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")


def _rel(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _rel_elem(a, b, floor=1e-3):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float(((a - b).abs() / b.abs().clamp(min=floor * float(b.abs().max()))).max())


@pytest.fixture(scope="module")
def state_dict():
    return synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)


@pytest.fixture(scope="module", params=[288, 352], ids=["crop288", "crop352"])
def engine(request, state_dict):
    eng = DiMPFrameEngine(state_dict, arch="resnet50", filter_size=4, memory_size=50, max_batch=1, crop_size=request.param, precision=0)
    yield eng
    eng.close()


@pytest.mark.parametrize("n", [32, 33, 50])
def test_sd_on_pitched_sample_memory(engine, state_dict, monkeypatch, n):
    eng = engine
    L = _lib.lib()
    cc, hc, wc = eng.feat_dims
    pitch = L.b200trk_dimp_state_memory_pitch(eng.state)
    assert pitch == (hc * wc + 31) // 32 * 32 and pitch > hc * wc
    raw = _view(L.b200trk_dimp_state_memory(eng.state), (eng.memory_size * cc * pitch,), eng, eng.device)
    pad = raw.view(eng.memory_size, cc, pitch)[:, :, hc * wc:]
    seed = 7 * n + hc
    raw.fill_(float("nan"))
    eng.memory.copy_(synth.make_clf_features(seed, eng.memory_size, cc, hc, wc).cuda())
    eng.boxes.copy_(synth.make_boxes(seed + 1, eng.memory_size, center=(hc * 16) / 2 - 25).cuda())
    g = torch.Generator().manual_seed(seed + 2)
    w0 = (0.01 * torch.randn(1, cc, 4, 4, generator=g)).cuda()
    sw = (torch.rand(n, generator=g) + 0.5).numpy().astype(np.float32)
    sw /= sw.sum(dtype=np.float32)
    crop = synth.make_crop(seed + 3, 1, eng.backbone.crop_size[0]).pin_memory()
    target_box = synth.make_boxes(seed + 4, 1, center=(hc * 16) / 2 - 25)[0].numpy()
    replace = n // 2
    eng.localize(crop)
    luts = [state_dict[PO + k].reshape(-1).cuda() for k in LUTS]
    params = {k[len(PO):]: v for k, v in state_dict.items() if k.startswith(PO)}

    from oracle import dimp_oracle as O
    results = {}
    for kernel, tc in (("tc", None), ("cuda", "0")):
        if tc is None:
            monkeypatch.delenv("B200TRK_SD_TC", raising=False)
        else:
            monkeypatch.setenv("B200TRK_SD_TC", tc)
        eng.filter.copy_(w0)
        # stores the crop's classification feature in slot `replace` (cudaMemcpy2D into the pitched rows), then 10 iterations
        eng.update(0, replace, target_box, sw, n, 10)
        torch.cuda.synchronize()
        assert L.b200trk_sd_last_kernel() == (1 if kernel == "tc" else 0)
        w = eng.filter.clone()
        assert bool(torch.isnan(pad).all()), "the padding of the sample memory was written"
        assert bool(torch.isfinite(w).all()), "%s kernel: non-finite filter (the pitch padding was read)" % kernel
        feat = eng.memory[:n].contiguous()
        bb, swd = eng.boxes[:n].clone(), eng.sample_weights[:n].clone()
        w_dense, _, _ = ops.dimp_sd_gn(w0, feat, bb, swd, *luts, 10, eng.step_length, eng.reg_weight)
        torch.cuda.synchronize()
        assert L.b200trk_sd_last_kernel() == (1 if kernel == "tc" else 0)
        assert torch.equal(w, w_dense), "%s kernel: pitched and dense sample memory give different filters (%.3e)" % (kernel, _rel(w, w_dense))
        _, _, losses = ops.dimp_sd_gn(w0, feat, bb, swd, *luts, 10, eng.step_length, eng.reg_weight, compute_losses=True)
        results[kernel] = (w, losses.cpu().numpy())

    args64 = (w0.double().cpu(), feat.double().cpu(), bb.double().cpu(), swd.double().cpu(), params, 10)
    w64, _, l64 = O.dimp_sd_gn(*args64, min_filter_reg=1e-3)
    w32, _, _ = O.dimp_sd_gn(*[a.float() for a in args64[:4]], params, 10, min_filter_reg=1e-3, compute_losses=False)
    l64 = np.array([float(x) for x in l64])
    bar, bar_elem = max(1e-4, 100 * _rel(w32, w64)), max(1e-3, 100 * _rel_elem(w32, w64))
    for kernel, (w, losses) in results.items():
        e, e_elem = _rel(w, w64), _rel_elem(w, w64)
        print("sd pitched: crop %d pitch %d n %d %s kernel: filter vs float64 oracle %.2e (element-wise %.2e); float32 oracle %.2e (%.2e)"
              % (eng.backbone.crop_size[0], pitch, n, kernel, e, e_elem, _rel(w32, w64), _rel_elem(w32, w64)))
        assert e < bar and e_elem < bar_elem, (kernel, e, e_elem, bar, bar_elem)
        assert np.allclose(losses, l64, rtol=1e-3), (kernel, losses, l64)
