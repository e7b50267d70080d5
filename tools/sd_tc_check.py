"""Tensor-core SD sweeps (B200TRK_SD_TC=1) against the CUDA-core kernel: per-iterate errors, losses, timing, phase trace."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from pytracking_b200 import ops, synth, _lib
from stage_bench import timeit

def rel(a, b):
    a = a.double().cpu(); b = b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))

p = synth.make_dimp_optimizer_params(seed=3)
luts = [p[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]

def run(mode, n, Cc, h, it, tc):
    os.environ["B200TRK_SD_TC"] = "1" if tc else "0"
    feat = synth.make_clf_features(3 + n, n, Cc, h, h).cuda()
    bb = synth.make_boxes(4, n, center=(h * 16) / 2 - 25).cuda()
    sw = (torch.rand(n, generator=torch.Generator().manual_seed(5)) + 0.5); sw = (sw / sw.sum()).cuda()
    w0 = (torch.randn(1, Cc, 4, 4, generator=torch.Generator().manual_seed(6)) * 0.01).cuda()
    if mode == 0:
        return ops.dimp_sd_gn(w0, feat, bb, sw, *luts, it, 0.9, 0.01, return_iterates=True, compute_losses=True)
    return ops.prdimp_sd_newton(w0, feat, bb, sw, it, 0.25, 1.0, 0.05 ** 2, alpha_eps=0.05, softmax_reg=None, label_threshold=0.0,
                                normalize_label=True, label_shrink=0.0, return_iterates=True, compute_losses=True)

for (mode, n, Cc, h, it) in [(0, 15, 512, 18, 0), (0, 15, 512, 18, 1), (0, 15, 512, 18, 3), (0, 50, 512, 18, 10), (0, 7, 128, 22, 4), (0, 3, 256, 18, 2),
                             (1, 15, 512, 22, 5), (0, 1, 512, 18, 2)]:
    try:
        w_r, its_r, l_r = run(mode, n, Cc, h, it, False)
        w_t, its_t, l_t = run(mode, n, Cc, h, it, True)
        torch.cuda.synchronize()
        print("mode %d n=%d C=%d h=%d it=%d: w rel %.2e | iterates %s | losses ref %s tc %s" % (
            mode, n, Cc, h, it, rel(w_t, w_r), " ".join("%.1e" % rel(a, b) for a, b in zip(its_t, its_r)),
            np.array2string(l_r.cpu().numpy(), precision=6), np.array2string(l_t.cpu().numpy(), precision=6)), flush=True)
        w_t2, _, _ = run(mode, n, Cc, h, it, True)
        print("   deterministic:", bool(torch.equal(w_t, w_t2)), flush=True)
    except Exception as e:
        print("mode %d n=%d C=%d h=%d it=%d: FAILED %r" % (mode, n, Cc, h, it, e), flush=True)
        raise

# timing (the stage_bench configuration)
for n in (15, 50):
    feat = synth.make_clf_features(3, n, 512, 18, 18).cuda()
    bb = synth.make_boxes(4, n).cuda()
    sw = torch.full((n,), 1.0 / n).cuda()
    w0 = torch.zeros(1, 512, 4, 4).cuda()
    out = torch.empty_like(w0)
    for tc in (0, 1):
        os.environ["B200TRK_SD_TC"] = str(tc)
        for it in (0, 1, 10):
            print("n=%d tc=%d it=%d: median %.1f us min %.1f us" % ((n, tc, it) + timeit(lambda: ops.dimp_sd_gn(w0, feat, bb, sw, *luts, it, 0.9, 0.01, out=out))), flush=True)

os.environ["B200TRK_SD_TC"] = "1"
os.environ["B200TRK_SD_TRACE"] = "1"
feat = synth.make_clf_features(3, 50, 512, 18, 18).cuda(); bb = synth.make_boxes(4, 50).cuda(); sw = torch.full((50,), 1.0 / 50).cuda()
w0 = torch.zeros(1, 512, 4, 4).cuda()
for _ in range(4):
    ops.dimp_sd_gn(w0, feat, bb, sw, *luts, 4, 0.9, 0.01)
torch.cuda.synchronize()
buf = (C.c_uint64 * 64)()
_lib.check(_lib.lib().b200trk_debug_sd_trace(buf))
t = np.array(list(buf), dtype=np.float64)
print("prologue %.2f | s0 sweep %.2f | barrier %.2f | s-sum %.2f" % ((t[1]-t[0])/1e3, (t[2]-t[1])/1e3, (t[3]-t[2])/1e3, (t[4]-t[3])/1e3))
for it in range(4):
    b = 8 + it * 10
    d = [(t[b+k+1]-t[b+k])/1e3 for k in range(8)]
    print("it %d: resid %.2f | sweepT %.2f | barrier1 %.2f | gsum+b1b+FT %.2f | sweepA %.2f | barrier2 %.2f | qsum+h %.2f | barrier3 %.2f" % (it, *d))
