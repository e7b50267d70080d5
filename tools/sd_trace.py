"""Phase trace of the tensor-core SD kernel (sd_tc.cu): CTA 0's globaltimer stamps of every phase of every iteration, and the
per-unit pipeline stamps (SM clocks) of its first adjoint sweep.  Usage: python tools/sd_trace.py [n] [iterations]"""
import sys, os, subprocess, ctypes as C
os.environ["B200TRK_SD_TRACE"] = "1"
os.environ["B200TRK_SD_TC"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from pytracking_b200 import ops, synth, _lib
n = int(sys.argv[1]) if len(sys.argv) > 1 else 50
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 10
try:
    plim = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:
    plim = "unknown"
print("device %s, power limit %s; n = %d, C = 512, 18x18, %d iterations" % (torch.cuda.get_device_name(0), plim, n, iters))
p = synth.make_dimp_optimizer_params(seed=3)
luts = [p[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
feat = synth.make_clf_features(3, n, 512, 18, 18).cuda()
bb = synth.make_boxes(4, n).cuda()
sw = torch.full((n,), 1.0 / n).cuda()
w0 = torch.zeros(1, 512, 4, 4).cuda()
for _ in range(4):
    ops.dimp_sd_gn(w0, feat, bb, sw, *luts, iters, 0.9, 0.01)
torch.cuda.synchronize()
buf = (C.c_uint64 * 128)()
_lib.check(_lib.lib().b200trk_debug_sd_trace(buf))
ubuf = (C.c_uint64 * 256)()
_lib.check(_lib.lib().b200trk_debug_sd_units(ubuf))
t = np.array(list(buf), dtype=np.float64)

print("phases of CTA 0 (us, globaltimer)")
print("prologue %.2f | s0 sweepA %.2f | barrier %.2f | s-sum %.2f" % ((t[1]-t[0])/1e3, (t[2]-t[1])/1e3, (t[3]-t[2])/1e3, (t[4]-t[3])/1e3))
# stamps of iteration `it` at tb = 8 + 10 it: +0 residual | +1 adjoint sweep | +2 barrier 1 | +3 gradient slice + barrier | +9
# F^T build | +4 apply sweep | +5 barrier 2 | +6 q + curvature | +7 barrier 3 | +8 step + update | next iteration's +0
cols = ("resid", "sweepT", "barrier1", "gsum+bar", "buildFT", "sweepA", "barrier2", "qsum+h", "barrier3", "update")
order = (0, 1, 2, 3, 9, 4, 5, 6, 7, 8, 10)
sums = np.zeros(len(cols))
for it in range(iters):
    b = 8 + it * 10
    d = np.array([(t[b + order[k + 1]] - t[b + order[k]]) / 1e3 for k in range(len(cols))])
    sums += d
    print("it %d: " % it + " | ".join("%s %.2f" % (c, v) for c, v in zip(cols, d)) + " | total %.2f" % d.sum())
print("mean: " + " | ".join("%s %.2f" % (c, v / iters) for c, v in zip(cols, sums)) + " | total %.2f" % (sums.sum() / iters))
print("call: %.1f us from the first stamp to the last iteration's residual" % ((t[8 + iters * 10] - t[0]) / 1e3))

u = np.array(list(ubuf), dtype=np.float64).reshape(16, 16)
print("CTA 0, first adjoint sweep, per unit (SM clocks after the earliest stamp; '-' = not recorded: the producer issued the")
print("first units during the previous sweep)")
print("  producer: 0 slot free, 1 TMA issued | consumer thread 0: 2 tile landed, 9 operands in registers, 5 stage released,")
print("  8 its warpgroup's turn at the MMAs came, 7 MMAs committed (the turn passes to the other warpgroup)")
t00 = u[u > 0].min() if (u > 0).any() else 0
for i in range(16):
    if u[i, 0] == 0 and u[i, 2] == 0:
        continue
    print("  unit %2d: " % i + "  ".join(("%d:%7d" % (k, u[i, k] - t00)) if u[i, k] else ("%d:      -" % k) for k in (0, 1, 2, 9, 5, 8, 7)))
d = np.diff(u[:, 2][u[:, 2] > 0])
if len(d):
    print("  consumer period (tile landed -> next tile landed): median %d clocks" % np.median(d))
for name, a, b in (("load + split (2 -> 9)", 2, 9), ("issue (8 -> 7)", 8, 7)):
    ok = (u[:, a] > 0) & (u[:, b] > 0)
    if ok.any():
        print("  %s: median %d clocks" % (name, np.median(u[ok, b] - u[ok, a])))
