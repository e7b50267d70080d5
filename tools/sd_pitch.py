"""Phase trace of the tensor-core SD kernel on the frame engine's pitched sample memory vs the dense C-ABI call."""
import sys, os, ctypes as C
os.environ["B200TRK_SD_TC"] = "1"; os.environ["B200TRK_SD_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from pytracking_b200 import ops, synth, _lib
from pytracking_b200.frame_engine import DiMPFrameEngine

def trace(tag):
    torch.cuda.synchronize()
    buf = (C.c_uint64 * 64)()
    _lib.check(_lib.lib().b200trk_debug_sd_trace(buf))
    t = np.array(list(buf), dtype=np.float64)
    b = 8 + 10
    d = [(t[b+k+1]-t[b+k])/1e3 for k in range(8)]
    print("%s: s0 sweepA %.2f | it1: resid %.2f | sweepT %.2f | barrier1 %.2f | gsum+b1b+FT %.2f | sweepA %.2f | barrier2 %.2f | qsum+h %.2f | barrier3 %.2f | total call %.1f" % (
        tag, (t[2]-t[1])/1e3, *d, (t[8 + 10 * 3] - t[0]) / 1e3), flush=True)

sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
eng = DiMPFrameEngine(sd, arch="resnet50", memory_size=50, max_batch=1, crop_size=288)
feat = synth.make_clf_features(3, 50, 512, 18, 18).cuda()
eng.memory.copy_(feat)
eng.boxes.copy_(synth.make_boxes(4, 50).cuda())
sw = np.full(50, 1.0 / 50, dtype=np.float32)
for _ in range(3):
    eng.filter.zero_()
    eng.update(0, 7, np.array([100., 100., 60., 60.], dtype=np.float32), sw, 50, 3)
trace("pitched (engine)")
p = synth.make_dimp_optimizer_params(seed=3)
luts = [sd["classifier.filter_optimizer." + k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
w0 = torch.zeros(1, 512, 4, 4).cuda()
dense = eng.memory.contiguous()
for _ in range(3):
    ops.dimp_sd_gn(w0, dense, eng.boxes, torch.from_numpy(sw).cuda(), *luts, 3, eng.step_length, eng.reg_weight)
trace("dense (C ABI)   ")
