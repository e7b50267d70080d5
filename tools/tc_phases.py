"""python tools/tc_phases.py [S] [precision]: per-layer phase timing of the tensor-core plan from in-kernel globaltimer stamps (warm, back-to-back launches).

Stamps per CTA: 0 start, 1 prologue done, 2 previous grid complete, 3 first operands landed, 4 accumulator complete,
5 all splits staged / arrived, 6 epilogue done.

The inter-layer time is the part of the forward in which no CTA of the plan is either loading or computing: summed over
consecutive tensor-core layers, (earliest "first operands landed" of layer L+1) - (latest "epilogue done" of layer L), plus,
for the first layer, its earliest landing minus its earliest "previous grid complete" (the maxpool's end)."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytracking_b200 import synth, _lib
from pytracking_b200.engine import BackboneEngine

S = int(sys.argv[1]) if len(sys.argv) > 1 else 1
PRECISION = int(sys.argv[2]) if len(sys.argv) > 2 else 0       # 0: 3xTF32, 2: single-pass TF32
sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
im = synth.make_crop(41, S, 288).cuda()
L = _lib.lib()
eng = BackboneEngine(sd, arch="resnet50", max_batch=S, crop_size=288, precision=PRECISION)
for _ in range(3):
    eng.forward(im, want=("classification",))
n = L.b200trk_net_num_ops(eng.handle)
bufs = {}
for i in range(n):
    info = (C.c_int * 8)()
    L.b200trk_net_op_info(eng.handle, i, C.byref(info))
    if info[7]:
        b = torch.zeros(4096, 8, dtype=torch.int64, device="cuda")
        bufs[i] = (b, list(info))
        _lib.check(L.b200trk_net_op_set_timing_buffer(eng.handle, i, C.c_void_p(b.data_ptr())))
for _ in range(3):
    eng.forward(im, want=("classification",))
torch.cuda.synchronize()
prev_end = None
print("op  cin cout k s  grid          BN | start-gap prolog  depwait firstld  mma    splitwait epi   | cta_total kernel_span |"
      "  kb/cta mma/kb  spread")
tot = 0.0
inter = 0.0
spread_sum = 0.0
phase_sum = [0.0] * 6          # per-layer CTA means, summed over layers: prolog, depwait, firstld, mma, splitwait, epi
first_t0 = None
last_end = None
for i, (b, info) in bufs.items():
    g = (C.c_int * 4)()
    L.b200trk_net_op_grid(eng.handle, i, C.byref(g))
    ctas = g[0] * g[1] * g[2]
    t = b[:ctas].cpu().double()
    t0 = t[:, 0].min()
    end = t[:, 6].max()
    land = t[:, 3].min()
    d = lambda a, bb: float((t[:, bb] - t[:, a]).mean()) / 1e3
    has_split = g[2] > 1
    sw = d(4, 5) if has_split else 0.0
    epi = d(5, 6) if has_split else d(4, 6)
    gap = float(t0 - prev_end) / 1e3 if prev_end is not None else 0.0
    inter += float(land - (prev_end if prev_end is not None else t[:, 2].min())) / 1e3
    # spread: the layer's landing -> last epilogue, less what its average CTA spends from its own landing to its epilogue's end
    spread = float(end - land) / 1e3 - d(3, 6)
    spread_sum += spread
    span = float(end - t0) / 1e3
    tot += span + max(gap, 0)
    for j, v in enumerate((d(0, 1), d(1, 2), d(2, 3), d(3, 4), sw, epi)):
        phase_sum[j] += v
    kb = info[3] * info[3] * info[1] / 32 / g[2]          # mean 32-channel k-blocks per CTA
    print("%2d %4d %4d %d %d  (%3d,%2d,%2d) %3d | %8.2f %6.2f %8.2f %6.2f %6.2f %8.2f %6.2f | %8.2f %8.2f | %7.2f %6.2f %7.2f" % (
        i, info[1], info[2], info[3], info[4], g[0], g[1], g[2], g[3], gap, d(0, 1), d(1, 2), d(2, 3), d(3, 4), sw, epi,
        float((t[:, 6] - t[:, 0]).mean()) / 1e3, span, kb, d(3, 4) / kb, spread))
    prev_end = end
    first_t0 = t0 if first_t0 is None else first_t0
    last_end = end
print("sum of spans+gaps (us):", tot)
print("first CTA start -> last epilogue done (us): %.2f" % (float(last_end - first_t0) / 1e3))
print("inter-layer time (us): %.2f over %d layers" % (inter, len(bufs)))
print("within-layer spread, summed (us): %.2f" % spread_sum)
print("per-layer CTA means summed over layers (us): prolog %.2f depwait %.2f firstld %.2f mma %.2f splitwait %.2f epi %.2f" %
      tuple(phase_sum))
