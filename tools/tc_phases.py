"""Per-layer phase timing of the tensor-core plan from in-kernel globaltimer stamps (warm, back-to-back launches)."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytracking_b200 import synth, _lib
from pytracking_b200.engine import BackboneEngine

S = int(sys.argv[1]) if len(sys.argv) > 1 else 1
sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
im = synth.make_crop(41, S, 288).cuda()
L = _lib.lib()
eng = BackboneEngine(sd, arch="resnet50", max_batch=S, crop_size=288, precision=0)
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
print("op  cin cout k s  grid          BN | start-gap prolog  depwait firstld  mma    splitwait epi   | cta_total kernel_span")
tot = 0.0
for i, (b, info) in bufs.items():
    g = (C.c_int * 4)()
    L.b200trk_net_op_grid(eng.handle, i, C.byref(g))
    ctas = g[0] * g[1] * g[2]
    t = b[:ctas].cpu().double()
    t0 = t[:, 0].min()
    end = t[:, 6].max()
    d = lambda a, bb: float((t[:, bb] - t[:, a]).mean()) / 1e3
    has_split = g[2] > 1
    sw = d(4, 5) if has_split else 0.0
    epi = d(5, 6) if has_split else d(4, 6)
    gap = float(t0 - prev_end) / 1e3 if prev_end is not None else 0.0
    span = float(end - t0) / 1e3
    tot += span + max(gap, 0)
    print("%2d %4d %4d %d %d  (%3d,%2d,%2d) %3d | %8.2f %6.2f %8.2f %6.2f %6.2f %8.2f %6.2f | %8.2f %8.2f" % (
        i, info[1], info[2], info[3], info[4], g[0], g[1], g[2], g[3], gap, d(0, 1), d(1, 2), d(2, 3), d(3, 4), sw, epi,
        float((t[:, 6] - t[:, 0]).mean()) / 1e3, span))
    prev_end = end
print("sum of spans+gaps (us):", tot)

