"""CUDA-event timing of the ECO row (SURVEY 8 f4): b200trk_eco_filter_cg at ECO's default block sizes (parameter/eco/default.py:
memory 200, CG_iter 5; deep block 64 channels on 15x8 Fourier coefficients, shallow block 16 channels on 63x32), with the roofline
figures of DESIGN 4.9: bytes of sample memory per call, the reference's traffic (2 (1 + num_iter) sweeps), achieved GB/s; the first-frame
joint optimisation; and the score computation of a tracked frame (apply_filter, sample_fs, max2d).

    python tools/eco_bench.py [--json PATH]    (on a GPU machine; prints the rows, or writes them to PATH)

bench.py runs this file in a SUBPROCESS after its timed regions (N = 1, rank 0) and appends the rows to `rooflines[]`, so that a defect in
these kernels cannot touch the headline measurement."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from pytracking_b200 import ops  # noqa: E402
from tools.stage_bench import timeit  # noqa: E402

BLOCKS = {"deep 15x8 x 200 x 64": (15, 8, 200, 64), "shallow 63x32 x 200 x 16": (63, 32, 200, 16)}
ITERS = 5
res = {}
for name, (h, wh, n, c) in BLOCKS.items():
    g = torch.Generator().manual_seed(h)
    samples = torch.randn(h, wh, n, c, 2, generator=g).cuda()
    sw = torch.rand(n, generator=g)
    sw = (sw / sw.sum()).cuda()
    yf = torch.rand(1, 1, h, wh, generator=g).cuda()
    reg = torch.tensor([[0.0, 0.23, 0.0], [0.16, 0.78, 0.16], [0.0, 0.23, 0.0]]).view(1, 1, 3, 3).cuda()
    hf = (0.01 * torch.randn(1, c, h, wh, 2, generator=g)).cuda()
    new_xf = torch.randn(1, c, h, wh, 2, generator=g).cuda()
    state = {"en": None, "st": None}

    def run():
        state["en"], state["st"] = ops.eco_filter_cg_(hf, samples, yf, sw, reg, state["en"], ITERS, new_xf, state["st"], False, True,
                                                      (1 - 0.0075) ** 75, 0.0075, 0.3, 0.15)
    med, mn = timeit(run, iters=20, warm=3)
    mem = samples.numel() * 4
    res[name] = {"us_median": med, "us_min": mn, "sample_memory_bytes": mem,
                 "reference_sweep_bytes": 2 * (1 + ITERS) * mem,                      # A = forward + adjoint product, b - A x and 5 x A p
                 "GBps_vs_one_read": mem / med / 1e3, "GBps_vs_reference_sweeps": 2 * (1 + ITERS) * mem / med / 1e3}
    print("%-28s median %8.1f us  min %8.1f us   %.1f MB memory: %.0f GB/s once-per-call, %.0f GB/s in the reference's traffic"
          % (name, med, mn, mem / 1e6, res[name]["GBps_vs_one_read"], res[name]["GBps_vs_reference_sweeps"]))
# first-frame joint optimisation: 30 augmented samples, init_CG_iter 100 / init_GN_iter 10 (parameter/eco/default.py)
JOINT = {"deep 15x8 x 30 x 256 -> 64": (15, 8, 30, 256, 64), "shallow 63x32 x 30 x 96 -> 16": (63, 32, 30, 96, 16)}
for name, (h, wh, n, cin, c) in JOINT.items():
    g = torch.Generator().manual_seed(h + 1)
    samples = torch.randn(h, wh, n, cin, 2, generator=g).cuda()
    P0 = torch.linalg.qr(torch.randn(cin, cin, generator=g))[0][:, :c].contiguous().cuda()
    yf = torch.rand(1, 1, h, wh, generator=g).cuda()
    reg = torch.tensor([[0.0, 0.23, 0.0], [0.16, 0.78, 0.16], [0.0, 0.23, 0.0]]).view(1, 1, 3, 3).cuda()
    sw_sqrt = torch.full((n,), (1.0 / n) ** 0.5).cuda()
    dMh = (torch.rand(1, c, h, wh, generator=g) + 0.5).cuda()

    def runj():
        ops.eco_joint_gn_(torch.zeros(1, c, h, wh, 2).cuda(), P0.clone(), samples, yf, sw_sqrt, reg, dMh, 35.0, 5e-8, 10, 10)
    med, mn = timeit(runj, iters=5, warm=2)
    res["joint " + name] = {"us_median": med, "us_min": mn, "gn_x_cg": "10 x 10", "sample_bytes": samples.numel() * 4}
    print("joint %-32s median %9.1f us  min %9.1f us   (10 GN x 10 CG, %.1f MB of samples)" % (name, med, mn, samples.numel() * 4 / 1e6))
# score computation of a tracked frame (eco.py:194-196): apply_filter of both blocks for 5 scales, sum_fs + sample_fs to 250x250, max2d
try:
    g = torch.Generator().manual_seed(9)
    sblocks = [(63, 32, 16), (15, 8, 64)]
    filt = [(0.1 * torch.randn(1, c, h, wh, 2, generator=g)).cuda() for (h, wh, c) in sblocks]
    xfs = [torch.randn(5, c, h, wh, 2, generator=g).cuda() for (h, wh, c) in sblocks]

    feats = [torch.randn(5, c, hw, hw, generator=g).cuda() for (hw, c) in ((62, 16), (15, 64))]      # projected test samples (eco.py:295)
    wins = [torch.ones(1, 1, hw, hw).cuda() for hw in (62, 15)]                                       # ones: x is windowed in place every call
    interps = [((torch.randn(1, 1, h, 1, 2, generator=g) / h).cuda(), (torch.randn(1, 1, 1, wh, 2, generator=g) / h).cuda()) for (h, wh, _) in sblocks]

    def runs():
        xs = [ops.eco_preprocess_sample_(x, w, iy, ix) for x, w, (iy, ix) in zip(feats, wins, interps)]
        sfs = [ops.eco_apply_filter(f, x) for f, x in zip(filt, xs)]
        ops.max2d(ops.eco_sample_fs(sfs, (250, 250), [1.0, 0.6]))
    med, mn = timeit(runs, iters=20, warm=3)
    nbytes = sum(t.numel() * 4 for t in filt + xfs + feats) + 5 * 250 * 250 * 4
    res["scores 5 scales, 62x62x16 + 15x15x64 features -> 250x250"] = {"us_median": med, "us_min": mn, "bytes": nbytes, "launches": 6}
    print("scores (preprocess_sample x 2 + apply_filter x 2 + sample_fs + max2d) median %8.1f us  min %8.1f us   (%.2f MB in + out)"
          % (med, mn, nbytes / 1e6))
except Exception as e:      # noqa: BLE001 -- the optimiser rows above must survive a defect here
    print("scores row failed: %r" % (e,))
out_path = sys.argv[sys.argv.index("--json") + 1] if "--json" in sys.argv else os.path.join("gpurun_out", "eco_bench.json")
os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
json.dump(res, open(out_path, "w"), indent=1)
