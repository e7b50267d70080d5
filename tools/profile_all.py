"""One launch of every kernel family of the library between cudaProfilerStart / Stop, for a single ncu pass:

    ncu --set full --clock-control none --import-source on --profile-from-start off -o /tmp/profile_all -f python tools/profile_all.py
    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file /tmp/profile_all_launches.csv \
        python tools/profile_all.py frames

Default: each family once at its BASELINE size (SURVEY.md 8(d)).  `frames`: three whole tracked frames of the native tracker (the
launch list whose kernel shares must agree with bench.py's per-kernel timings)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytracking_b200 import ops, synth                       # noqa: E402
from pytracking_b200.engine import BackboneEngine            # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "kernels"


def tracker():
    sys.path.insert(0, os.path.join(ROOT))
    import bench
    from pytracking_b200.tracker import DiMPTracker, make_params
    frames, bb, _ = bench.make_frames(0, bench.PREROLL + 8)
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    trk = DiMPTracker(sd, make_params(**bench.TRACKER_PARAMS))
    trk.initialize(frames[0], {"init_bbox": bb})
    for i in range(1, bench.PREROLL + 4):
        trk.track(frames[i])
    return trk, frames[bench.PREROLL + 4:]


if what == "frames":
    trk, rest = tracker()
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    for f in rest[:3]:
        trk.track(f)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    sys.exit(0)

if what == "convonly":            # one backbone + head forward pass (the 44 conv_tc launches of a frame), eager so that ncu sees plain launches
    os.environ["B200TRK_GRAPH"] = "0"
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    eng = BackboneEngine(sd, arch="resnet50", max_batch=1, crop_size=288)
    im = synth.make_crop(1, 1, 288).cuda()
    for _ in range(3):
        eng.forward(im, want=("classification",))
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    eng.forward(im, want=("classification",))
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    sys.exit(0)

runs = []
p = synth.make_dimp_optimizer_params(seed=3)
luts = [p[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
feat50 = synth.make_clf_features(3, 50, 512, 18, 18).cuda()
bb50 = synth.make_boxes(4, 50).cuda()
sw50 = torch.full((50,), 1.0 / 50).cuda()
w0 = torch.zeros(1, 512, 4, 4).cuda()
runs.append(("sd_tc_kernel DiMP n=50 10it", lambda: ops.dimp_sd_gn(w0, feat50, bb50, sw50, *luts, 10, 0.9, 0.01)))
runs.append(("sd_kernel DiMP n=15 10it", lambda: ops.dimp_sd_gn(w0, feat50[:15], bb50[:15], None, *luts, 10, 0.9, 0.01)))
f22 = synth.make_clf_features(5, 50, 512, 22, 22).cuda()
bb22 = synth.make_boxes(6, 50, center=151.0).cuda()
runs.append(("sd_tc_kernel PrDiMP n=50 22x22 10it", lambda: ops.prdimp_sd_newton(0.01 * torch.ones(1, 512, 4, 4).cuda(), f22, bb22, sw50, 10, 1.1, 1.0,
                                                                                   0.0025, alpha_eps=0.05, normalize_label=True)))
w1 = torch.randn(1, 512, 4, 4).cuda()
runs.append(("apply_filter n=1 (+max2d)", lambda: ops.apply_filter(feat50[:1], w1, return_max=True)))
r50 = torch.randn(50, 1, 19, 19).cuda()
runs.append(("apply_feat_transpose n=50", lambda: ops.apply_feat_transpose(feat50, r50, 4)))
sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
eng = BackboneEngine(sd, arch="resnet50", max_batch=1, crop_size=288)
im = synth.make_crop(1, 1, 288).cuda()
runs.append(("backbone + head (conv_tc chain)", lambda: eng.forward(im, want=("classification",))))
x, y, sw = synth.make_atom_memory(77, 250, 64, 18, 18, n_filled=250)
x, y, sw = x.cuda(), y.cuda(), sw.cuda()
wa = (torch.randn(1, 64, 4, 4) * 0.02).cuda()
out = torch.empty_like(wa)
runs.append(("atom_cg_kernel n=250 C=64 5it", lambda: ops.atom_cg_filter(wa, x, y, sw, 0.1, 5, "mlu", 0.05, False, out=out)))
xi, yi, swi = synth.make_atom_memory(111, 30, 256, 18, 18)
xi, yi, swi = xi.cuda(), yi.cuda(), swi.cuda()
P0 = (torch.randn(64, 256, 1, 1) / 16).cuda()
runs.append(("atom_gn_joint 1 GN x 2 CG", lambda: ops.atom_gn_joint_(torch.zeros(1, 64, 4, 4, device="cuda"), P0.clone(), xi, yi, swi, 0.1, 1e-4, 2, 1,
                                                                    "mlu", 0.05, True)))
s5 = torch.randn(5, 256, 18, 18).cuda()
Pm = (torch.randn(64, 256, 1, 1) * 0.05).cuda()


def atom_stage2():
    xn = ops.feature_normalize_(s5.clone(), 2.0)
    sc = ops.conv2d_same(ops.conv1x1(xn, Pm), wa)
    return ops.max2d(ops.fourier_interp(sc, (4, 4), (288, 288))[:, 0])


runs.append(("ATOM stage 2 (normalise, conv1x1, conv2d_same, fourier_interp, max2d)", atom_stage2))
fr = torch.relu(torch.randn(1, 256, 36, 36)).cuda()
rois = torch.tensor([[0, 60.0, 70.0, 150.0, 140.0]] * 10).cuda()


def prroi():
    o = ops.prroi_pool_forward(fr, rois, 5, 5, 1 / 8)
    ops.prroi_pool_backward(fr, rois, o, torch.ones_like(o), 5, 5, 1 / 8)
    ops.prroi_pool_coor_backward(fr, rois, o, torch.ones_like(o), 5, 5, 1 / 8)


runs.append(("prroi forward / backward / coor_backward R=10 256x36x36", prroi))
from pytracking_b200.transformer_engine import TransformerEngine   # noqa: E402
tsd = synth.make_transformer_state_dict(95, 256, 8, 2048, 6, 6)
te = TransformerEngine(tsd, 972, 2, 256, 8, 2048, 6, 6)
src, pos, qe = torch.randn(972, 2, 256).cuda(), (torch.randn(972, 1, 256) * 0.5).cuda(), torch.randn(1, 256).cuda()
runs.append(("ToMP transformer 972x2 (attention_kernel, layernorm, conv_tc GEMMs)", lambda: te.forward(src, None, qe, pos)))
try:
    from baseline import ref_env, ref_tracker
    if ref_env.reference_available():
        from pytracking_b200.iou import IoUPredictor
        net = ref_tracker.build_dimp_net()
        pred = IoUPredictor(net.state_dict())
        f3, f4 = torch.relu(torch.randn(1, 256, 36, 36)).cuda(), torch.relu(torch.randn(1, 256, 18, 18)).cuda()
        mod = [torch.rand(256).cuda(), torch.rand(256).cuda()]
        boxes = torch.tensor([[100.0, 110.0, 70.0, 55.0]] * 10).cuda()
        runs.append(("iou_refine R=10 5 steps (fc_forward / fc_backward / prroi)", lambda: pred.refine(mod, [f3, f4], boxes, 5, 1.0)))
except Exception as e:      # the IoU head weights come from the staged reference; skip quietly without it
    print("iou family skipped:", repr(e))

for name, fn in runs:       # warm-up (lazy allocations, graphs, attribute settings)
    for _ in range(3):
        fn()
trk, rest = tracker()
torch.cuda.synchronize()
torch.cuda.profiler.start()
trk.track(rest[0])          # sample_patch_kernel, localize_kernel and the frame's kernels in context (first: ncu's -c limit cuts the tail)
for name, fn in runs:
    fn()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("profiled:", [n for n, _ in runs])
