"""-m gpu: precision 2, single-pass TF32 on the tensor cores (conv_tc_kernel<BN + TC_SINGLE>).

Every convolution the tensor-core kernel takes rounds each operand once to TF32 (cvt.rna) and accumulates one product per K step
in fp32. For every such layer, on the operands the kernel read (`b200trk_net_op_io` / `_op_output` / `_op_weights`), two float64
results are formed: R_t on the cvt.rna-rounded operands, R_raw on the raw ones. Each layer must satisfy
    max|D - R_t| / max|R_t|  <=  (1/16) max|R_t - R_raw| / max|R_raw|
i.e. the kernel sits much closer to the exact product of its rounded operands than rounding moves that product: a 3xTF32 layer,
a truncated operand or a lost MMA all fail it. The one exception is a long accumulation chain: the tensor core's fp32 accumulator
loses more than IEEE summation would, and on the unsplit 3x3 1024 -> 512 head (one chain of K = 9216 products per CTA, batch 16) the
ratio reached 0.073 on an H100 80GB HBM3 (700 W). Chains longer than 4608 products per CTA are therefore held to 1/8, which the
failures above still exceed several times over. The cases reach the launch plans of tests/test_tc_conv_layers_gpu.py through the same
switches, and the file asserts which plan features were reached. Further: bitwise repeatability, CUDA-graph replay, batch-row
permutation, the batch tracker against the solo tracker, tracking accuracy against precision 0, refusals and device memory."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from pytracking_b200 import _lib, synth
from pytracking_b200.engine import BackboneEngine
from test_tc_conv_layers_gpu import OP_CONV, _crop, _forward, _grid, _output, _plan, _reference, _tc_outputs, _weights

pytestmark = pytest.mark.gpu

TINY = 1e-30
REACHED = set()


def _ratio(y, x, w, b, res, stride, pad, relu):
    """max|D - R_t| / max|R_t| over max|R_t - R_raw| / max|R_raw|, NHWC operands."""
    r_raw, _, r_t = _reference(x, w, b, res, stride, pad, relu)
    d = float((y.double() - r_t).abs().max() / (r_t.abs().max() + TINY))
    moved = float((r_t - r_raw).abs().max() / (r_raw.abs().max() + TINY))
    assert bool(torch.isfinite(y).all())
    return d / max(moved, TINY), d, moved


def _reduction(eng, i):
    m = C.c_int()
    _lib.check(_lib.lib().b200trk_net_op_splitk_reduction(eng.handle, i, C.byref(m)), "net_op_splitk_reduction")
    return m.value


def _check_plan(eng, S, rows, label, only=None):
    """Every tensor-core step of the last forward pass (or the steps in `only`) against the rounded / raw float64 pair."""
    steps = _plan(eng)
    info_of = {i: info for i, info, _ in steps}
    recs = []
    for i, info, io in steps:
        if info[0] != OP_CONV or not info[7] or (only is not None and i not in only):
            continue
        y = _output(eng, i, info, S)[list(rows)]
        x = _output(eng, io[0], info_of[io[0]], S)[list(rows)]
        res = _output(eng, io[1], info_of[io[1]], S)[list(rows)] if io[1] >= 0 else None
        w, b = _weights(eng, i, info)
        ratio, d, moved = _ratio(y, x, w, b, res, info[4], io[3], io[2])
        g = _grid(eng, i)
        K = info[3] * info[3] * info[1]
        chain = -(-K // 32 // g[2]) * 32                          # products one CTA accumulates (k-blocks of the first split)
        recs.append(dict(index=i, K=K, chain=chain, limit=1.0 / 16 if chain <= 4608 else 1.0 / 8, grid=g, red=_reduction(eng, i),
                         ratio=ratio, d=d, moved=moved))
    assert recs, "%s: no step runs on the tensor cores" % label
    worst = max(recs, key=lambda r: r["ratio"])
    short = [r["ratio"] for r in recs if r["chain"] <= 4608]
    print("%s: %d layers, worst ratio %.4f (step %d, grid %s, chain %d, d %.2e, rounding %.2e); worst at chains <= 4608: %.4f" % (
        label, len(recs), worst["ratio"], worst["index"], worst["grid"], worst["chain"], worst["d"], worst["moved"], max(short or [0.0])))
    for r in recs:
        assert r["ratio"] <= r["limit"], "%s step %d (grid %s, chain %d): %.4f" % (label, r["index"], r["grid"], r["chain"], r["ratio"])
        g = r["grid"]
        if r["red"] == 1:
            REACHED.add("cluster split-K")
        if r["red"] == 2:
            REACHED.add("workspace split-K")
        if g[2] > 1 and (r["K"] // 32) % g[2] != 0:
            REACHED.add("uneven last split")
        if g[2] == 1:
            REACHED.add("BN %d unsplit" % g[3])
    return recs


R288 = dict(arch="resnet50", crop=(288, 288), S=1)
CASES = {
    "r50_288_s1_iou": dict(R288, iou=True),
    "r50_288_s5": dict(R288, S=5, rows=(0, 4)),
    "r50_288_s16": dict(R288, S=16, rows=(0, 15)),
    "prdimp_352_s1": dict(R288, crop=(352, 352)),
    "prdimp_352_s5": dict(R288, crop=(352, 352), S=5, rows=(0, 4)),
    "prdimp_352_s16": dict(R288, crop=(352, 352), S=16, rows=(0, 15)),
    "r18_288": dict(R288, arch="resnet18"),
    "cluster0": dict(R288, env={"B200TRK_TC_CLUSTER": "0"}),
    "minkb1": dict(R288, env={"B200TRK_TC_MINKB": "1"}),
    "bn64_nosplitk": dict(R288, env={"B200TRK_TC_BN": "64", "B200TRK_TC_SPLITK": "0"}),
    "bn128_nosplitk": dict(R288, env={"B200TRK_TC_BN": "128", "B200TRK_TC_SPLITK": "0"}),
}


@pytest.mark.parametrize("name", list(CASES))
def test_layers_vs_float64(name, monkeypatch):
    c = CASES[name]
    for k, v in c.get("env", {}).items():
        monkeypatch.setenv(k, v)
    S = c["S"]
    sd = synth.make_dimp_state_dict(c["arch"], seed=0, lut_seed=3)
    if c.get("iou"):
        from ref_weights import GOLDEN, iou_state_dict
        sd = iou_state_dict(np.load(GOLDEN))
    eng = BackboneEngine(sd, arch=c["arch"], max_batch=S, crop_size=c["crop"], precision=2)
    try:
        if c.get("iou"):
            eng.attach_iou_head(sd)
        _forward(eng, _crop(11, S, c["crop"]), c.get("iou", False))
        _check_plan(eng, S, c.get("rows", range(S)), name)
    finally:
        eng.close()


def test_plan_features_reached():
    """Runs after the cases above (file order): the single-pass kernel was checked on every plan feature."""
    need = {"cluster split-K", "workspace split-K", "uneven last split", "BN 64 unsplit", "BN 128 unsplit"}
    assert need <= REACHED, sorted(need - REACHED)


def test_first_frame_heads_vs_float64():
    """filter_conv (FilterInitializerLinear) and conv3_1r / conv4_1r (the IoUNet reference branch) follow the handle's precision."""
    from pytracking_b200.iou import IoUModulation
    from test_iou_modulation_gpu import _setup
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    S, H = 3, 18
    eng = BackboneEngine(sd, "resnet50", 4, S, 16 * H, 2)
    try:
        eng.attach_filter_init(sd, 4, False, False)
        feat = synth.make_clf_features(10, S, 512, H, H).cuda()
        boxes = np.array([[0.3, 0.35, 0.25, 0.2], [-0.08, 0.4, 0.2, 0.15], [0.9, 0.2, 0.2, 0.3]], np.float32) * 16 * H
        eng.filter_init(feat, boxes)
        torch.cuda.synchronize()
        last = _lib.lib().b200trk_net_num_ops(eng.handle) - 1
        _check_plan(eng, S, range(S), "filter_conv", only={last})
    finally:
        eng.close()
    _, sd, _, _ = _setup()
    eng = BackboneEngine(sd, "resnet50", 4, S, 352, 2)
    try:
        eng.attach_iou_ref(sd)
        head = IoUModulation(sd)
        eng.forward(synth.make_crop(11, S, 352).cuda(), want=("classification",))
        head.get(eng, S, np.array([[100, 120, 90, 70], [-20, 150, 80, 60], [300, 10, 40, 110]], np.float32))
        torch.cuda.synchronize()
        n = _lib.lib().b200trk_net_num_ops(eng.handle)
        assert len(_check_plan(eng, S, range(S), "conv3_1r/conv4_1r", only={n - 2, n - 1})) == 2
    finally:
        eng.close()


def test_tomp_tower_convolutions_vs_float64():
    from pytracking_b200.transformer_engine import BoxTower
    from ref_weights import GOLDEN, tower_state_dict
    sd = tower_state_dict(np.load(GOLDEN))
    tw = BoxTower(sd, 18, 18, max_batch=4, precision=2)
    L = _lib.lib()
    try:
        n = L.b200trk_tower_debug_num_launches(tw.handle)
        nconv = (n - 1) // 2
        for S in (1, 4):
            g = torch.Generator().manual_seed(20 + S)
            feat = (torch.randn(S, 256, 18, 18, generator=g) * 0.3).cuda()
            att = torch.rand(S, 18, 18, generator=g).cuda()

            def buf(i, c):
                t = torch.empty(S, 18, 18, c, device="cuda")
                _lib.check(L.b200trk_tower_debug_buffer(tw.handle, i, S, C.c_void_p(t.data_ptr()), None), "tower_debug_buffer")
                torch.cuda.synchronize()
                return t
            ntc = 0
            for ci in range(nconv):
                info = (C.c_int * 10)()
                _lib.check(L.b200trk_tower_debug_conv(tw.handle, ci, C.byref(info)), "tower_debug_conv")
                if not info[2]:
                    continue
                k = 1 + 2 * ci                                    # the launch of convolution ci
                _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k - 1), "tower_debug_stop_after")
                tw.forward(feat, att)
                x = buf(ci, 256)
                _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k), "tower_debug_stop_after")
                tw.forward(feat, att)
                y = buf(ci + 1, info[1])
                key = "tower.%d" % (3 * ci)
                w = sd[key + ".weight"].float().permute(0, 2, 3, 1).contiguous().cuda()
                ratio, d, moved = _ratio(y, x, w, sd[key + ".bias"].float().cuda(), None, 1, 1, False)
                print("tower S=%d conv %d grid %s: ratio %.4f" % (S, ci, list(info[3:7]), ratio))
                assert ratio <= 1.0 / 16, (S, ci, ratio)
                ntc += 1
            assert ntc >= 1
            _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, -1), "tower_debug_stop_after")
    finally:
        tw.close()


# ---- bitwise properties -------------------------------------------------------------------------------------------------------------
def _net_forward(eng, im, outs):
    _lib.check(_lib.lib().b200trk_net_forward_iou(eng.handle, C.c_void_p(im.data_ptr()), im.shape[0],
                                                  *[C.c_void_p(t.data_ptr()) for t in outs], None, None,
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)), "net_forward")
    torch.cuda.synchronize()


def test_repeat_graph_replay_and_row_permutation_are_bitwise():
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    S = 5
    eng = BackboneEngine(sd, "resnet50", 4, S, 288, 2)
    try:
        im = _crop(21, S, (288, 288))
        d = eng.dims
        outs = [torch.empty(S, d[3 * i], d[3 * i + 1], d[3 * i + 2], device="cuda") for i in range(3)]
        steps = _plan(eng)
        runs = []
        for _ in range(5):      # calls 1-2 eager, 3 records the CUDA graph, 4-5 replay it (same pointers)
            _net_forward(eng, im, outs)
            runs.append(([o.clone() for o in outs], _tc_outputs(eng, steps, S)))
        for r in runs[1:]:
            for a, b in zip(r[0], runs[0][0]):
                assert torch.equal(a, b), "a repeat / the graph replay differs from the first eager pass"
            for i, y in r[1].items():
                assert torch.equal(y, runs[0][1][i]), "step %d differs between passes" % i
        perm = [3, 0, 4, 2, 1]
        eng.forward(im[perm].contiguous())
        torch.cuda.synchronize()
        py = _tc_outputs(eng, steps, S)
        for i, y in py.items():
            assert torch.equal(y, runs[0][1][i][perm]), "step %d: permuting the batch rows does not permute the output" % i
    finally:
        eng.close()


@pytest.mark.parametrize("kind", ["dimp", "prdimp"])
def test_batch_capacity_one_equals_solo_tracker_bitwise(kind):
    from pytracking_b200.batch import DiMPBatchTracker
    from pytracking_b200.tracker import DiMPTracker, make_params
    from test_batch_tracker_gpu import BENCH, PRDIMP, _bits, _sd, _seq
    cfg, newton = (BENCH, None) if kind == "dimp" else (PRDIMP, {})
    frames, bb = _seq(0, 60)
    trk = DiMPTracker(_sd(), make_params(**cfg), newton=newton, precision=2)
    trk.initialize(frames[0], {"init_bbox": bb})
    solo = [(list(bb), 0, None, _bits(trk.engine.filter))]
    for f in frames[1:]:
        box = trk.track(f)["target_bbox"]
        solo.append((box, int(trk.info.flag), _bits(trk.engine.scores[0]), _bits(trk.engine.filter)))
    trk.close()
    bt = DiMPBatchTracker(_sd(), make_params(**cfg), 1, newton=newton, precision=2)
    bt.step({0: (frames[0], {"init_bbox": bb})})
    assert np.array_equal(_bits(bt.filter(0)), solo[0][3])
    for t in range(1, len(frames)):
        out = bt.step({0: (frames[t], None)})
        box, flag, scores, filt = solo[t]
        assert out[0]["target_bbox"] == box, (kind, t)
        assert int(bt.last_info[0].flag) == flag, (kind, t)
        assert np.array_equal(_bits(bt.scores(0)), scores), (kind, t)
        assert np.array_equal(_bits(bt.filter(0)), filt), (kind, t)
    bt.close()


# ---- trackers --------------------------------------------------------------------------------------------------------------------
def _iou(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    x0, y0 = np.maximum(a[:, 0], b[:, 0]), np.maximum(a[:, 1], b[:, 1])
    x1, y1 = np.minimum(a[:, 0] + a[:, 2], b[:, 0] + b[:, 2]), np.minimum(a[:, 1] + a[:, 3], b[:, 1] + b[:, 3])
    inter = np.clip(x1 - x0, 0, None) * np.clip(y1 - y0, 0, None)
    return inter / (a[:, 2] * a[:, 3] + b[:, 2] * b[:, 3] - inter)


@pytest.mark.parametrize("kind", ["dimp", "prdimp"])
def test_tracker_mean_iou_within_001_of_precision_0(kind):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from pytracking_b200.tracker import DiMPTracker, make_params
    from test_batch_tracker_gpu import PRDIMP
    cfg, newton = (bench.TRACKER_PARAMS, None) if kind == "dimp" else (dict(bench.TRACKER_PARAMS, **{k: PRDIMP[k] for k in (
        "image_sample_size", "search_area_scale", "border_mode", "patch_max_scale_change", "score_preprocess")}), {})
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    mean = {}
    for precision in (0, 2):
        ious = []
        for q in range(3):
            frames, bb, gt = bench.make_frames(q, 60)
            trk = DiMPTracker(sd, make_params(**cfg), newton=newton, precision=precision)
            trk.initialize(frames[0], {"init_bbox": bb})
            boxes = [trk.track(f)["target_bbox"] for f in frames[1:]]
            trk.close()
            ious.append(_iou(boxes, np.asarray(gt)[1:len(frames)]))
        mean[precision] = float(np.concatenate(ious).mean())
    print("%s mean IoU over 3 x 60 frames: precision 0 %.4f, precision 2 %.4f" % (kind, mean[0], mean[2]))
    assert abs(mean[2] - mean[0]) <= 0.01, mean


# ---- refusals and memory -----------------------------------------------------------------------------------------------------------
def test_out_of_range_precisions_are_refused_without_allocating():
    from pytracking_b200.engine import ARCH_ID, conv_descs_from_state_dict
    from pytracking_b200.transformer_engine import BoxTower
    from ref_weights import GOLDEN, tower_state_dict
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    tsd = tower_state_dict(np.load(GOLDEN))
    descs, keep = conv_descs_from_state_dict(sd, "resnet50", head=True)
    arr = (_lib.ConvDesc * len(descs))(*descs)
    L = _lib.lib()
    torch.cuda.synchronize()
    for p in (3, -1):
        free0 = torch.cuda.mem_get_info()[0]
        h = C.c_void_p()
        assert L.b200trk_net_create(C.byref(h), ARCH_ID["resnet50"], arr, len(descs), 1.0, 1, 288, 288, p) != 0
        assert not h.value
        assert b"precision" in L.b200trk_last_error()
        with pytest.raises(RuntimeError, match="precision"):
            BoxTower(tsd, 18, 18, max_batch=1, precision=p)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0, "a refused create changed the device memory"
    # the refusals left nothing behind: a valid plan still builds and runs
    eng = BackboneEngine(sd, "resnet50", 4, 1, 96, 2)
    eng.forward(_crop(3, 1, (96, 96)))
    eng.close()
    del keep


def test_precision_2_plan_holds_no_split_weight_copy():
    from pytracking_b200.engine import conv_descs_from_state_dict
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    used = {}
    for p in (0, 2):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        eng = BackboneEngine(sd, "resnet50", 4, 1, 288, p)
        torch.cuda.synchronize()
        used[p] = free0 - torch.cuda.mem_get_info()[0]
        # the B operand of every tensor-core step: K x Cout floats (the hi | lo copy holds twice that)
        if p == 2:
            nw = sum(info[2] * info[3] * info[3] * info[1] for _, info, _ in _plan(eng) if info[0] == OP_CONV and info[7])
        eng.close()
    saved = used[0] - used[2]
    print("device memory of a DiMP-50 plan at 288: precision 0 %.1f MB, precision 2 %.1f MB, saved %.1f MB (one weight copy: %.1f MB)" % (
        used[0] / 1e6, used[2] / 1e6, saved / 1e6, 4 * nw / 1e6))
    assert abs(saved - 4 * nw) <= 0.05 * 4 * nw, (saved, 4 * nw)
