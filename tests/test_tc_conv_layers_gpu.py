"""-m gpu: every tensor-core convolution of the network plan (conv_tc.cu), layer by layer, against a float64 reference of the same
operation on the operands the kernel consumed -- across the launch plans `tc_configure` can choose.

For each step that runs on the tensor cores, the step's input, residual and folded weights are read back from the handle
(`b200trk_net_op_io`, `b200trk_net_op_output`, `b200trk_net_op_weights`) and three float64 quantities are formed with torch's conv2d:
  z64    = relu?(conv(x, w) + b + res)                      the exact result of the layer
  m      = conv(|x|, |w|) + |b| + |res|                      the magnitude that normalises the error
  z_tf32 = relu?(conv(tf32(x), tf32(w)) + b + res)           a plain TF32 GEMM on the same operands (cvt.rna emulated bitwise)
With e = max |y - z64| / m and e_tf32 the same for z_tf32, every layer must satisfy
  e <= e_tf32 / 16                                           3xTF32 error compensation in place (losing a correction product or
                                                             the second accumulator leaves an error of the size of e_tf32)
  e <= (K + 2) 2^-23 + 2^-20,  K = k*k*Cin                   worst case of fp32 summation (truncating accumulation included)
                                                             plus the dropped lo*lo term: a ceiling for wrong tiles and NaNs
and each case asserts, through `b200trk_net_op_grid`, that it reached the launch plan it is named for.

Where e / e_tf32 is largest: the 3x3 1024 -> 512 classification head launched without split-K (batch 13, or B200TRK_TC_SPLITK=0),
where one fp32 accumulator chain runs over all K = 9216 products; its fp32 summation error grows with the chain while e_tf32 shrinks
as 1 / sqrt(K). Measured on an H100 80GB HBM3 (700 W): 0.057 there, at most 0.012 on every other plan's worst layer."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from pytracking_b200 import _lib, synth
from pytracking_b200.engine import BackboneEngine

pytestmark = pytest.mark.gpu

OP_CONV, OP_L2NORM = 3, 5
TINY = 1e-30


def _tf32(x):
    """float32 -> nearest TF32 value (10 explicit mantissa bits), ties away from zero: what cvt.rna.tf32.f32 computes. Adding half
    a unit of the 13 dropped bits to the sign-magnitude pattern rounds the magnitude, then the dropped bits are cleared."""
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def _pick_tile(wout, hout, stride):
    """The pixel rectangle conv_tc.cu's pick_tile chooses (checked against the launched grid.x wherever it is used)."""
    best, bw_, bh_ = -1.0, 0, 0
    for bw in range(1, min(wout, 128) + 1):
        if bw * stride > 256:
            break
        bh = min(128 // bw, hout)
        if bh * stride > 256:
            bh = 256 // stride
        if bh < 1:
            continue
        eff = wout * hout / (((wout + bw - 1) // bw) * ((hout + bh - 1) // bh) * 128.0)
        if eff > best + 1e-9:
            best, bw_, bh_ = eff, bw, bh
    return bw_, bh_


def _plan(eng):
    """[(index, info, io)] of every plan step."""
    L = _lib.lib()
    steps = []
    for i in range(L.b200trk_net_num_ops(eng.handle)):
        info, io = (C.c_int * 8)(), (C.c_int * 4)()
        _lib.check(L.b200trk_net_op_info(eng.handle, i, C.byref(info)), "net_op_info")
        _lib.check(L.b200trk_net_op_io(eng.handle, i, C.byref(io)), "net_op_io")
        steps.append((i, list(info), list(io)))
    return steps


def _output(eng, index, info, S):
    """NHWC output [S, Hout, Wout, Cout] of plan step `index` after the last forward pass."""
    t = torch.empty(S, info[5], info[6], info[2], device="cuda")
    _lib.check(_lib.lib().b200trk_net_op_output(eng.handle, index, S, C.c_void_p(t.data_ptr()), None), "net_op_output")
    return t


def _weights(eng, index, info):
    cout, cin, k = info[2], info[1], info[3]
    w = torch.empty(cout, k, k, cin, device="cuda")
    b = torch.zeros(cout, device="cuda")
    _lib.check(_lib.lib().b200trk_net_op_weights(eng.handle, index, C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()), None),
               "net_op_weights")
    return w, b


def _grid(eng, index):
    g = (C.c_int * 4)()
    _lib.check(_lib.lib().b200trk_net_op_grid(eng.handle, index, C.byref(g)), "net_op_grid")
    return list(g)


def _reference(x, w, b, res, stride, pad, relu):
    """(z64, m, z_tf32), NHWC float64, from NHWC float32 operands."""
    def conv(a, f):
        return F.conv2d(a.permute(0, 3, 1, 2).double(), f.permute(0, 3, 1, 2).double(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    bd = b.double()
    z, m, zt = conv(x, w) + bd, conv(x.abs(), w.abs()) + bd.abs(), conv(_tf32(x), _tf32(w)) + bd
    if res is not None:
        r = res.double()
        z, m, zt = z + r, m + r.abs(), zt + r
    if relu:
        z, zt = z.clamp(min=0), zt.clamp(min=0)
    return z, m, zt


def _forward(eng, im, iou):
    want = ("layer2", "layer3", "classification") + (("iou3", "iou4") if iou else ())
    out = eng.forward(im, want=want)
    torch.cuda.synchronize()
    return out


def _tc_outputs(eng, steps, S):
    return {i: _output(eng, i, info, S) for i, info, _ in steps if info[0] == OP_CONV and info[7]}


def _check_layers(eng, steps, S, rows, label):
    """Compares every tensor-core step of the last forward pass (batch S, batch rows `rows`) with its float64 reference; returns one
    record per step."""
    info_of = {i: info for i, info, _ in steps}
    clf_index = max([i for i, info, _ in steps if info[0] == OP_L2NORM], default=len(steps))
    recs = []
    for i, info, io in steps:
        if info[0] != OP_CONV or not info[7]:
            continue
        kind, cin, cout, k, stride, ho, wo, _ = info
        y = _output(eng, i, info, S)
        assert bool(torch.isfinite(y).all()), "%s step %d: NaN / Inf in the output" % (label, i)
        x = _output(eng, io[0], info_of[io[0]], S)[list(rows)]
        res = _output(eng, io[1], info_of[io[1]], S)[list(rows)] if io[1] >= 0 else None
        w, b = _weights(eng, i, info)
        z, m, zt = _reference(x, w, b, res, stride, io[3], io[2])
        yd = y[list(rows)].double()
        e = float(((yd - z).abs() / (m + TINY)).max())
        e_tf32 = float(((zt - z).abs() / (m + TINY)).max())
        K = k * k * cin
        recs.append(dict(index=i, cin=cin, cout=cout, k=k, stride=stride, ho=ho, wo=wo, io=io, grid=_grid(eng, i), K=K, e=e,
                         e_tf32=e_tf32, ratio=e / max(e_tf32, TINY), iou=i > clf_index))
    assert recs, "%s: no step runs on the tensor cores" % label
    for r in recs:
        print("%s step %3d %4d->%4d k%d s%d %3dx%-3d grid %-16s e %.2e  e_tf32 %.2e  e/e_tf32 %.4f" % (
            label, r["index"], r["cin"], r["cout"], r["k"], r["stride"], r["ho"], r["wo"], r["grid"], r["e"], r["e_tf32"], r["ratio"]))
    we, wr = max(recs, key=lambda r: r["e"]), max(recs, key=lambda r: r["ratio"])
    print("%s: %d layers; worst e %.2e (step %d), worst e/e_tf32 %.4f (step %d)" % (label, len(recs), we["e"], we["index"], wr["ratio"],
                                                                                       wr["index"]))
    for r in recs:
        assert r["e"] <= r["e_tf32"] / 16, "%s step %d: e %.3e is not 16x below plain TF32 (%.3e)" % (label, r["index"], r["e"], r["e_tf32"])
        bound = (r["K"] + 2) * 2.0 ** -23 + 2.0 ** -20
        assert r["e"] <= bound, "%s step %d: e %.3e above the fp32 summation bound %.3e" % (label, r["index"], r["e"], bound)
    return recs


def _crop(seed, S, crop):
    h, w = crop
    return synth.make_crop(seed, S, max(h, w))[:, :, :h, :w].contiguous().cuda()


# ---- what each case must reach ------------------------------------------------------------------------------------------------
def _reaches_bench_plan(recs, S):
    assert any(1 < r["grid"][2] <= 8 and r["ho"] == 18 for r in recs), "no cluster split-K on the 18x18 layers"
    head = [r for r in recs if not r["iou"] and r["cin"] == 1024 and r["cout"] == 512 and r["k"] == 3]
    assert len(head) == 1 and head[0]["grid"][3] == 128, "the classification head is not a BN = 128 launch"
    iou = [r for r in recs if r["iou"]]
    assert len(iou) == 4, "IoU convolutions missing"
    assert sorted(r["cin"] for r in iou[0::2]) == [512, 1024], "IoU convolutions not fed by layer2 / layer3"


def _reaches_batch13(recs, S):
    assert all(r["grid"][2] == 1 for r in recs), "S = 13 fills the GPU without split-K"
    assert any(r["grid"][3] == 128 for r in recs)


def _reaches_22x22(recs, S):
    assert any(r["ho"] == 22 and r["wo"] == 22 for r in recs)


def _reaches_basic_blocks(recs, S):
    assert any(r["k"] == 3 and r["io"][1] >= 0 for r in recs), "no basic-block convolution with a residual"
    assert sum(1 for r in recs if r["cin"] == 256 and r["cout"] == 256 and r["k"] == 3 and r["ho"] == 18) >= 3


def _reaches_partial_tiles(recs, S):
    both = 0
    for r in recs:
        assert r["ho"] != r["wo"]
        bw, bh = _pick_tile(r["wo"], r["ho"], r["stride"])
        tw, th = (r["wo"] + bw - 1) // bw, (r["ho"] + bh - 1) // bh
        assert r["grid"][0] == tw * th * S, "tile mirror out of date for step %d" % r["index"]
        both += r["wo"] % bw != 0 and r["ho"] % bh != 0
    assert both > 0, "no layer with partial tiles in both directions"


def _reaches_small_maps(recs, S):
    assert any(r["ho"] * r["wo"] < 128 for r in recs)
    assert max(r["grid"][2] for r in recs) == 8


def _reaches_workspace(recs, S):
    assert any(r["grid"][2] > 8 for r in recs), "no split-K beyond the cluster size (L2 workspace path)"


def _reaches_uneven_split(recs, S):
    assert any(r["grid"][2] > 1 and (r["K"] // 32) % r["grid"][2] != 0 for r in recs), "no uneven last split"


def _all_bn(bn):
    def check(recs, S):
        for r in recs:
            assert r["grid"][3] == (bn if r["cout"] % bn == 0 else 64), r
    return check


def _no_splitk(recs, S):
    assert all(r["grid"][2] == 1 for r in recs)


R288 = dict(arch="resnet50", crop=(288, 288), S=1)
CASES = {
    "r50_288_s1_iou": dict(R288, iou=True, reach=_reaches_bench_plan, repeat=True),
    "r50_288_s13": dict(R288, S=13, rows=(0, 12), reach=_reaches_batch13),
    "r50_352": dict(R288, crop=(352, 352), reach=_reaches_22x22),
    "r18_288": dict(R288, arch="resnet18", reach=_reaches_basic_blocks),
    "r50_272x352": dict(R288, crop=(272, 352), reach=_reaches_partial_tiles),      # 68x88, 34x44: partial tiles both ways
    "r50_96_s2": dict(R288, crop=(96, 96), S=2, reach=_reaches_small_maps),
    "cluster0": dict(R288, env={"B200TRK_TC_CLUSTER": "0"}, reach=_reaches_workspace, repeat=True),
    "minkb1": dict(R288, env={"B200TRK_TC_MINKB": "1"}, reach=_reaches_uneven_split, repeat=True),
    "bn64": dict(R288, env={"B200TRK_TC_BN": "64"}, reach=_all_bn(64)),
    "bn128": dict(R288, env={"B200TRK_TC_BN": "128"}, reach=_all_bn(128)),
    "nosplitk": dict(R288, env={"B200TRK_TC_SPLITK": "0"}, reach=_no_splitk),
}


def _run_case(name, setenv):
    c = CASES[name]
    for k, v in c.get("env", {}).items():
        setenv(k, v)
    S = c["S"]
    sd = synth.make_dimp_state_dict(c["arch"], seed=0, lut_seed=3)
    if c.get("iou"):
        from ref_weights import GOLDEN, iou_state_dict
        import numpy as np
        sd = iou_state_dict(np.load(GOLDEN))
    eng = BackboneEngine(sd, arch=c["arch"], max_batch=S, crop_size=c["crop"], precision=0)
    try:
        if c.get("iou"):
            eng.attach_iou_head(sd)
        im = _crop(11, S, c["crop"])
        _forward(eng, im, c.get("iou", False))
        steps = _plan(eng)
        recs = _check_layers(eng, steps, S, c.get("rows", range(S)), name)
        c["reach"](recs, S)
        if c.get("repeat"):
            # every plan reduces its split-K partials in a fixed order: a second pass is bitwise identical, layer by layer
            first = _tc_outputs(eng, steps, S)
            _forward(eng, im, c.get("iou", False))
            for i, y in _tc_outputs(eng, steps, S).items():
                assert torch.equal(y, first[i]), "%s step %d: two passes of the same crop differ" % (name, i)
    finally:
        eng.close()


@pytest.mark.parametrize("name", sorted(CASES))
def test_tc_conv_layers_vs_float64(name, monkeypatch):
    _run_case(name, monkeypatch.setenv)


def test_tc_conv_batch_size_switch_on_one_handle():
    """S = 1 -> 13 -> 1 on one handle re-configures every tensor-core step (tile count, BN, split-K, weight tensor map) twice. The
    two S = 1 passes are bitwise identical; row 0 of the S = 13 pass (the same crop) is each layer's S = 1 output within the fp32
    summation bound, and every layer of the S = 13 pass is checked against float64 on rows 0 and 12."""
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    eng = BackboneEngine(sd, arch="resnet50", max_batch=13, crop_size=288, precision=0)
    try:
        im1 = _crop(11, 1, (288, 288))
        im13 = torch.cat([im1, _crop(12, 12, (288, 288))])
        _forward(eng, im1, False)
        steps = _plan(eng)
        recs1 = _check_layers(eng, steps, 1, range(1), "switch S=1")
        y1 = _tc_outputs(eng, steps, 1)
        _forward(eng, im13, False)
        recs13 = _check_layers(eng, steps, 13, (0, 12), "switch S=13")
        y13 = _tc_outputs(eng, steps, 13)
        assert any(a["grid"][1:] != b["grid"][1:] for a, b in zip(recs1, recs13)), "S = 13 did not change any plan"
        _forward(eng, im1, False)
        y1b = _tc_outputs(eng, steps, 1)
        info_of = {i: (info, io) for i, info, io in steps}
        for r in recs1:
            i = r["index"]
            assert torch.equal(y1b[i], y1[i]), "step %d: S = 1 after S = 13 differs from the first S = 1 pass" % i
            info, io = info_of[i]
            x = _output(eng, io[0], info_of[io[0]][0], 1)
            res = _output(eng, io[1], info_of[io[1]][0], 1) if io[1] >= 0 else None
            w, b = _weights(eng, i, info)
            _, m, _ = _reference(x, w, b, res, info[4], io[3], io[2])
            d = float(((y13[i][:1].double() - y1[i].double()).abs() / (m + TINY)).max())
            assert d <= (r["K"] + 2) * 2.0 ** -23 + 2.0 ** -20, "step %d: row 0 of S = 13 is %.3e from S = 1" % (i, d)
    finally:
        eng.close()
