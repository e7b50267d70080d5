"""-m gpu: every step of the network plan (net.cu) at every batch size the lock-step batch runs (S = 1..16), row by row, against a
reference of the same operation on the operands the step read back (`b200trk_net_op_io`, `_op_output`, `_op_weights`).

One network of max_batch 16 per configuration is stepped through the batch sizes on the same handle; every row of a batch is a
different seeded crop, and rows {0, S // 2, S - 1} are compared:
  OP_PREPROCESS     torch-CPU float32 (x / 255 - mean) / std in the reference's order (oracle.dimp_oracle), 4th lane 0   bitwise
  OP_STEM           float64 conv 7x7/2/3 + bias + ReLU of the preprocess output, with conv1 / bn1 folded in double as
                    net.cu's fold_and_repack folds them, then rounded to float32                   e <= (K + 2) 2^-23 + 2^-20
  OP_MAXPOOL        F.max_pool2d(3, 2, 1) of the stem output                                                          bitwise
  OP_CONV, wgmma    test_tc_conv_layers_gpu._check_layers: 16x below a plain TF32 GEMM, and the fp32 summation bound
  OP_CONV, fp32     float64 conv of its operands                                                   e <= (K + 2) 2^-23 + 2^-20
  OP_EXPORT_NCHW    permute of the producer's NHWC output                                                             bitwise
  OP_L2NORM_EXPORT  float64 InstanceL2Norm of the head's NHWC output with the net's float32 norm_scale    _l2norm_bound below
e is the error normalised by conv(|x|, |w|) + |b| (+ |res|), as in test_tc_conv_layers_gpu: K products summed in fp32 in any order
are off by at most (K - 1) u of that magnitude (u = 2^-24), plus the bias / residual adds and the output rounding; (K + 2) 2^-23
doubles that, and 2^-20 absorbs the 3xTF32 split's dropped lo * lo term.

And at every S:
  * permuting the rows of the batch permutes every step's output rows, both exports and `classification` bit for bit (DESIGN 4.10:
    every output tile belongs to one sample and split-K sums in a fixed order), for the reversed order and a rotation by one;
  * the second eager pass, the third (recorded into the network's CUDA graph and replayed) and a fourth (a plain replay) equal the
    first eager pass bit for bit, step by step;
  * one line per S lists every tensor-core step's launch {grid.x, grid.y, grid.z, BN} (`b200trk_net_op_grid`) and its split-K
    reduction (`b200trk_net_op_splitk_reduction`: c = cluster, w = L2 workspace). Over the S = 1..16 sweep of each ResNet-50
    configuration some S reaches the cluster reduction, the L2 workspace for a cluster grid the device cannot hold at once (at
    most 8 splits; clusters of 3 and 5 on a 132-SM H100) and an unsplit BN = 128 launch; at 288^2 also an uneven last split
    (S = 1..3 on an H100). At 352^2 no S <= 16 splits unevenly: every split layer's k-block count is a multiple of its split
    count there. More than 8 splits (the workspace by split count) never happens without B200TRK_TC_CLUSTER=0: splits are capped
    at the cluster size; test_tc_conv_layers_gpu covers both plans with that switch.

The exact-fp32 path (precision 1) runs at 288^2 for S in {1, 5, 16}. Its split-K (`launch_conv_fp32`, mirrored by `_fp32_splits`)
splits the 36x36 and 18x18 layers at S = 1 and 5; at S = 16 every layer fills two waves of CTAs and runs unsplit, so its
workspace is exercised at S = 1 and 5."""
import contextlib
import ctypes as C
from io import StringIO

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pytracking_b200 import _lib, synth
from pytracking_b200.engine import BackboneEngine
from test_tc_conv_layers_gpu import TINY, _check_layers, _grid, _plan, _reference, _weights

pytestmark = pytest.mark.gpu

OP_PREPROCESS, OP_STEM, OP_MAXPOOL, OP_CONV, OP_EXPORT, OP_L2NORM = range(6)
MAX_BATCH = 16
U = 2.0 ** -24
REDUCTION = {0: "", 1: "c", 2: "w"}


def _sum_bound(K):
    """fp32 summation bound of a K-term dot product + bias + residual, normalised (module docstring)."""
    return (K + 2) * 2.0 ** -23 + 2.0 ** -20


def _l2norm_bound(n_per_sample):
    """Element-wise relative error bound of launch_l2norm_nhwc_to_nchw (conv_fp32_kernels.cuh) against float64 InstanceL2Norm.

    sumsq_kernel splits a sample's n4 = n / 4 float4s into 64 ranges of per = ceil(n4 / 64); each of 256 threads squares and
    accumulates t = ceil(per / 256) float4s into one fp32 register (4t terms: at most 4t + 1 roundings along any term's path,
    the square's included; fma contraction only removes roundings), block_sum adds the 256 thread sums in 2 x 5 shuffle levels
    (the second warp_sum pads 8 warp sums with exact zeros), and nhwc_to_nchw_kernel adds the 64 ordered partials one after the
    other (63 roundings) and then eps (1). All terms are non-negative, so the computed sum s' = s (1 + d), |d| <= gamma_D,
    gamma_D = D u / (1 - D u), D = 4t + 1 + 10 + 63 + 1. The factor scale * sqrt(C*H*W / (s' + eps)) adds a rounding for the
    division, halves the relative error of its argument in the sqrt and adds one, one for * scale (the reference uses the same
    float32 scale), and the product with the element one more: |y / y64 - 1| <= (gamma_D + u) / 2 + 3 u to first order; 1 %
    covers the second-order terms. Around 3e-6 at 18x18x512 (D = 87), not a measured figure."""
    n4 = n_per_sample // 4
    per = -(-n4 // 64)
    t = -(-per // 256)
    D = 4 * t + 1 + 10 + 63 + 1
    gamma = D * U / (1 - D * U)
    return ((gamma + U) / 2 + 3 * U) * 1.01


def _fp32_splits(M, cout, K, sms, ws_floats=8 << 20):
    """Split-K factor launch_conv_fp32 (conv_fp32.cu) picks for an M x cout x K convolution (64 x 64 CTA tiles, K in steps of 16)."""
    ctas, kst = -(-M // 64) * -(-cout // 64), K // 16
    s = 1
    if ctas < 2 * sms:
        s = max(1, min(-(-3 * sms // ctas), kst // 4, 32))
        while s > 1 and s * M * cout > ws_floats:
            s -= 1
    per = -(-kst // s)
    return -(-kst // per)


class _Net:
    """A BackboneEngine of max_batch 16 driven through b200trk_net_forward_iou with one input and one set of output buffers for
    every S, so that repeated calls at one S hit the network's CUDA-graph cache (keyed on the pointers and S)."""

    def __init__(self, arch, crop, precision=0):
        self.sd = synth.make_dimp_state_dict(arch, seed=0, lut_seed=3)
        self.eng = BackboneEngine(self.sd, arch=arch, max_batch=MAX_BATCH, crop_size=crop, precision=precision)
        self.crop = crop
        d = self.eng.dims
        self.im = torch.empty(MAX_BATCH, 3, crop, crop, device="cuda")
        self.exports = [torch.empty(MAX_BATCH, d[3 * i], d[3 * i + 1], d[3 * i + 2], device="cuda") for i in range(3)]
        self.steps = _plan(self.eng)
        self.info = {i: (info, io) for i, info, io in self.steps}

    def close(self):
        self.eng.close()

    def forward(self, x):
        S = x.shape[0]
        self.im[:S].copy_(x)
        ptr = [C.c_void_p(t.data_ptr()) for t in [self.im] + self.exports]
        _lib.check(_lib.lib().b200trk_net_forward_iou(self.eng.handle, ptr[0], S, ptr[1], ptr[2], ptr[3], None, None,
                                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)), "net_forward_iou")
        torch.cuda.synchronize()

    def output(self, i, S):
        """NHWC output of plan step i after the last pass, rows 0..S-1 ([S, crop, crop, 4] for the preprocess step)."""
        info = self.info[i][0]
        shape = (S, self.crop, self.crop, 4) if info[0] == OP_PREPROCESS else (S, info[5], info[6], info[2])
        t = torch.empty(shape, device="cuda")
        _lib.check(_lib.lib().b200trk_net_op_output(self.eng.handle, i, S, C.c_void_p(t.data_ptr()), None), "net_op_output")
        torch.cuda.synchronize()
        return t

    def snapshot(self, S):
        """Every step's output and the three exports of the last pass, rows 0..S-1."""
        snap = {i: self.output(i, S) for i, info, _ in self.steps if info[0] not in (OP_EXPORT, OP_L2NORM)}
        for name, t in zip(("layer2", "layer3", "classification"), self.exports):
            snap[name] = t[:S].clone()
        return snap

    def export_names(self):
        """plan step -> the export it writes (the NCHW exports run in the order layer2, layer3)."""
        ex = [i for i, info, _ in self.steps if info[0] == OP_EXPORT]
        names = dict(zip(ex, ("layer2", "layer3")))
        names.update({i: "classification" for i, info, _ in self.steps if info[0] == OP_L2NORM})
        return names


def _folded_stem(sd):
    """conv1 + bn1 folded in double exactly as fold_and_repack (net.cu) folds them, rounded to float32: NHWC weights, bias."""
    p = "feature_extractor."
    w = sd[p + "conv1.weight"].double()
    g, b, m, v = (sd[p + "bn1." + k].double() for k in ("weight", "bias", "running_mean", "running_var"))
    sc = g / torch.sqrt(v + 1e-5)
    return (w * sc.view(-1, 1, 1, 1)).float().permute(0, 2, 3, 1).contiguous().cuda(), (b - m * sc).float().cuda()


def _norm_err(y, z, m):
    return float(((y.double() - z).abs() / (m + TINY)).max())


def _check_stages(net, crops, snap, S, rows, worst):
    """Compares rows `rows` of every plan step of the pass in `snap` (still the arena's last pass) with its reference; updates
    worst[kind] = (error, S, step)."""
    from oracle import dimp_oracle as O
    rows = list(rows)

    def note(kind, e, i):
        if kind not in worst or e > worst[kind][0]:
            worst[kind] = (e, S, i)

    names = net.export_names()
    for i, info, io in net.steps:
        kind = info[0]
        if kind == OP_PREPROCESS:
            ref = O.preprocess_image(crops[rows].cpu()).permute(0, 2, 3, 1)
            ref = torch.cat([ref, torch.zeros_like(ref[..., :1])], dim=3)
            assert torch.equal(snap[i][rows].cpu(), ref), "S=%d: preprocess differs from torch-CPU" % S
            note("preprocess", 0.0, i)
        elif kind == OP_STEM:
            w, b = _folded_stem(net.sd)
            x = snap[io[0]][rows][..., :3]
            z, m, _ = _reference(x, w, b, None, 2, 3, True)
            e = _norm_err(snap[i][rows], z, m)
            assert e <= _sum_bound(147), "S=%d: stem e %.3e above the fp32 summation bound" % (S, e)
            note("stem", e, i)
        elif kind == OP_MAXPOOL:
            ref = F.max_pool2d(snap[io[0]][rows].permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
            assert torch.equal(snap[i][rows], ref), "S=%d: max-pool differs from F.max_pool2d" % S
            note("maxpool", 0.0, i)
        elif kind == OP_CONV and not info[7]:
            _, cin, _, k, stride = info[:5]
            w, b = _weights(net.eng, i, info)
            res = snap[io[1]][rows] if io[1] >= 0 else None
            z, m, _ = _reference(snap[io[0]][rows], w, b, res, stride, io[3], io[2])
            e = _norm_err(snap[i][rows], z, m)
            assert e <= _sum_bound(k * k * cin), "S=%d step %d: fp32 conv e %.3e above the summation bound" % (S, i, e)
            note("conv_fp32", e, i)
        elif kind == OP_EXPORT:
            ref = snap[io[0]][rows].permute(0, 3, 1, 2)
            assert torch.equal(snap[names[i]][rows], ref), "S=%d: %s export is not the permuted NHWC output" % (S, names[i])
            note("export_nchw", 0.0, i)
        elif kind == OP_L2NORM:
            h = snap[io[0]][rows].double()
            n = h[0].numel()
            ss = (h * h).reshape(len(rows), -1).sum(1).view(-1, 1, 1, 1)
            ref = (float(np.float32(net.eng.norm_scale)) * torch.sqrt(n / (ss + 1e-5)) * h).permute(0, 3, 1, 2)
            y = snap["classification"][rows].double()
            assert bool(((y == 0) == (ref == 0)).all()), "S=%d: InstanceL2Norm zero pattern differs" % S
            e = float(((y - ref).abs() / (ref.abs() + TINY)).max())
            bound = _l2norm_bound(n)
            assert e <= bound, "S=%d: InstanceL2Norm relative error %.3e above %.3e" % (S, e, bound)
            note("l2norm_export", e, i)
    if any(info[0] == OP_CONV and info[7] for _, info, _ in net.steps):
        with contextlib.redirect_stdout(StringIO()):                # the per-layer table of the tc test, 50+ lines per S
            recs = _check_layers(net.eng, net.steps, S, rows, "S=%d" % S)
        for r in recs:
            note("conv_tc", r["e"], r["index"])
            note("conv_tc e/e_tf32", r["ratio"], r["index"])


def _plan_line(net, S):
    """(printable line, records) of every tensor-core step's launch at the last configured S."""
    recs, parts = [], []
    for i, info, _ in net.steps:
        if info[0] != OP_CONV or not info[7]:
            continue
        g = _grid(net.eng, i)
        mode = C.c_int()
        _lib.check(_lib.lib().b200trk_net_op_splitk_reduction(net.eng.handle, i, C.byref(mode)), "net_op_splitk_reduction")
        recs.append(dict(index=i, grid=g, mode=mode.value, total_kb=info[3] * info[3] * info[1] // 32))
        parts.append("%d.%d.%d/%d%s" % (g[0], g[1], g[2], g[3], REDUCTION[mode.value]))
    return "S=%2d %s" % (S, " ".join(parts)), recs


def _coverage(recs):
    return dict(zip(BRANCHES, (any(r["mode"] == 1 for r in recs),
                               any(r["mode"] == 2 and r["grid"][2] <= 8 for r in recs),
                               any(r["grid"][2] == 1 and r["grid"][3] == 128 for r in recs),
                               any(r["grid"][2] > 1 and r["total_kb"] % r["grid"][2] != 0 for r in recs))))


CONFIGS = {"r50_288": ("resnet50", 288, range(1, MAX_BATCH + 1)), "r50_352": ("resnet50", 352, range(1, MAX_BATCH + 1)),
           "r18_288": ("resnet18", 288, (1, 7, 16))}
BRANCHES = ("cluster split-K", "L2 workspace, cluster grid does not fit", "unsplit BN = 128", "uneven last split")
MUST_REACH = {"r50_288": BRANCHES, "r50_352": BRANCHES[:3], "r18_288": ()}     # module docstring: no uneven split at 352^2


def _crops(crop, S):
    """S different seeded crops, one per row."""
    return torch.cat([synth.make_crop(1000 * crop + 37 * S + r, 1, crop) for r in range(S)]).cuda()


def _stage_sweep(arch, crop, batch_sizes, precision=0):
    net = _Net(arch, crop, precision)
    label = "%s %d^2 precision %d" % (arch, crop, precision)
    worst, reached = {}, {}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        for S in batch_sizes:
            crops = _crops(crop, S)
            net.forward(crops)
            _check_stages(net, crops, net.snapshot(S), S, sorted({0, S // 2, S - 1}), worst)
            if precision == 0:
                line, recs = _plan_line(net, S)
                print(line)
                for k, v in _coverage(recs).items():
                    reached.setdefault(k, []).extend([S] if v else [])
            else:
                splits = [(i, _fp32_splits(S * info[5] * info[6], info[2], info[3] ** 2 * info[1], sms)) for i, info, _ in net.steps
                          if info[0] == OP_CONV]
                print("%s S=%2d fp32 split-K steps (step:splits): %s" % (label, S, " ".join("%d:%d" % (i, s) for i, s in splits if s > 1)
                                                                         or "none"))
                reached.setdefault("fp32 split-K", []).extend([S] if any(s > 1 for _, s in splits) else [])
        print("%s worst per step kind: %s" % (label, ", ".join("%s %.3g (S=%d, step %d)" % (k, e, s, i) for k, (e, s, i) in
                                                                 sorted(worst.items()))))
        print("%s plan branches reached at S = %s" % (label, "; ".join("%s: %s" % (k, v) for k, v in reached.items())))
        return reached
    finally:
        net.close()


def _bitwise_sweep(arch, crop, batch_sizes, precision=0):
    """At every S: the second eager pass, the recorded-and-replayed third and a replayed fourth equal the first eager pass, and
    permuted rows permute every step's output bit for bit."""
    net = _Net(arch, crop, precision)
    label = "%s %d^2 precision %d" % (arch, crop, precision)
    try:
        for S in batch_sizes:
            crops = _crops(crop, S)
            net.forward(crops)                                   # first pass at this S: eager
            first = net.snapshot(S)
            for call in ("second eager pass", "recorded and replayed pass", "replayed pass"):
                net.forward(crops)
                got = net.snapshot(S)
                for k in first:
                    assert torch.equal(got[k], first[k]), "%s S=%d: %s differs from the first eager pass at step %s" % (label, S, call, k)
            for pname, perm in (("reversed", list(range(S))[::-1]), ("rotated by one", list(range(1, S)) + [0])):
                net.forward(crops[perm])
                got = net.snapshot(S)
                for k in first:
                    assert torch.equal(got[k], first[k][perm]), "%s S=%d: rows %s -> step %s is not the same permutation" % (
                        label, S, pname, k)
    finally:
        net.close()


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_every_step_vs_reference(config):
    arch, crop, sizes = CONFIGS[config]
    reached = _stage_sweep(arch, crop, sizes)
    for branch in MUST_REACH[config]:
        assert reached[branch], "%s: no S in 1..16 reaches %s" % (config, branch)


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_permuted_rows_and_graph_replay_bitwise(config):
    arch, crop, sizes = CONFIGS[config]
    _bitwise_sweep(arch, crop, sizes)


def test_exact_fp32_path_every_step():
    reached = _stage_sweep("resnet50", 288, (1, 5, 16), precision=1)
    assert reached["fp32 split-K"], "no exact-fp32 layer ran split-K"
    _bitwise_sweep("resnet50", 288, (1, 5, 16), precision=1)
