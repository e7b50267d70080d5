"""-m gpu: both steepest-descent kernels checked step by step against float64, at every sample count the trackers run.

For each case (tests/sd_step_ref.py `cases()`, plus the two realistic memories of case D) one 10-iteration call with iterates and losses
gives w_0 .. w_10.  Each step is compared with the float64 step d_ref = alpha g from the same w_k (tests/sd_step_ref.py) and with the
step d_TF32 taken on TF32-rounded features and w_k, e_TF32 = max|d_TF32 - d_ref| / max|d_ref|:

  * single step: num_iter = 1 launched from w_0, w_4, w_9 (every w_k in case D); e = max|d_ker - d_ref| / max|d_ref|, each entry first
    allowed the float32 rounding of w_{k+1} (2^-24 |w_{k+1}|) and the kink allowance below, must be <= max(e_TF32 / 16, the float32
    bound of the kernel's cross-CTA reductions).  The same rule holds for losses[0] against the float64 loss at w_k.
  * carried scores: step k of the 10-iteration call (both kernels carry s <- s - alpha q across iterations) with the bar widened to
    (k + 1) times the single-step bar; the same for losses[k].
  * kinks: a GN-family cell whose float64 score is within 2^-16 (|X| * |w|) of 0 may land on either side in the kernel; the step with
    that cell's derivative from the other side widens each entry's allowance by |d_flip - d_ref|.  Newton's max(gHg, 0) likewise.

The 10-iteration call must equal the call without iterates and losses and its own last iterate bit for bit, and a repeat bit for bit;
the single launch from w_0 must give w_1 bit for bit.  One line per case reports the partition features reached and the worst ratios."""
import collections
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sd_step_ref as R
from pytracking_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu

ITERS = 10
U = 2.0 ** -24
TAU = 2.0 ** -16
REPORT = collections.defaultdict(lambda: [0.0, 0.0, 0.0, 0, 0])     # (kernel, mode) -> worst single, carried, loss ratio; kink steps; cases
FEATS = set()


def f32(v):
    return float(np.float32(v))


GN_P = synth.make_dimp_optimizer_params(seed=3)
GN_HP = dict(step_length=f32(math.exp(float(GN_P["log_step_length"]))), reg=f32(max(float(GN_P["filter_reg"]) ** 2, 1e-6)))
NEWTON_HP = dict(gauss_sigma=f32(0.25 * 22 / 5), step_length=1.0, reg=f32(0.05 ** 2), alpha_eps=f32(0.05), softmax_reg=None,
                 label_threshold=0.0, normalize_label=True)
L2_HP = dict(gauss_sigma=f32(1.3), hinge_threshold=f32(0.05), step_length=f32(0.9), reg=f32(0.01), alpha_eps=f32(0.01))
HINGE_HP = dict(filter_reg=f32(0.1), hinge_threshold=f32(0.1), activation_leak=f32(0.1), act_param=f32(0.7), steplength_reg=f32(0.02))


def _call(mode, X, bb, sw, lab, w, num_iter, full):
    kw = dict(return_iterates=full, compute_losses=full)
    if mode == "gn":
        luts = [GN_P[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
        return ops.dimp_sd_gn(w, X, bb, sw, *luts, num_iter, GN_HP["step_length"], GN_HP["reg"], **kw)
    if mode == "newton":
        h = NEWTON_HP
        return ops.prdimp_sd_newton(w, X, bb, sw, num_iter, h["gauss_sigma"], h["step_length"], h["reg"], alpha_eps=h["alpha_eps"],
                                    softmax_reg=None, label_threshold=0.0, normalize_label=True, **kw)
    if mode == "l2":
        h = L2_HP
        return ops.dimp_l2_sd_gn(w, X, bb, sw, num_iter, h["gauss_sigma"], h["hinge_threshold"], h["step_length"], h["reg"],
                                 alpha_eps=h["alpha_eps"], **kw)
    h = HINGE_HP
    return ops.gn_sd_hinge(w, X, lab, sw, num_iter, h["filter_reg"], h["hinge_threshold"], h["activation_leak"],
                           "relu" if mode == "hinge_relu" else "bentpar", h["act_param"], h["steplength_reg"], **kw)


def _problem(mode, X, bb, sw, lab):
    if mode == "gn":
        luts = [GN_P[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
        return R.Problem("gn", X, sw, bb=bb, luts=luts, **GN_HP)
    if mode == "newton":
        return R.Problem("newton", X, sw, bb=bb, **NEWTON_HP)
    if mode == "l2":
        return R.Problem("l2", X, sw, bb=bb, **L2_HP)
    return R.Problem("hinge", X, sw, label=lab, score_act="relu" if mode == "hinge_relu" else "bentpar", **HINGE_HP)


_MEM = {}


def _memory(fs, C):
    """Seeded synthetic memory of 50 samples (features, boxes, raw sample weights, hinge labels, w0) for one feature size and channel
    count; a case of n samples takes the first n."""
    key = (fs, C)
    if key not in _MEM:
        seed = 1000 + 7 * fs + C
        g = torch.Generator().manual_seed(seed)
        X = synth.make_clf_features(seed, 50, C, fs, fs).cuda()
        bb = synth.make_boxes(seed + 1, 50, center=(fs * 16) / 2 - 25).cuda()
        sw = (torch.rand(50, generator=g) + 0.5).cuda()
        lab = torch.rand(50, 1, fs + 1, fs + 1, generator=g).cuda()
        w0 = (0.01 * torch.randn(1, C, 4, 4, generator=g)).cuda()
        _MEM[key] = (X, bb, sw, lab, w0)
    return _MEM[key]


def _sequence_memory(crop):
    """Classification features of 50 crops of synthetic sequence 0 (the target box moves +3 / +2 px per frame; the crop is centred near
    it, 4x the target's size): near-duplicate samples, as a tracker's memory holds them.  Returns (features, boxes in crop pixels)."""
    from pytracking_b200.engine import BackboneEngine
    frames, _ = synth.make_sequence(0, num_frames=49)
    gt = synth.sequence_ground_truth(0, 49)
    side = 4.0 * math.sqrt(80 * 60)
    crops, boxes = [], []
    for t in range(50):
        x, y, w, h = gt[t]
        cx, cy = x + w / 2 + ((7 * t) % 11 - 5), y + h / 2 + ((5 * t) % 9 - 4)
        im = torch.from_numpy(frames[t]).permute(2, 0, 1).float().unsqueeze(0)
        x0, y0 = int(round(cx - side / 2)), int(round(cy - side / 2))
        pad = int(side)
        im = F.pad(im, (pad, pad, pad, pad), mode="replicate")[:, :, y0 + pad:y0 + pad + int(side), x0 + pad:x0 + pad + int(side)]
        crops.append(F.interpolate(im, size=(crop, crop), mode="bilinear", align_corners=False))
        sc = crop / int(side)
        boxes.append([(x - x0) * sc, (y - y0) * sc, w * sc, h * sc])
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    eng = BackboneEngine(sd, arch="resnet50", max_batch=10, crop_size=crop)
    feats = torch.cat([eng.forward(torch.cat(crops[i:i + 10]).contiguous().cuda(), want=("classification",))["classification"]
                       for i in range(0, 50, 10)])
    torch.cuda.synchronize()
    eng.close()
    return feats.contiguous(), torch.tensor(boxes, dtype=torch.float32).cuda()


def _depths(kind, n, C, fs, G):
    """Chain depths of the kernel's float32 cross-CTA reductions (gradient entries, A g cells, scalars), for fp32_bound."""
    if kind == "tc":
        p = R.tc_partition(n, C, fs, G)
        return math.ceil(p["contrib"] / 32) + 6, p["qn"], 48 + math.ceil(G / 32), p
    ng = min(n, G)
    return ng + 1, C // 16, 48 + ng + C // 16, None


def _check(kernel, mode, fs, C, n, X, bb, sw, lab, w0, single_from, monkeypatch, label):
    kind = R.kernel_for(kernel, n)
    if kernel == "default":
        monkeypatch.delenv("B200TRK_SD_TC", raising=False)
    else:
        monkeypatch.setenv("B200TRK_SD_TC", "1" if kernel == "tc" else "0")
    L = _lib.lib()
    want = 1 if kind == "tc" else 0

    def run(w, it, full):
        out = _call(mode, X, bb, sw, lab, w, it, full)
        torch.cuda.synchronize()
        assert L.b200trk_sd_last_kernel() == want, "%s: ran the wrong kernel" % label
        return out

    w, its, losses = run(w0, ITERS, True)
    w, its, losses = w.clone(), its.clone(), losses.clone()
    w_plain, _, _ = run(w0, ITERS, False)
    assert torch.equal(w, w_plain), "%s: iterates / losses change the filter" % label
    assert torch.equal(its[0], w0[0]) and torch.equal(its[-1], w[0]), label
    w_rep, its_rep, losses_rep = run(w0, ITERS, True)
    assert torch.equal(w_rep, w) and torch.equal(its_rep, its) and torch.equal(losses_rep, losses), "%s: not deterministic" % label
    singles = {}
    for k in single_from:
        w1, _, l1 = run(its[k:k + 1].contiguous(), 1, True)
        singles[k] = (w1[0].clone(), float(l1[0]))
    if 0 in singles:
        assert torch.equal(singles[0][0], its[1]), "%s: one iteration from w_0 differs from the first of ten" % label

    # float64 references from every iterate (w_10 for the last loss only)
    prob = _problem(mode, X, bb, sw, lab)
    assert prob.label_margin() > 1e-6, "%s: a label lies within 1e-6 of its threshold; the seed must change, not the kernel" % label
    ref = R.step(prob, its, detail=True)
    t32 = R.step(prob, its, tf32=True)
    dg, dq, ds, part = _depths(kind, n, C, fs, torch.cuda.get_device_properties(0).multi_processor_count)
    fb = R.fp32_bound(prob, ref, dg, dq, ds)
    d_ref = ref["d"][:ITERS]
    dmax = d_ref.flatten(1).abs().max(1).values
    e_t32 = (t32["d"][:ITERS] - d_ref).flatten(1).abs().max(1).values / dmax
    el_t32 = (t32["loss"] - ref["loss"]).abs() / ref["loss"].abs()
    lb = ds * U * ref["loss_abs"] / ref["loss"].abs() + 4 * U

    # kink allowance: per step, the sum of |d_flip - d_ref| over the ambiguous cells / samples.  A cell is ambiguous when its float64
    # score lies within tau of 0, tau = 1/16 of the largest score error of the TF32 step (the score error a kernel within the bar can
    # make), times k + 1 for the carried scores.  (2^-16 (|X| * |w|) is 30-60x wider at C = 512: it makes nearly every GN step ambiguous
    # at ~20 cells, and the allowance then exceeds the bar 10^3-fold.)
    allow = torch.zeros_like(d_ref)
    allow1 = torch.zeros_like(d_ref)
    kink_steps = 0
    tau = (t32["s"][:ITERS] - ref["s"][:ITERS]).flatten(1).abs().max(1).values / 16
    for k in range(ITERS):
        cells = []
        if R.has_kinks(prob):
            sk = ref["s"][k].abs()
            cells = torch.nonzero(sk <= (k + 1) * tau[k])
            for c0 in range(0, len(cells), 256):
                cc = cells[c0:c0 + 256]
                dd = (R.kink_steps(prob, ref, k, cc) - d_ref[k]).abs()
                allow[k] += dd.sum(0)
                allow1[k] += (dd * (sk[cc[:, 0], cc[:, 1], cc[:, 2]] <= tau[k]).view(-1, 1, 1, 1)).sum(0)
        elif mode == "newton":
            cells = torch.nonzero(ref["ghg"][k].abs() <= TAU * ref["tau_ghg"][k]).flatten()
            if len(cells):
                allow[k] += (R.ghg_steps(prob, ref, k, cells) - d_ref[k]).abs().sum(0)
                allow1[k] = allow[k]
        if len(cells):
            kink_steps += 1

    def ratio(d_ker, w_next, k, widen):
        ex = ((d_ker - d_ref[k]).abs() - U * w_next.abs() - (allow if widen > 1 else allow1)[k]).clamp(min=0)
        e = float(ex.max() / dmax[k])
        bar = widen * max(float(e_t32[k]) / 16, float(fb[k]))
        return e, bar

    def lratio(l_ker, k, widen):
        e = abs(l_ker - float(ref["loss"][k])) / abs(float(ref["loss"][k]))
        return e, widen * max(float(el_t32[k]) / 16, float(lb[k]))

    its64 = its.double()
    worst = [0.0, 0.0, 0.0]
    fails = []
    for k in range(ITERS):
        e, bar = ratio(its64[k] - its64[k + 1], its64[k + 1], k, k + 1)
        worst[1] = max(worst[1], e / float(e_t32[k]))
        if e > bar:
            fails.append("carried step %d: e %.3e > bar %.3e (e_TF32 %.3e, fp32 %.3e)" % (k, e, bar, e_t32[k], fb[k]))
    for k in range(ITERS + 1):
        e, bar = lratio(float(losses[k]), k, k + 1)
        worst[2] = max(worst[2], e / max(float(el_t32[k]), 1e-300))
        if e > bar:
            fails.append("carried loss %d: e %.3e > bar %.3e" % (k, e, bar))
    for k, (w1, l0) in singles.items():
        w1 = w1.double()
        e, bar = ratio(its64[k] - w1, w1, k, 1)
        worst[0] = max(worst[0], e / float(e_t32[k]))
        if e > bar:
            fails.append("single step %d: e %.3e > bar %.3e (e_TF32 %.3e, fp32 %.3e)" % (k, e, bar, e_t32[k], fb[k]))
        e, bar = lratio(l0, k, 1)
        if e > bar:
            fails.append("single loss %d: e %.3e > bar %.3e" % (k, e, bar))

    feats = sorted(part["features"]) if part else []
    FEATS.update(feats)
    rep = REPORT[(kind, mode)]
    rep[0], rep[1], rep[2] = max(rep[0], worst[0]), max(rep[1], worst[1]), max(rep[2], worst[2])
    rep[3] += kink_steps
    rep[4] += 1
    share = float((allow.flatten(1).max(1).values / dmax).max()) / max(float(e_t32.min()) / 16, 1e-300)
    print("sd f64 %-6s %-10s n %2d C %3d fs %d | single %.4f carried %.4f loss %.4f (e / e_TF32) | e_TF32 %.1e fp32 %.1e | kink steps %d "
          "(largest share of the bar %.2f) | smax %s %s" % (kind, mode, n, C, fs, worst[0], worst[1], worst[2], float(e_t32.max()),
                                                          float(fb.max()), kink_steps, share, part["smax"] if part else "-",
                                                          "; ".join(feats)))
    assert not fails, "%s:\n  %s" % (label, "\n  ".join(fails))


CASES = R.cases()


@pytest.mark.parametrize("kernel,mode,fs,C,n,use_sw", CASES,
                         ids=["%s-%s-fs%d-C%d-n%d%s" % (c[0], c[1], c[2], c[3], c[4], "" if c[5] else "-nosw") for c in CASES])
def test_sd_steps_vs_float64(kernel, mode, fs, C, n, use_sw, monkeypatch):
    X, bb, sw, lab, w0 = _memory(fs, C)
    swn = sw[:n] / sw[:n].sum() if use_sw else None
    _check(kernel, mode, fs, C, n, X[:n].contiguous(), bb[:n].contiguous(), swn, lab[:n].contiguous(), w0, (0, 4, 9), monkeypatch,
           "%s %s fs %d C %d n %d" % (kernel, mode, fs, C, n))


@pytest.mark.parametrize("mode,crop", [("gn", 288), ("newton", 352)])
def test_sd_steps_vs_float64_sequence_memory(mode, crop, monkeypatch):
    """Case D: 50 near-duplicate samples from the backbone, every step checked from its own iterate."""
    X, bb = _sequence_memory(crop)
    fs = X.shape[-1]
    g = torch.Generator().manual_seed(crop)
    sw = (torch.rand(50, generator=g) + 0.5).cuda()
    w0 = (0.01 * torch.randn(1, 512, 4, 4, generator=g)).cuda()
    _check("default", mode, fs, 512, 50, X, bb, sw / sw.sum(), None, w0, range(ITERS), monkeypatch, "sequence %s %d" % (mode, crop))


def test_zz_report_and_coverage():
    """The worst ratios per kernel and mode over the cases above, and the partition features they reached (all of those that exist on
    the device when it has 132 SMs; see test_sd_step_ref_cpu.py)."""
    if not REPORT:
        pytest.skip("no case ran")
    for (kind, mode), (s, c, l, k, cnt) in sorted(REPORT.items()):
        print("sd f64 worst %-4s %-10s over %3d cases: single %.4f carried %.4f loss %.4f (e / e_TF32); steps with a kink allowance %d"
              % (kind, mode, cnt, s, c, l, k))
    print("sd f64 partition features reached: %s" % "; ".join(sorted(FEATS)))
    if torch.cuda.get_device_properties(0).multi_processor_count == 132 and sum(v[4] for v in REPORT.values()) >= len(CASES):
        assert FEATS == set(R.FEATURES) - {"range crosses a chunk boundary"}, set(R.FEATURES) - FEATS
