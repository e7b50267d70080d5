"""-m gpu: ATOM's filter optimisers checked step by step against float64, and its score ops entry by entry.

Steps, not filters: a kernel's step is d_ker = w_out - w_start (exact in float64), the reference d_ref the float64 step from the same
start (tests/atom_step_ref.py), e = max|d_ker - d_ref| / max|d_ref| after each entry is allowed the float32 rounding of the output
(2^-24 |w_out|) and its kink allowance.

  * atom_cg_filter, cases chosen through `cg_plan` so that together they reach every launch plan feature of the device (channel passes
    1 / 2 / 4, NCH = 1 and > 1, NG = n and uneven groups, spc = CG_SPC_MAX with n = NG * 8, pipeline depths 4 / 3 / 2, FS 18 and 22):
      single step (num_iter = 1) from w_0 and from two later iterates: e <= the float32 single-step bound of that start;
      k = 2..5 and 10 iterations from w_0: e(k) <= max(4 e_f32(k), k * bound(w_0)), e_f32(k) the error of independent float32 runs;
      every step also e <= 16 e_f32 (the worst-case bound is 10^3-10^4 times what float32 really does: see tests/atom_step_ref.py);
      the tracker chain: 8 consecutive 5-iteration calls on a 250-slot memory that fills by one slot per call, each from the kernel's own
      previous output, each against float64 from that same start;
      exact properties bit for bit: repeat, out= the input buffer, num_iter = 0, all-zero sample weights.
  * atom_gn_joint_: one GN iteration with num_cg_iter = 1..10 from the same (w, P) under the same rule, the w and P blocks separately
    (the P block's bound carries the preconditioner's 1 / projection_reg); a chain of six single-GN calls; six GN iterations in one
    call equal to the chain bit for bit.
  * feature_normalize_, conv1x1, conv2d_same, fourier_interp: |k - f64| <= depth 2^-24 sum|terms| per entry; the arg-max on the
    upsampled grid within twice the bound of the float64 maximum, and exactly the float64 arg-max when the top-two gap exceeds that.

One line per case reports the plan reached, the worst ratio of error to bar and the number of kink cells."""
import math

import pytest
import torch
import torch.nn.functional as F

import atom_step_ref as R
from oracle import atom_oracle as A
from pytracking_b200 import ops, synth

pytestmark = pytest.mark.gpu

U = R.U
REACHED = set()
ACTS = {"mlu", "relu", "elu", "none"}
SEEN = {"act": set(), "fr": set()}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _err(d_ker, d_ref, allow):
    return float(((d_ker - d_ref).abs() - allow).clamp(min=0).max() / d_ref.abs().max())


# ---- atom_cg_filter -------------------------------------------------------------------------------------------------------------------
# (FS, C, n, filled slots, activation, Fletcher-Reeves): well-conditioned memories (synth.make_atom_memory), zero-weight tails where
# filled < n.  On 132 SMs they reach: 1/1/12/1/4, 1/4/33/2/4, 1/4/33/8/3 (the tracker), 1/4/33/8/3 with n = 264 = 33 * 8, 2/2/66/5/4,
# 4/1/132/5/3, 1/4/33/2/3 and 1/4/33/8/2 at FS 22, 4/4/33/8/3 (passes / NCH / NG / spc / NST).  n = 224 is 28 * 8 on 114 SMs.
CG_CASES = [(18, 16, 12, 12, "mlu", False), (18, 64, 40, 25, "relu", False), (18, 64, 250, 60, "mlu", False),
            (18, 64, 264, 90, "none", True), (18, 64, 224, 80, "elu", False), (18, 64, 330, 100, "elu", False),
            (18, 64, 600, 100, "mlu", True), (22, 64, 40, 40, "elu", True), (22, 64, 250, 70, "mlu", False),
            (18, 256, 250, 24, "relu", False)]


def _w0(C, seed):
    return (0.02 * torch.randn(1, C, 4, 4, generator=torch.Generator().manual_seed(seed))).cuda()


def _check_cg(label, X, y, sw, w0, act, fr, reg=0.1):
    n, C, fs = X.shape[0], X.shape[1], X.shape[-1]
    sms = _sms()
    plan = R.cg_plan(n, C, fs, sms)
    assert plan is not None, label
    REACHED.update(R.plan_features(n, C, fs, sms))
    SEEN["act"].add(act)
    SEEN["fr"].add(fr)
    prob = R.ConvProblem(X, y, sw, reg, act, 0.05, fr)
    depths = R.cg_depths(n, C, fs, sms)

    def run(w, k, out=None):
        r = ops.atom_cg_filter(w, X, y, sw, reg, k, act, 0.05, fr, out=out)
        torch.cuda.synchronize()
        return r

    fails, worst, kinks = [], [0.0, 0.0, 0.0], 0
    # single steps from w_0 and two later iterates (the kernel's own 5- and 10-iteration results)
    w5 = run(w0, 5).clone()
    w10 = run(w5, 5).clone()
    for tag, ws in (("w0", w0), ("w5", w5), ("w10", w10)):
        w1 = run(ws, 1)
        ref = prob.step(ws, 1)
        cells = prob.kink_cells(ws)
        kinks += len(cells)
        allow = prob.kink_allowance(ws, 1, cells, ref) + U * w1.double().cpu().abs()
        e, bar = _err(w1.double().cpu() - ws.double().cpu(), ref, allow), prob.single_bound(ws, depths)
        e32 = prob.e32(ws, 1, ref)
        worst[0] = max(worst[0], e / bar)
        worst[2] = max(worst[2], e / e32)
        if e > bar or e > R.F32_FACTOR * e32:
            fails.append("single step from %s: e %.3e > bound %.3e or %d x e_f32 %.3e" % (tag, e, bar, R.F32_FACTOR, e32))
    # k iterations from w_0
    sb0 = prob.single_bound(w0, depths)
    cells0 = prob.kink_cells(w0)
    for k in (2, 3, 4, 5, 10):
        wk = run(w0, k)
        ref = prob.step(w0, k)
        e32 = prob.e32(w0, k, ref)
        allow = prob.kink_allowance(w0, k, cells0, ref) + U * wk.double().cpu().abs()
        e, bar = _err(wk.double().cpu() - w0.double().cpu(), ref, allow), max(4 * e32, k * sb0)
        worst[1] = max(worst[1], e / bar)
        worst[2] = max(worst[2], e / e32)
        if e > bar or e > R.F32_FACTOR * e32:
            fails.append("%d iterations: e %.3e > bar %.3e (e_f32 %.3e, bound %.3e)" % (k, e, bar, e32, sb0))
    # exact properties
    a = run(w0, 5).clone()
    assert torch.equal(run(w0, 5), a), "%s: a repeat differs" % label
    buf = w0.clone()
    run(buf, 5, out=buf)
    assert torch.equal(buf, a), "%s: out= the input buffer differs from out of place" % label
    assert torch.equal(run(w0, 0), w0), "%s: num_iter = 0 is not the identity" % label
    p = plan
    print("atom f64 cg %-26s plan %d/%d/%d/%d/%d | single %.4f iterates %.4f (e / bar) | e / e_f32 %.2f | bound(w0) %.1e | kink cells %d"
          % (label, p["passes"], p["NCH"], p["NG"], p["spc"], p["NST"], worst[0], worst[1], worst[2], sb0, kinks))
    assert not fails, "%s:\n  %s" % (label, "\n  ".join(fails))


@pytest.mark.parametrize("fs,C,n,filled,act,fr", CG_CASES, ids=["fs%d-C%d-n%d-f%d-%s-%s" % (c[0], c[1], c[2], c[3], c[4], "fr" if c[5] else "pr")
                                                                for c in CG_CASES])
def test_atom_cg_steps_vs_float64(fs, C, n, filled, act, fr):
    if R.cg_plan(n, C, fs, _sms()) is None:
        pytest.skip("plan fs %d C %d n %d: refused by launch_cg on %d SMs (does not fit)" % (fs, C, n, _sms()))
    x, y, sw = synth.make_atom_memory(300 + n + C + fs, n, C, fs, fs, n_filled=filled)
    _check_cg("fs%d C%d n%d f%d %s %s" % (fs, C, n, filled, act, "fr" if fr else "pr"), x.cuda(), y.cuda(), sw.cuda(), _w0(C, n), act, fr)


def _sequence_memory(crop, slots, filled):
    """ATOM's memory as the tracker fills it: ResNet-18 layer3 features of crops of synthetic sequence 1 (the crop follows the target
    with a few pixels of jitter), p-norm normalised and projected to 64 channels by a fixed matrix; near-duplicate samples.  Labels are
    Gaussians at the target's cell, weights decay as the tracker's learning rate makes them; slots past `filled` are zero."""
    from pytracking_b200.engine import BackboneEngine
    frames, _ = synth.make_sequence(1, num_frames=filled - 1)
    gt = synth.sequence_ground_truth(1, filled - 1)
    crops = []
    for t in range(filled):
        x, y, w, h = gt[t]
        side = 5.0 * math.sqrt(w * h)
        cx, cy = x + w / 2 + ((7 * t) % 11 - 5), y + h / 2 + ((5 * t) % 9 - 4)
        im = torch.from_numpy(frames[t]).permute(2, 0, 1).float().unsqueeze(0)
        x0, y0, pad = int(round(cx - side / 2)), int(round(cy - side / 2)), int(side)
        im = F.pad(im, (pad, pad, pad, pad), mode="replicate")[:, :, y0 + pad:y0 + pad + int(side), x0 + pad:x0 + pad + int(side)]
        crops.append(F.interpolate(im, size=(crop, crop), mode="bilinear", align_corners=False))
    sd = synth.make_backbone_state_dict("resnet18", seed=5)
    eng = BackboneEngine(sd, arch="resnet18", max_batch=10, crop_size=crop, precision=0, head=False)
    feats = []
    for i in range(0, filled, 10):
        f = eng.forward(torch.cat(crops[i:i + 10]).contiguous().cuda(), want=("layer3",))["layer3"]
        feats.append(ops.feature_normalize_(f.contiguous(), 2.0).clone())
    torch.cuda.synchronize()
    eng.close()
    feats = torch.cat(feats)
    P = (torch.randn(64, feats.shape[1], 1, 1, generator=torch.Generator().manual_seed(crop)) / 16).cuda()
    proj = ops.conv1x1(feats, P)
    fs = proj.shape[-1]
    X = torch.zeros(slots, 64, fs, fs, device="cuda")
    X[:filled] = proj
    k0 = torch.arange(fs, dtype=torch.float32).view(1, -1, 1) - (fs - 1) / 2
    yy = torch.zeros(slots, 1, fs, fs)
    yy[:filled, 0] = torch.exp(-0.5 / 1.5 ** 2 * (k0 ** 2 + k0.transpose(1, 2) ** 2))
    sw = torch.zeros(slots)
    sw[:filled] = torch.tensor([0.99 ** (filled - 1 - i) for i in range(filled)])
    return X.contiguous(), yy.cuda(), (sw / sw.sum()).cuda()


@pytest.mark.parametrize("crop,slots,filled,act", [(288, 250, 40, "mlu"), (352, 40, 30, "relu")])
def test_atom_cg_steps_vs_float64_sequence_memory(crop, slots, filled, act):
    X, y, sw = _sequence_memory(crop, slots, filled)
    _check_cg("sequence %d n%d f%d %s" % (crop, slots, filled, act), X, y, sw, _w0(64, crop), act, False)


def test_atom_cg_tracker_chain():
    """8 consecutive 5-iteration calls on the tracker's 250-slot memory (C = 64, 18 x 18, mlu, Polak-Ribiere), one more slot filled per
    call, each from the kernel's own previous output."""
    X, y, sw_full = synth.make_atom_memory(404, 250, 64, 18, 18, n_filled=40)
    X, y = X.cuda(), y.cuda()
    w = _w0(64, 404)
    REACHED.update(R.plan_features(250, 64, 18, _sms()))
    worst = 0.0
    for call in range(8):
        nf = 10 + call
        sw = sw_full.clone()
        sw[nf:] = 0
        sw = (sw / sw.sum()).cuda()
        prob = R.ConvProblem(X, y, sw, 0.1, "mlu", 0.05, False)
        w1 = ops.atom_cg_filter(w, X, y, sw, 0.1, 5, "mlu", 0.05, False)
        torch.cuda.synchronize()
        ref = prob.step(w, 5)
        e32 = prob.e32(w, 5, ref)
        cells = prob.kink_cells(w)
        allow = prob.kink_allowance(w, 5, cells, ref) + U * w1.double().cpu().abs()
        e = _err(w1.double().cpu() - w.double().cpu(), ref, allow)
        bar = max(4 * e32, 5 * prob.single_bound(w, R.cg_depths(250, 64, 18, _sms())))
        worst = max(worst, e / bar, e / (R.F32_FACTOR * e32))
        assert e <= bar and e <= R.F32_FACTOR * e32, "call %d (%d filled): e %.3e > bar %.3e or %d x e_f32 %.3e" % (call, nf, e, bar, R.F32_FACTOR, e32)
        w = w1.clone()
    print("atom f64 cg tracker chain: 8 calls, worst e / bar %.4f" % worst)


def test_atom_cg_zero_weights():
    """All-zero sample weights: from w_0 = 0 the rho == 0 break returns 0 (no NaN); from w_0 != 0 the problem is reg |w + x|^2 alone and
    one CG step lands on 0 (alpha = 1 / reg), the later iterations stop at rho == 0."""
    x, y, _ = synth.make_atom_memory(5, 40, 64, 18, 18)
    x, y, sw = x.cuda(), y.cuda(), torch.zeros(40, device="cuda")
    z = torch.zeros(1, 64, 4, 4, device="cuda")
    out = ops.atom_cg_filter(z, x, y, sw, 0.1, 5, "mlu", 0.05, False)
    assert torch.equal(out, z)
    w0 = _w0(64, 6)
    for k in (1, 5):
        out = ops.atom_cg_filter(w0, x, y, sw, 0.1, k, "mlu", 0.05, False)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        assert float(out.abs().max()) <= 8 * U * float(w0.abs().max()), (k, float(out.abs().max()))


def test_atom_cg_zz_plan_coverage():
    """The plans the cases above reached cover every plan feature that exists on this device."""
    if not REACHED:
        pytest.skip("no case ran")
    sms = _sms()
    reachable = set()
    for fs in (18, 22):
        for C in (16, 64, 256):
            for n in range(1, 700):
                if R.cg_plan(n, C, fs, sms):
                    reachable |= R.plan_features(n, C, fs, sms)
    for f in sorted(set(R.PLAN_FEATURES) - reachable):
        print("atom f64 cg plan feature %r: not reachable on %d SMs (C 16 / 64 / 256, n < 700)" % (f, sms))
    print("atom f64 cg plan features reached on %d SMs: %s" % (sms, "; ".join(sorted(REACHED))))
    assert reachable <= REACHED, sorted(reachable - REACHED)
    assert SEEN["act"] == ACTS and SEEN["fr"] == {True, False}, SEEN


# ---- atom_gn_joint_ -------------------------------------------------------------------------------------------------------------------
# (n, Cin, Cc, FS, activation, Fletcher-Reeves, projection_reg)
GN_CASES = [(1, 256, 64, 18, "mlu", True, 1e-4), (30, 256, 64, 18, "mlu", True, 1e-4), (1, 256, 64, 22, "elu", False, 1e-2),
            (30, 256, 64, 22, "relu", True, 1e-2), (7, 100, 48, 18, "elu", False, 1e-4)]


def _gn_e32(prob, w, P, k, ref):
    runs = [prob.step32(w, P, k, seed) for seed in (0, 1)]
    return [max(float((d[b] - ref[b]).abs().max() / ref[b].abs().max()) for d in runs) for b in (0, 1)]


@pytest.mark.parametrize("n,cin,cc,fs,act,fr,preg", GN_CASES,
                         ids=["n%d-cin%d-cc%d-fs%d-%s-%s-%g" % (c[0], c[1], c[2], c[3], c[4], "fr" if c[5] else "pr", c[6]) for c in GN_CASES])
def test_atom_gn_steps_vs_float64(n, cin, cc, fs, act, fr, preg):
    x, y, sw = synth.make_atom_memory(700 + n + cin + fs, n, cin, fs, fs)
    if n == 1:
        sw = torch.ones(1)
    g = torch.Generator().manual_seed(701 + n)
    w0 = 0.02 * torch.randn(1, cc, 4, 4, generator=g)
    P0 = torch.randn(cc, cin, 1, 1, generator=g) / math.sqrt(cin)
    xc, yc, swc = x.cuda(), y.cuda(), sw.cuda()
    prob = R.FactorizedProblem(x, y, sw, 0.1, preg, act, 0.05, fr)

    def run(w, P, ncg, ngn):
        wk, Pk = w.clone().cuda().contiguous(), P.clone().cuda().contiguous()
        ops.atom_gn_joint_(wk, Pk, xc, yc, swc, 0.1, preg, ncg, ngn, act, 0.05, fr)
        torch.cuda.synchronize()
        return wk.cpu(), Pk.cpu()

    def errs(w, P, w1, P1, ref):
        return [_err(a1.double() - a.double(), r, U * a1.double().abs()) for a, a1, r in ((w, w1, ref[0]), (P, P1, ref[1]))]

    fails, worst = [], [0.0, 0.0]
    sb = prob.single_bound(w0, P0)
    for k in range(1, 11):
        w1, P1 = run(w0, P0, k, 1)
        ref = prob.step(w0, P0, k)
        e = errs(w0, P0, w1, P1, ref)
        e32 = _gn_e32(prob, w0, P0, k, ref)
        bars = [min(sb[b] if k == 1 else max(4 * e32[b], k * sb[b]), R.F32_FACTOR * e32[b]) for b in (0, 1)]
        for b, name in ((0, "dw"), (1, "dP")):
            worst[0 if k == 1 else 1] = max(worst[0 if k == 1 else 1], e[b] / bars[b])
            if e[b] > bars[b]:
                fails.append("%d CG iterations, %s: e %.3e > bar %.3e" % (k, name, e[b], bars[b]))
    # chain of six single-GN calls, each from the kernel's own output, against float64 from that point
    w, P = w0, P0
    chain_worst = 0.0
    for it in range(6):
        w1, P1 = run(w, P, 10, 1)
        ref = prob.step(w, P, 10)
        e32 = _gn_e32(prob, w, P, 10, ref)
        sbi = prob.single_bound(w, P)
        e = errs(w, P, w1, P1, ref)
        for b, name in ((0, "dw"), (1, "dP")):
            bar = min(max(4 * e32[b], 10 * sbi[b]), R.F32_FACTOR * e32[b])
            chain_worst = max(chain_worst, e[b] / bar)
            if e[b] > bar:
                fails.append("GN chain %d, %s: e %.3e > bar %.3e" % (it, name, e[b], bar))
        w, P = w1, P1
    w6, P6 = run(w0, P0, 10, 6)
    assert torch.equal(w6, w) and torch.equal(P6, P), "six GN iterations in one call differ from six chained calls"
    print("atom f64 gn n %2d Cin %3d Cc %2d fs %d %-4s %s preg %g | single %.4f CG iterates %.4f chain %.4f (e / bar) | bound w %.1e P %.1e"
          % (n, cin, cc, fs, act, "fr" if fr else "pr", preg, worst[0], worst[1], chain_worst, sb[0], sb[1]))
    assert not fails, "\n  ".join(fails)


# ---- score ops --------------------------------------------------------------------------------------------------------------------------
def _entrywise(ker, ref, terms, depth, label):
    bound = depth * U * terms + U * ref.abs()
    r = float(((ker.double().cpu() - ref).abs() / bound.clamp(min=1e-300)).max())
    assert r <= 1.0, "%s: worst |k - f64| / bound %.3f" % (label, r)
    return r


def test_atom_score_ops_vs_float64():
    g = torch.Generator().manual_seed(19)
    worst = {}
    # feature_normalize_ (p = 2): y = x / sqrt(mean x^2 + 1e-10); the mean's N terms, the root and the division
    x = torch.randn(5, 256, 18, 18, generator=g)
    xn = ops.feature_normalize_(x.clone().cuda(), 2.0)
    ref = A.feature_normalize(x.double(), 2.0)
    worst["feature_normalize"] = _entrywise(xn, ref, ref.abs(), 256 * 18 * 18 / 2 + 4, "feature_normalize")
    # conv1x1: 256 -> 64 at 5 scales, a K tail (Cin = 100), Cout = 48, HW tails at 18^2 and 22^2
    for S, cin, cout, hw in ((5, 256, 64, 18), (3, 100, 64, 18), (2, 256, 48, 22), (1, 100, 48, 22)):
        x = torch.randn(S, cin, hw, hw, generator=g)
        P = torch.randn(cout, cin, 1, 1, generator=g) / math.sqrt(cin)
        out = ops.conv1x1(x.cuda(), P.cuda())
        worst["conv1x1"] = max(worst.get("conv1x1", 0), _entrywise(out, A.conv1x1(x.double(), P.double()),
                                                                    A.conv1x1(x.double().abs(), P.double().abs()), cin, "conv1x1 %d->%d" % (cin, cout)))
    # conv2d_same at n = 5 and n = 250
    for n, fs in ((5, 18), (250, 18), (5, 22)):
        x = torch.randn(n, 64, fs, fs, generator=g)
        w = 0.1 * torch.randn(1, 64, 4, 4, generator=g)
        out = ops.conv2d_same(x.cuda(), w.cuda())
        worst["conv2d_same"] = max(worst.get("conv2d_same", 0), _entrywise(out, A.conv_same(x.double(), w.double()),
                                                                            A.conv_same(x.double().abs(), w.double().abs()), 16 * 64, "conv2d_same n %d" % n))
    # fourier_interp: 18 -> 288, 22 -> 352, odd 17 with k = 5 -> 64, an output size that is not a multiple of FI_ROWS (8)
    nb = 0
    for S, H, ksz, osz in ((5, 18, 4, 288), (5, 22, 4, 352), (2, 17, 5, 64), (3, 18, 4, 75)):
        sc = torch.randn(S, 1, H, H, generator=g)
        sc = sc + 4 * torch.exp(-0.1 * ((torch.arange(H) - H / 2.3).view(-1, 1) ** 2 + (torch.arange(H) - H / 1.7).view(1, -1) ** 2))
        up = ops.fourier_interp(sc.cuda(), (ksz, ksz), (osz, osz))
        ref = A.fourier_interp(sc.double(), (ksz, ksz), (osz, osz))
        terms = sc.double().abs().sum((2, 3), keepdim=True).expand_as(ref)
        depth = 2 * H * H + 16
        worst["fourier_interp"] = max(worst.get("fourier_interp", 0), _entrywise(up, ref, terms, depth, "fourier_interp %d -> %d" % (H, osz)))
        # arg-max on the upsampled grid
        flat_k, flat_r = up.double().cpu().reshape(S, -1), ref.reshape(S, -1)
        bnd = 2 * (depth * U * terms.reshape(S, -1)[:, 0] + U * flat_r.abs().max(1).values)
        ik = flat_k.argmax(1)
        top2 = flat_r.topk(2, 1).values
        for s in range(S):
            assert float(flat_r[s].max() - flat_r[s, ik[s]]) <= float(bnd[s]), "fourier_interp %d: arg-max cell too far below the maximum" % H
            if float(top2[s, 0] - top2[s, 1]) > float(bnd[s]):
                nb += 1
                assert int(ik[s]) == int(flat_r[s].argmax()), "fourier_interp %d: arg-max differs from float64" % H
    print("atom f64 score ops: worst |k - f64| / bound %s; arg-max exact where the gap allows: %d maps"
          % (", ".join("%s %.4f" % kv for kv in worst.items()), nb))
