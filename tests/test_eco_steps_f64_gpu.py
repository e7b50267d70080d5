"""-m gpu: ECO's Fourier-domain optimisers checked step by step against float64, and its score path entry by entry.

Steps, not filters: a kernel's step is d_ker = hf_out - hf_in (exact in float64), the reference d_ref the float64 step from the same float32
start and the same carried state (tests/eco_step_ref.py), e = max|d_ker - d_ref| / max|d_ref| after each entry is allowed the float32
rounding of the output (2^-24 |hf_out|).  The exported CG state (p, r_prev, rho) is held to the same bars as the filter.

  * eco_filter_cg_, cases chosen through the kernel's plan (pytracking_b200/eco_plan.py) so that together they reach every plan feature
    at the device's SM count (G 16 / 32, CPL 1 / 2 / 4, GPP 1 .. 16, all slabs resident, some, none, a grid smaller than the SM count,
    uneven coefficient ranges, N not a multiple of 4 GPP), with 1x1, dense 3x3, ECO's sparse 5x5 and spectrum-sized regularisation
    filters, Polak-Ribiere and Fletcher-Reeves, both alphas, direction_forget_factor 0 and not, the energy from new_xf and carried:
      one iteration from hf_0 and from two later iterates with the kernel's own carried state: e <= the single-step bound and 16 e_f32;
      k = 2..5 and 10 iterations from hf_0: e(k) <= max(4 e_f32(k), k bound) and 16 e_f32(k);
      the sample energy entry by entry within 4 ulps of float64;
      the tracker chain: 8 consecutive 5-iteration calls, one memory slot filled and the weights renormalised between calls;
      exact properties bit for bit: a repeat, num_iter = 0, NaN in zero-weight memory rows, NaN state buffers the call must not read.
  * eco_joint_gn_: one GN iteration with 1..10 CG iterations from the same (hf, P), the two blocks separately (the P block's bound carries
    1 / diag_M_proj); a chain of single-GN calls against float64 from each start, and equal bit for bit to the same GN iterations in one
    call (ECO's GN resets the CG state every iteration).
  * eco_apply_filter, eco_sample_fs, eco_preprocess_sample_, eco_shift_fs: |k - f64| <= depth 2^-24 sum|terms| per entry; the arg-max of
    the score map equal to the float64 one wherever the top-two gap exceeds twice the bound.

Under B200_EMUL_SMS (the CPU run of this file, tests/test_eco_step_ref_cpu.py) the plans are those of that SM count."""
import os

import pytest
import torch

import eco_step_ref as R
from oracle import eco_oracle as E
from pytracking_b200 import ops
from pytracking_b200.eco_plan import eco_joint_plan, eco_plan

pytestmark = pytest.mark.gpu

U = R.U
REACHED = set()
JREACHED = set()
SEEN = {"reg": set(), "fr": set(), "sa": set(), "dff": set(), "energy": set()}
DEV = "cuda" if torch.cuda.is_available() else "cpu"


def _sms():
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return int(os.environ.get("B200_EMUL_SMS", "132"))


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    """The float32 oracle runs are the e_f32 yardstick: no TF32 in their convolutions and products."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


# ---- eco_filter_cg_ -------------------------------------------------------------------------------------------------------------------
def _reg(kind, h, wh, g):
    if kind == "1x1":
        return torch.tensor([[0.3]]).view(1, 1, 1, 1)
    if kind == "dense3":
        return (0.05 + torch.rand(1, 1, 3, 3, generator=g)) * 0.3
    if kind == "eco":                                               # ECO's sparsified filter: small taps cut to exactly 0
        return torch.tensor([[0.0, 0.02, 0.05, 0.02, 0.0], [0.02, 0.1, 0.2, 0.1, 0.02], [0.05, 0.2, 0.9, 0.2, 0.05],
                             [0.02, 0.1, 0.2, 0.1, 0.02], [0.0, 0.02, 0.05, 0.02, 0.0]]).view(1, 1, 5, 5)
    return 0.02 + 0.2 * torch.rand(1, 1, h, wh, generator=g)      # "edge": rh == H and rw == Wh


def _memory(h, wh, n, c, filled, seed):
    g = torch.Generator().manual_seed(seed)
    samples = torch.zeros(h, wh, n, c, 2)
    samples[:, :, :filled] = torch.randn(h, wh, filled, c, 2, generator=g)
    sw = torch.zeros(n)
    sw[:filled] = torch.rand(filled, generator=g) + 0.1
    sw /= sw.sum()
    ky = torch.arange(-(h - 1) // 2, h // 2 + 1, dtype=torch.float32).view(-1, 1)
    kx = torch.arange(0, wh, dtype=torch.float32).view(1, -1)
    yf = torch.exp(-0.05 * (ky ** 2 + kx ** 2)).view(1, 1, h, wh)
    return samples, sw, yf, g


class Call:
    """The kernel's state between calls: filter, sample energy, CG state (device tensors)."""

    def __init__(self, hf, energy=None, state=None):
        self.hf, self.energy, self.state = hf, energy, state

    def clone(self):
        st = None if self.state is None else {k: (None if v is None else v.clone()) for k, v in self.state.items()}
        return Call(self.hf.clone(), None if self.energy is None else self.energy.clone(), st)


def _run(call, samples, yf, sw, reg, k, new_xf, kw):
    c = call.clone()
    en, st = ops.eco_filter_cg_(c.hf, samples, yf, sw, reg, c.energy, k, new_xf, c.state, **kw)
    torch.cuda.synchronize()
    return Call(c.hf, en, st)


def _check_step(prob, start, out, k, new_xf, sms, sb, fails, tag):
    """Bars of one call of k iterations: filter step, p, r_prev, rho and the energy.  Returns (worst e / bar, worst e / e_f32)."""
    ref = prob.step(start.hf, start.energy, start.state, k, new_xf)
    e32 = prob.e32(start.hf, start.energy, start.state, k, new_xf, ref)
    hf_in = start.hf.detach().to(ref["d"].device).double().reshape(ref["d"].shape)
    hf_out = out.hf.detach().to(ref["d"].device).double().reshape(ref["d"].shape)
    errs = {"d": R.rel_err(hf_out - hf_in, ref["d"], U * hf_out.abs()), "p": R.rel_err(out.state["p"], ref["p"]),
            "rho": R.rel_err(out.state["rho"].reshape(-1)[0], ref["rho"])}
    if not prob.fr:
        errs["r_prev"] = R.rel_err(out.state["r_prev"], ref["r_prev"])
    # rho is one sum over the whole spectrum: torch's float32 reductions of the permuted runs sum it far more accurately than the fields it
    # sums are known, so its float32 yardstick is the larger of its own e_f32 and the step's
    e32["rho"] = max(e32["rho"], e32["d"])
    wb = wf = 0.0
    for key, e in errs.items():
        bar = sb[key] if k == 1 else max(4 * e32[key], k * sb[key])
        wb, wf = max(wb, e / bar), max(wf, e / max(e32[key], 1e-300))
        if e > bar or e > R.F32_FACTOR * e32[key]:
            fails.append("%s, %d iteration(s), %s: e %.3e > bar %.3e or %d x e_f32 %.3e" % (tag, k, key, e, bar, R.F32_FACTOR, e32[key]))
    en_ref = ref["energy"].reshape(-1)
    en_k = out.energy.detach().to(en_ref.device).double().reshape(-1)
    ee = float(((en_k - en_ref).abs() / en_ref.abs()).max())
    if ee > 8 * U:
        fails.append("%s: sample energy %.2f ulps from float64" % (tag, ee / (2 * U)))
    return wb, wf


# (H, Wh, N, C, filled, regularisation filter, Fletcher-Reeves, standard alpha, direction_forget_factor, energy carried in).  At 132 SMs:
# GPP 8 res 1/1 grid 120; GPP 1 8 of 16 resident; GPP 4 grid 132; CPL 4 GPP 2 streamed; GPP 16 grid 15; streamed grid 66; GPP 2 (114 SMs).
DFF = (1 - 0.0075) ** 75
CG_CASES = [(15, 8, 200, 64, 200, "eco", False, True, DFF, True), (63, 32, 200, 16, 170, "eco", False, True, DFF, False),
            (17, 9, 200, 32, 37, "dense3", True, True, DFF, True), (31, 16, 250, 128, 250, "1x1", False, False, DFF, True),
            (5, 3, 40, 16, 33, "edge", False, True, 0.0, False), (11, 6, 500, 64, 300, "eco", True, False, 0.0, True),
            (23, 12, 120, 32, 120, "dense3", False, True, 0.5, False)]


def _cg_id(c):
    return "%dx%d-n%d-c%d-f%d-%s-%s-%s-dff%s-%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "fr" if c[6] else "pr", "sa" if c[7] else "nsa",
                                                    "0" if c[8] == 0 else "1", "en" if c[9] else "new")


@pytest.mark.parametrize("h,wh,n,c,filled,regk,fr,sa,dff,has_en", CG_CASES, ids=[_cg_id(c) for c in CG_CASES])
def test_eco_filter_cg_steps_vs_float64(h, wh, n, c, filled, regk, fr, sa, dff, has_en):
    sms = _sms()
    pl = eco_plan(h, wh, n, c, 1, sms)
    REACHED.update(R.plan_features(h, wh, n, c, sms))
    SEEN["reg"].add(regk), SEEN["fr"].add(fr), SEEN["sa"].add(sa), SEEN["dff"].add(dff != 0), SEEN["energy"].add(has_en)
    samples, sw, yf, g = _memory(h, wh, n, c, filled, seed=h * 1000 + n + c)
    reg = _reg(regk, h, wh, g)
    hf0 = 0.01 * torch.randn(1, c, h, wh, 2, generator=g)
    en0 = (torch.randn(1, c, h, wh, generator=g) ** 2 + torch.randn(1, c, h, wh, generator=g) ** 2 + 0.05) if has_en else None
    nxs = [torch.randn(1, c, h, wh, 2, generator=g) for _ in range(4)]
    kw = dict(fletcher_reeves=fr, standard_alpha=sa, direction_forget_factor=dff)
    S, Y, W, G_ = samples.cuda(), yf.cuda(), sw.cuda(), reg.cuda()
    NX = [x.cuda() for x in nxs]
    prob = R.FilterProblem(samples, yf, sw, reg, fr, sa, dff, dev=DEV)
    fails, worst = [], [0.0, 0.0, 0.0]
    c0 = Call(hf0.cuda(), None if en0 is None else en0.cuda())
    # single iterations from hf_0 and from two later iterates with the kernel's own carried state
    c5 = _run(c0, S, Y, W, G_, 5, NX[0], kw)
    c10 = _run(c5, S, Y, W, G_, 5, NX[1], kw)
    for tag, st, nx in (("hf_0", c0, NX[0]), ("hf_5", c5, NX[1]), ("hf_10", c10, NX[2])):
        out = _run(st, S, Y, W, G_, 1, nx, kw)
        sb = prob.single_bound(st.hf, st.energy, st.state, nx, sms)
        wb, wf = _check_step(prob, st, out, 1, nx, sms, sb, fails, "single step from " + tag)
        worst[0], worst[2] = max(worst[0], wb), max(worst[2], wf)
    sb0 = prob.single_bound(c0.hf, c0.energy, c0.state, NX[0], sms)
    for k in (2, 3, 4, 5, 10):
        out = _run(c0, S, Y, W, G_, k, NX[0], kw)
        wb, wf = _check_step(prob, c0, out, k, NX[0], sms, sb0, fails, "from hf_0")
        worst[1], worst[2] = max(worst[1], wb), max(worst[2], wf)
    # exact properties
    a = _run(c5, S, Y, W, G_, 5, NX[1], kw)
    b = _run(c5, S, Y, W, G_, 5, NX[1], kw)
    assert torch.equal(a.hf, b.hf) and torch.equal(a.state["p"], b.state["p"]) and torch.equal(a.state["rho"], b.state["rho"]) and \
        torch.equal(a.energy, b.energy), "a repeat differs"
    z = _run(c5, S, Y, W, G_, 0, NX[1], kw)
    assert torch.equal(z.hf, c5.hf) and torch.equal(z.energy, c5.energy) and torch.equal(z.state["p"], c5.state["p"]), "num_iter = 0 changed something"
    if filled < n:
        Sn = samples.clone()
        Sn[:, :, filled:] = float("nan")
        an = _run(c5, Sn.cuda(), Y, W, G_, 5, NX[1], kw)
        assert torch.equal(an.hf, a.hf) and torch.equal(an.state["p"], a.state["p"]), "NaN in zero-weight memory rows changed the result"
    nan = {"p": torch.full_like(c0.hf, float("nan")), "r_prev": torch.full_like(c0.hf, float("nan")), "rho": torch.full((1,), float("nan"), device=c0.hf.device)}
    fresh = _run(c0, S, Y, W, G_, 3, NX[0], dict(kw, direction_forget_factor=0.0))
    poisoned = _run(Call(c0.hf, c0.energy, nan), S, Y, W, G_, 3, NX[0], dict(kw, direction_forget_factor=0.0))
    assert torch.equal(poisoned.hf, fresh.hf), "direction_forget_factor 0 read the NaN CG state"
    if fr and dff != 0:
        st = dict(c5.state, r_prev=torch.full_like(c5.hf, float("nan")))
        fr_nan = _run(Call(c5.hf, c5.energy, st), S, Y, W, G_, 5, NX[1], kw)
        assert torch.equal(fr_nan.hf, a.hf), "Fletcher-Reeves read the NaN r_prev buffer"
    print("eco f64 cg %-40s %s | single %.4f iterates %.4f (e / bar) | e / e_f32 %.2f | bound(hf_0) %.1e"
          % (_cg_id((h, wh, n, c, filled, regk, fr, sa, dff, has_en)), R.plan_label(pl), worst[0], worst[1], worst[2], sb0["d"]))
    assert not fails, "\n  ".join(fails)


def test_eco_filter_cg_tracker_chain():
    """8 consecutive 5-iteration calls on the deep block (15x8, C 64, a 200-slot memory filling from 40), Polak-Ribiere with ECO's
    direction_forget_factor: between calls one slot is filled, the weights renormalised (the new sample weighted by the learning rate),
    new_xf updates the energy and the state is carried; each call from the kernel's own previous output against float64 from there."""
    h, wh, n, c = 15, 8, 200, 64
    sms = _sms()
    REACHED.update(R.plan_features(h, wh, n, c, sms))
    samples, sw, yf, g = _memory(h, wh, n, c, 40, seed=77)
    reg = _reg("eco", h, wh, g)
    kw = dict(fletcher_reeves=False, standard_alpha=True, direction_forget_factor=DFF)
    call = Call((0.01 * torch.randn(1, c, h, wh, 2, generator=g)).cuda())
    worst = [0.0, 0.0]
    for it in range(8):
        nx = torch.randn(1, c, h, wh, 2, generator=g)
        if it:
            slot = 40 + it - 1
            samples[:, :, slot] = nx[0].permute(1, 2, 0, 3)
            sw *= 1 - 0.0075
            sw[slot] = 0.0075
            sw /= sw.sum()
        prob = R.FilterProblem(samples, yf, sw, reg, False, True, DFF, dev=DEV)
        out = _run(call, samples.cuda(), yf.cuda(), sw.cuda(), reg.cuda(), 5, nx.cuda(), kw)
        fails = []
        sb = prob.single_bound(call.hf, call.energy, call.state, nx, sms)
        wb, wf = _check_step(prob, call, out, 5, nx, sms, sb, fails, "call %d" % it)
        worst = [max(worst[0], wb), max(worst[1], wf)]
        assert not fails, "\n  ".join(fails)
        call = out
    print("eco f64 cg tracker chain: 8 calls, worst e / bar %.4f, e / e_f32 %.2f" % tuple(worst))


def test_eco_filter_cg_zz_plan_coverage():
    """The cases above reach every plan feature of the online kernel at this SM count."""
    if not REACHED:
        pytest.skip("no case ran")
    sms = _sms()
    print("eco f64 cg plan features reached on %d SMs: %s" % (sms, "; ".join(sorted(REACHED))))
    assert set(R.PLAN_FEATURES) <= REACHED, sorted(set(R.PLAN_FEATURES) - REACHED)
    assert SEEN == {"reg": {"1x1", "dense3", "eco", "edge"}, "fr": {True, False}, "sa": {True, False}, "dff": {True, False},
                    "energy": {True, False}}, SEEN


# ---- eco_joint_gn_ --------------------------------------------------------------------------------------------------------------------
# (H, Wh, N, Cin, C): at 132 SMs wide 0 with 9 of 16 slabs resident and SPL 16; wide 1 stage_pm 1; stage_pm 0 (Cin 512); all slabs
# streamed (N 200); a grid of 15 with SPL 3 and several tiles per CTA.
JOINT_CASES = [(63, 32, 30, 96, 16), (15, 8, 30, 256, 64), (15, 8, 30, 512, 128), (15, 8, 200, 256, 64), (5, 3, 20, 64, 16)]


@pytest.mark.parametrize("h,wh,n,cin,c", JOINT_CASES, ids=["%dx%d-n%d-%d-%d" % jc for jc in JOINT_CASES])
def test_eco_joint_gn_steps_vs_float64(h, wh, n, cin, c):
    sms = _sms()
    pl = eco_joint_plan(h, wh, n, cin, c, 1, 1, sms)
    JREACHED.update(R.joint_plan_features(h, wh, n, cin, c, sms))
    g = torch.Generator().manual_seed(h * 31 + cin + c)
    samples = torch.randn(h, wh, n, cin, 2, generator=g)
    P0 = torch.linalg.qr(torch.randn(cin, cin, generator=g))[0][:, :c].contiguous()
    _, _, yf, _ = _memory(h, wh, 1, 16, 1, seed=3)
    reg = _reg("eco" if h >= 5 and wh >= 5 else "dense3", h, wh, g)
    sw = torch.full((n,), 1.0 / n)
    hf0 = 0.01 * torch.randn(1, c, h, wh, 2, generator=g)
    dMh, dMP, _ = E.joint_precond(samples, P0, yf, reg, 0.3, 0.15, 35.0, 5e-8)
    dMh = dMh.reshape(1, c, h, wh).contiguous()
    lam = 5e-8
    prob = R.JointProblem(samples, yf, sw.sqrt(), reg, dMh, float(dMP), lam, dev=DEV)
    S, Y, W, G_, D = samples.cuda(), yf.cuda(), sw.sqrt().cuda(), reg.cuda(), dMh.cuda()

    def run(hf, P, ncg, ngn):
        hk, Pk = hf.clone().cuda().contiguous(), P.clone().cuda().contiguous()
        ops.eco_joint_gn_(hk, Pk, S, Y, W, G_, D, float(dMP), lam, ncg, ngn)
        torch.cuda.synchronize()
        return hk, Pk

    def errs(hf, P, h1, P1, ref):
        out = []
        for a, a1, r in ((hf, h1, ref[0]), (P, P1, ref[1])):
            a1d = a1.detach().to(r.device).double().reshape(r.shape)
            out.append(R.rel_err(a1d - a.detach().to(r.device).double().reshape(r.shape), r, U * a1d.abs()))
        return out

    fails, worst = [], [0.0, 0.0, 0.0, 0.0]
    sb = prob.single_bound(hf0, P0, sms)
    for k in range(1, 11):
        h1, P1 = run(hf0, P0, k, 1)
        ref = prob.step(hf0, P0, k)
        e = errs(hf0, P0, h1, P1, ref)
        e32 = prob.e32(hf0, P0, k, ref)
        for b, name in ((0, "dh"), (1, "dP")):
            bar = sb[b] if k == 1 else max(4 * e32[b], k * sb[b])
            worst[0 if k == 1 else 1] = max(worst[0 if k == 1 else 1], e[b] / bar)
            worst[3] = max(worst[3], e[b] / e32[b])
            if e[b] > bar or e[b] > R.F32_FACTOR * e32[b]:
                fails.append("%d CG iterations, %s: e %.3e > bar %.3e or %d x e_f32 %.3e" % (k, name, e[b], bar, R.F32_FACTOR, e32[b]))
    # a chain of single-GN calls, each from the kernel's own output, against float64 from that point
    hf, P = hf0.cuda(), P0.cuda()
    for it in range(3):
        h1, P1 = run(hf, P, 5, 1)
        ref = prob.step(hf, P, 5)
        e32 = prob.e32(hf, P, 5, ref)
        sbi = prob.single_bound(hf, P, sms)
        e = errs(hf, P, h1, P1, ref)
        for b, name in ((0, "dh"), (1, "dP")):
            bar = max(4 * e32[b], 5 * sbi[b])
            worst[2] = max(worst[2], e[b] / bar)
            if e[b] > bar or e[b] > R.F32_FACTOR * e32[b]:
                fails.append("GN chain %d, %s: e %.3e > bar %.3e or %d x e_f32 %.3e" % (it, name, e[b], bar, R.F32_FACTOR, e32[b]))
        hf, P = h1, P1
    h3, P3 = run(hf0, P0, 5, 3)
    assert torch.equal(h3, hf) and torch.equal(P3, P), "three GN iterations in one call differ from three chained calls"
    print("eco f64 gn %-22s %s | single %.4f CG iterates %.4f chain %.4f (e / bar) | e / e_f32 %.2f | bound dh %.1e dP %.1e"
          % ("%dx%d n%d %d->%d" % (h, wh, n, cin, c), R.joint_plan_label(pl), worst[0], worst[1], worst[2], worst[3], sb[0], sb[1]))
    assert not fails, "\n  ".join(fails)


def test_eco_joint_gn_zz_plan_coverage():
    if not JREACHED:
        pytest.skip("no case ran")
    print("eco f64 gn plan features reached on %d SMs: %s" % (_sms(), "; ".join(sorted(JREACHED))))
    assert set(R.JOINT_PLAN_FEATURES) <= JREACHED, sorted(set(R.JOINT_PLAN_FEATURES) - JREACHED)


# ---- score path -------------------------------------------------------------------------------------------------------------------------
def _entrywise(ker, ref, terms, depth, label):
    bound = depth * U * terms + U * ref.abs()
    r = float(((ker.detach().double().cpu() - ref).abs() / bound.clamp(min=1e-300)).max())
    assert r <= 1.0, "%s: worst |k - f64| / bound %.3f" % (label, r)
    return r


def test_eco_score_path_vs_float64():
    g = torch.Generator().manual_seed(29)
    worst = {}
    # eco_apply_filter: a chain of C complex products per entry
    for S, C, h, wh in ((5, 16, 63, 32), (5, 64, 15, 8), (3, 128, 13, 7)):
        hf, xf = 0.1 * torch.randn(1, C, h, wh, 2, generator=g), torch.randn(S, C, h, wh, 2, generator=g)
        sf = ops.eco_apply_filter(hf.cuda(), xf.cuda())
        terms = (R.mag(hf.double()) * R.mag(xf.double())).sum(1, keepdim=True).unsqueeze(-1)
        worst["apply_filter"] = max(worst.get("apply_filter", 0), _entrywise(sf, E.apply_filter(hf.double(), xf.double()), terms, R.S2 * (2 * C + 2),
                                                                               "apply_filter C %d" % C))
    # eco_sample_fs: two weighted blocks at 5 scales on odd, even, non-square grids, a grid smaller than the series' 2 Wh - 1 columns
    # would be refused; 250 x 250 is ECO's
    nmaps = 0
    for (hb, wb), (h2, w2), out in (((63, 32), (15, 8), (250, 250)), ((15, 8), (9, 5), (17, 17)), ((15, 8), (9, 5), (16, 16)),
                                    ((21, 11), (7, 4), (40, 23)), ((9, 5), (5, 3), (12, 10))):
        blocks = [torch.randn(5, 1, hb, wb, 2, generator=g), 0.5 * torch.randn(5, 1, h2, w2, 2, generator=g)]
        yy = torch.arange(hb).view(-1, 1) - (hb - 1) / 2
        blocks[0] = blocks[0] + 6 * torch.exp(-0.1 * (yy ** 2 + torch.arange(wb).view(1, -1) ** 2)).view(1, 1, hb, wb, 1)
        wts = [1.0, 0.6]
        sc = ops.eco_sample_fs([b.cuda() for b in blocks], out, wts)
        fused = E.sum_fs([b.double() for b in blocks], wts)
        ref = E.sample_fs(fused, out)
        fa = E.sum_fs([R.cplx(R.mag(b.double())) for b in blocks], [abs(w) for w in wts])[..., 0]   # |F| summed at its positions
        c = torch.full((fa.shape[-1],), 2.0, dtype=torch.float64)
        c[0] = 1.0
        terms = (fa * c).sum((-2, -1), keepdim=True).expand_as(ref)
        depth = 2 * hb + 4 * wb + 2 * len(blocks) + 30                           # the two series, the fusion, sincospif's twiddles
        worst["sample_fs"] = max(worst.get("sample_fs", 0), _entrywise(sc, ref, terms, depth, "sample_fs %s" % (out,)))
        bnd = 2 * (depth * U * terms.reshape(5, -1)[:, 0] + U * ref.reshape(5, -1).abs().max(1).values)
        flat_k, flat_r = sc.double().cpu().reshape(5, -1), ref.reshape(5, -1)
        top2 = flat_r.topk(2, 1).values
        for s in range(5):
            if float(top2[s, 0] - top2[s, 1]) > float(bnd[s]):
                nmaps += 1
                assert int(flat_k[s].argmax()) == int(flat_r[s].argmax()), "sample_fs %s: arg-max differs from float64" % (out,)
    # eco_preprocess_sample_: window (compared bit for bit), the two DFT stages, the interpolation; contiguous and the tracker's permuted view
    for S, C, hh, ww, permuted in ((3, 16, 62, 62, True), (2, 64, 15, 15, False), (2, 8, 14, 20, True), (1, 4, 9, 8, False)):
        x = torch.randn(S, C, hh, ww, generator=g)
        win = torch.rand(1, 1, hh, ww, generator=g)
        hp, whp = hh + (hh + 1) % 2, ww // 2 + 1
        iy, ix = torch.randn(1, 1, hp, 1, 2, generator=g), torch.randn(1, 1, 1, whp, 2, generator=g)
        xd = x.clone().cuda()
        if permuted:
            xd = xd.permute(2, 3, 0, 1).contiguous().permute(2, 3, 0, 1)
        xf = ops.eco_preprocess_sample_(xd, win.cuda(), iy.cuda(), ix.cuda())
        v = x * win
        assert torch.equal(xd.cpu(), v), "preprocess_sample: the window is not applied in place bit for bit"
        ref, _ = E.preprocess_sample(v.double(), torch.ones(1, 1, hh, ww, dtype=torch.float64), iy.double(), ix.double())
        terms = v.double().abs().sum((2, 3)).view(S, C, 1, 1) * R.mag(iy.double()).view(1, 1, hp, 1) * R.mag(ix.double()).view(1, 1, 1, whp)
        worst["preprocess"] = max(worst.get("preprocess", 0), _entrywise(xf, ref, terms.unsqueeze(-1), R.S2 * (ww + 2 * hh + 30),
                                                                         "preprocess %dx%d" % (hh, ww)))
    # eco_shift_fs: against float64 at the phase the reference forms in float32 (the shift times the frequency, DESIGN 4.9)
    for S, C, hh, wh, sy, sx in ((5, 16, 63, 32, 0.731, -2.9), (1, 64, 15, 8, -11.37, 4.02), (2, 8, 9, 5, 0.0, 1e-3)):
        a = torch.randn(S, C, hh, wh, 2, generator=g)
        out = ops.eco_shift_fs(a.cuda(), sy, sx)
        ky = torch.arange(-((hh - 1) // 2), hh // 2 + 1, dtype=torch.float32)
        kx = torch.arange(0, wh, dtype=torch.float32)
        py = (torch.tensor(sy, dtype=torch.float32) * ky).double().view(1, 1, hh, 1)
        px = (torch.tensor(sx, dtype=torch.float32) * kx).double().view(1, 1, 1, wh)
        ref = E.cmul(E.cmul(a.double(), torch.stack((py.cos(), py.sin()), -1)), torch.stack((px.cos(), px.sin()), -1))
        worst["shift_fs"] = max(worst.get("shift_fs", 0), _entrywise(out, ref, R.mag(a.double()).unsqueeze(-1), 16, "shift_fs %dx%d" % (hh, wh)))
    assert nmaps >= 10, nmaps
    print("eco f64 score path: worst |k - f64| / bound %s; arg-max exact on %d maps where the gap allows"
          % (", ".join("%s %.4f" % kv for kv in worst.items()), nmaps))
