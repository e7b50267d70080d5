"""-m gpu: the stage-2 kernels (csrc/corr_kernels.cuh: apply_filter with its last-CTA reduction and fused arg-max, conv2d_same,
feat_transpose, max2d) entry by entry against float64 (tests/corr_ref.py), at cases chosen through the launch plan at this device's SM
count so that between them they reach every plan feature (corr_ref.required_features; the zz test asserts it and prints one report line
per case).

  float      seeded normal operands; every entry within gamma_D sum|terms| + u|k| for the plan's depth D; the fused arg-max equals
             dcf.max2d of the kernel's own map bit for bit, and the float64 arg-max wherever the float64 top-two gap exceeds twice the bar;
             conv2d_same equals apply_filter's map cropped to [:FS, :FS] bit for bit; adjointness <A w, r> = <w, A^T r>.
  integer    operands from {-2, ..., 2}: every partial sum is an integer below 2^24, so apply, conv2d_same and the adjoint equal float64
             bit for bit at every plan, and the exact ties pin the arg-max tie order against float64.
  sequence   one process through interleaved calls of both feature sizes with n going 50 -> 3 -> 1024 -> 1 (the workspace grows in the
             middle): every output equals the first run of the same call bit for bit.
  refusals   unsupported shapes and arguments return an error and leave the output untouched.
  max2d      bit for bit against dcf.max2d on shapes from 1x1 to 289x300 with ties, +-0, +-inf, denormals and NaN.
  localize   the score pre-processing of the localisation kernel ('exp', 'softmax' with and without softmax_reg) against softmax_reg_kernel
             bit for bit and float64 within a bound of its arithmetic; softmax_reg_kernel itself entry by entry.
Every output buffer is filled with NaN before each call, so that a stale result cannot pass."""
import ctypes as C

import numpy as np
import pytest
import torch

import corr_ref as R

pytestmark = pytest.mark.gpu
U = R.U
REPORT = {}
REACHED = set()


@pytest.fixture(scope="module")
def L():
    from pytracking_b200 import _lib
    return _lib.lib()


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _err(L):
    m = L.b200trk_last_error()
    return m.decode() if m else ""


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def _run(L, op, x, y, want_max=False):
    """One call through the C ABI into NaN-filled outputs: op 'apply' (y = w; with the fused arg-max when want_max), 'same' or 'adjoint'
    (y = r).  Returns (out, max_val, max_idx)."""
    n, Cc, H, W = x.shape
    mv = mi = None
    if op == "adjoint":
        out = _nan(1, Cc, 4, 4)
        rc = L.b200trk_apply_feat_transpose(_p(x), _p(y), _p(out), n, Cc, H, W, 4, _st())
    elif op == "same":
        out = _nan(n, 1, H, W)
        rc = L.b200trk_conv2d_same(_p(x), _p(y), _p(out), n, Cc, H, W, 4, _st())
    else:
        out = _nan(n, 1, H + 1, W + 1)
        if want_max:
            mv, mi = _nan(n), torch.full((n, 2), -7, dtype=torch.int64, device="cuda")
        rc = L.b200trk_apply_filter(_p(x), _p(y), _p(out), n, Cc, H, W, 4, _p(mv), _p(mi), _st())
    assert rc == 0, (op, x.shape, _err(L))
    torch.cuda.synchronize()
    return out, mv, mi


def _operands(FS, n, Cc, integer, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if integer:
        draw = lambda *s: torch.randint(-2, 3, s, generator=g, device="cuda").float()
        return draw(n, Cc, FS, FS), draw(1, Cc, 4, 4), draw(n, 1, FS + 1, FS + 1)
    return (torch.randn(n, Cc, FS, FS, generator=g, device="cuda"), 0.3 * torch.randn(1, Cc, 4, 4, generator=g, device="cuda"),
            torch.randn(n, 1, FS + 1, FS + 1, generator=g, device="cuda"))


def _ratio(k, ref, mag, D, what):
    """Assert every entry within the bar; return the worst error-to-bar ratio."""
    assert not torch.isnan(k).any(), "%s: entries left unwritten (NaN)" % what
    err = (k.double() - ref).abs()
    b = R.bar(k, mag, D)
    bad = err > b
    assert not bad.any(), "%s: %d entries above the bar, worst |k - f64| %.3e at bar %.3e" % (what, int(bad.sum()), float(err[bad].max()),
                                                                                              float(b[bad][err[bad].argmax()]))
    return float((err / b.clamp_min(1e-300)).max())


def _argmax_vs_f64(s, mi, ref, mag, D):
    """The kernel's cell is within twice the bar of the float64 maximum, and is the float64 arg-max where the top-two gap exceeds twice the
    bar (corr_ref: test_atom_score_ops_vs_float64's rule).  Returns the number of maps where it was checked exactly."""
    n = s.shape[0]
    fr = ref.reshape(n, -1).cpu()
    bnd = 2 * R.bar(s, mag, D).reshape(n, -1).max(1).values.cpu()
    top2 = fr.topk(2, 1).values
    idx = (mi[:, 0] * s.shape[-1] + mi[:, 1]).cpu()
    exact = 0
    for i in range(n):
        assert float(top2[i, 0] - fr[i, idx[i]]) <= float(bnd[i]), "arg-max cell too far below the float64 maximum (map %d)" % i
        if float(top2[i, 0] - top2[i, 1]) > float(bnd[i]):
            exact += 1
            assert int(idx[i]) == int(fr[i].argmax()), "arg-max differs from float64 (map %d)" % i
    return exact


def _check_case(L, op, FS, n, Cc, integer, seed):
    from oracle import dimp_oracle as O
    plan = R.corr_plan(op, n, Cc, FS, _sms())
    D = plan["depth"]
    x, w, r = _operands(FS, n, Cc, integer, seed)
    tag = "%s FS %d n %d C %d %s" % (op, FS, n, Cc, "int" if integer else "float")
    worst, exact = 0.0, 0
    if op == "apply":
        s, mv, mi = _run(L, "apply", x, w, want_max=True)
        s_nomax, _, _ = _run(L, "apply", x, w)
        sc, _, _ = _run(L, "same", x, w)
        assert torch.equal(_bits(s_nomax), _bits(s)), tag + ": the map without the fused arg-max differs"
        assert torch.equal(_bits(sc), _bits(s[..., :FS, :FS].contiguous())), tag + ": conv2d_same is not apply_filter's map cropped"
        mv_ref, mi_ref = O.max2d(s.cpu()[:, 0])
        assert torch.equal(mi.cpu(), mi_ref) and torch.equal(_bits(mv).cpu(), _bits(mv_ref)), tag + ": fused arg-max is not dcf.max2d"
        ref = R.apply(x, w)
        if integer:
            assert torch.equal(s.double(), ref), tag + ": apply_filter not exact on integers"
            _, mi64 = O.max2d(ref.cpu()[:, 0])
            assert torch.equal(mi.cpu(), mi64), tag + ": arg-max tie order differs from float64"
            exact = n
        else:
            mag = R.magnitude("apply", x, w)
            worst = max(_ratio(s, ref, mag, D, tag), _ratio(sc, ref[..., :FS, :FS], mag[..., :FS, :FS], D, tag + " same"))
            exact = _argmax_vs_f64(s, mi, ref, mag, D)
    else:
        g, _, _ = _run(L, "adjoint", x, r)
        ref = R.adjoint(x, r)
        if integer:
            assert torch.equal(g.double(), ref), tag + ": adjoint not exact on integers"
        else:
            worst = _ratio(g, ref, R.magnitude("adjoint", x, r), D, tag)
            s, _, _ = _run(L, "apply", x, w)
            lhs = float((s.double() * r.double()).sum())
            rhs = float((w.double() * g.double()).sum())
            assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs)), tag + ": <A w, r> != <w, A^T r>"
    REACHED.update(R.features(plan))
    key = (op, FS, n, Cc)
    w0, e0, k0 = REPORT.get(key, (0.0, 0, ""))
    REPORT[key] = (max(w0, worst), e0 + exact, "%s%d n %4d C %4d: passes %d NCH %3d NG %4d spc %d grid %s D %3d" % (
        op, FS, n, Cc, plan["passes"], plan["nch"], plan["ng"], plan["spc_max"], plan["grid"], D))


@pytest.mark.parametrize("op,FS,n,Cc", R.cases(132))
def test_corr_vs_float64(L, op, FS, n, Cc):
    """The case list is fixed; the plan each case gets is the one corr_plan gives at this device's SM count."""
    seed = 100003 * FS + 1009 * n + Cc + (op == "adjoint")
    _check_case(L, op, FS, n, Cc, False, seed)
    _check_case(L, op, FS, n, Cc, True, seed + 1)


def test_corr_call_sequence_bitwise(L):
    """Interleaved apply / conv2d_same / adjoint at FS 18 and 22, n 50 -> 3 -> 1024 -> 1: workspace slots 0 and 1 grow in the middle
    and the arrival counters must have reset after every call.  Integer operands: every first run also equals float64 exactly."""
    seq = [("apply", 18, 50, 512), ("adjoint", 18, 50, 512), ("same", 22, 3, 512), ("adjoint", 22, 3, 64), ("apply", 22, 3, 512),
           ("apply", 22, 1024, 32), ("adjoint", 18, 1024, 512), ("same", 18, 1024, 64), ("apply", 18, 1, 512), ("adjoint", 22, 1, 512),
           ("same", 22, 1, 512)]
    ops_ = {}
    first = {}
    for rnd, order in enumerate((seq, seq[::-1], seq)):
        for key in order:
            op, FS, n, Cc = key
            if key not in ops_:
                ops_[key] = _operands(FS, n, Cc, True, 1000 + len(ops_))
            x, w, r = ops_[key]
            out, mv, mi = _run(L, op, x, r if op == "adjoint" else w, want_max=(op == "apply"))
            res = [out] + ([mv, mi] if op == "apply" else [])
            if key not in first:
                ref = R.adjoint(x, r) if op == "adjoint" else R.apply(x, w, crop=(op == "same"))
                assert torch.equal(out.double(), ref), "%s: first run not exact" % (key,)
                first[key] = res
            else:
                for a, b in zip(res, first[key]):
                    assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                       b.view(torch.int32) if b.dtype == torch.float32 else b), "round %d %s differs from its first run" % (rnd, key)


def test_corr_refusals(L):
    """Each unsupported call returns an error naming the problem and leaves its output untouched."""
    dev = "cuda"

    def refuse(call, out, text):
        before = out.clone()
        rc = call()
        torch.cuda.synchronize()
        assert rc != 0, text
        assert text in _err(L), (text, _err(L))
        assert torch.equal(_bits(out) if out.dtype == torch.float32 else out, _bits(before) if out.dtype == torch.float32 else before), text

    x = torch.zeros(1025, 16, 18, 18, device=dev)
    w = torch.zeros(1, 16, 4, 4, device=dev)
    s = _nan(1025, 1, 19, 19)
    refuse(lambda: L.b200trk_apply_filter(_p(x), _p(w), _p(s), 1025, 16, 18, 18, 4, None, None, _st()), s, "n=1025 > 1024")
    sc = _nan(1025, 1, 18, 18)
    refuse(lambda: L.b200trk_conv2d_same(_p(x), _p(w), _p(sc), 1025, 16, 18, 18, 4, _st()), sc, "n=1025 > 1024")
    x = torch.zeros(2, 20, 18, 18, device=dev)
    w = torch.zeros(1, 20, 4, 4, device=dev)
    s = _nan(2, 1, 19, 19)
    refuse(lambda: L.b200trk_apply_filter(_p(x), _p(w), _p(s), 2, 20, 18, 18, 4, None, None, _st()), s, "must be a multiple of 16")
    g = _nan(1, 20, 4, 4)
    r = torch.zeros(2, 1, 19, 19, device=dev)
    refuse(lambda: L.b200trk_apply_feat_transpose(_p(x), _p(r), _p(g), 2, 20, 18, 18, 4, _st()), g, "must be a multiple of 16")
    x = torch.zeros(2, 16, 22, 22, device=dev)
    s = _nan(2, 1, 23, 23)
    for H, W, text in ((20, 20, "20x20 not supported"), (18, 22, "18x22 not supported")):
        refuse(lambda: L.b200trk_apply_filter(_p(x), _p(w), _p(s), 2, 16, H, W, 4, None, None, _st()), s, text)
        refuse(lambda: L.b200trk_conv2d_same(_p(x), _p(w), _p(s), 2, 16, H, W, 4, _st()), s, text)
        refuse(lambda: L.b200trk_apply_feat_transpose(_p(x), _p(s), _p(g), 2, 16, H, W, 4, _st()), g, "not supported")
    refuse(lambda: L.b200trk_apply_filter(_p(x), _p(w), _p(s), 2, 16, 18, 18, 5, None, None, _st()), s, "filter size 5")
    refuse(lambda: L.b200trk_conv2d_same(_p(x), _p(w), _p(s), 2, 16, 18, 18, 5, _st()), s, "filter size 5")
    refuse(lambda: L.b200trk_apply_feat_transpose(_p(x), _p(s), _p(g), 2, 16, 18, 18, 5, _st()), g, "filter size 5")
    mv = _nan(2)
    refuse(lambda: L.b200trk_apply_filter(_p(x), _p(w), _p(s), 2, 16, 18, 18, 4, _p(mv), None, _st()), mv, "must both be given")
    x = torch.zeros(1, 8200, 22, 22, device=dev)
    r = torch.zeros(1, 1, 23, 23, device=dev)
    g = _nan(1, 8200, 4, 4)
    refuse(lambda: L.b200trk_apply_feat_transpose(_p(x), _p(r), _p(g), 1, 8200, 22, 22, 4, _st()), g, "too many channel chunks (1025)")


MAX2D_SHAPES = [(1024, 1, 1), (1024, 1, 37), (1024, 41, 1), (1024, 19, 19), (1024, 23, 23), (40, 288, 288), (20, 289, 300)]


@pytest.mark.parametrize("N,H,W", MAX2D_SHAPES)
def test_max2d_bitwise_vs_dcf_max2d(L, N, H, W):
    from oracle import dimp_oracle as O
    a = R.max2d_maps(N, H, W, 7 * H + W)
    mv, mi = _nan(N), torch.full((N, 2), -7, dtype=torch.int64, device="cuda")
    assert L.b200trk_max2d(_p(a.cuda()), N, H, W, _p(mv), _p(mi), _st()) == 0, _err(L)
    v_ref, i_ref = O.max2d(a)
    bad = ((_bits(mv).cpu() != _bits(v_ref)) | (mi.cpu() != i_ref).any(1)).nonzero().flatten().tolist()
    assert not bad, "max2d %dx%d differs from dcf.max2d on maps %s (classes %s)" % (H, W, bad[:8], sorted({b % 10 for b in bad}))


def test_fused_argmax_nan(L):
    """NaN in the features reaches the map; the fused arg-max must report it as dcf.max2d does (first NaN cell in the tie order)."""
    from oracle import dimp_oracle as O
    for FS, n, Cc in ((18, 4, 512), (22, 1, 512), (18, 20, 64)):
        x, w, _ = _operands(FS, n, Cc, False, 31 + FS)
        x[0, 5, 3, 7] = float("nan")
        if n > 1:
            x[1].fill_(float("nan"))
            x[2, 0, 17, 0] = float("nan")
        s, mv, mi = _run(L, "apply", x, w, want_max=True)
        v_ref, i_ref = O.max2d(s.cpu()[:, 0])
        assert torch.isnan(v_ref[0])
        assert torch.equal(mi.cpu(), i_ref) and torch.equal(_bits(mv).cpu(), _bits(v_ref)), (FS, n, mi.cpu()[:3], i_ref[:3])


# ------------------------------------------------------------------------------------------------------------------------------------
# the localisation kernel's score pre-processing
# ------------------------------------------------------------------------------------------------------------------------------------
def softmax_f64_bound(x, reg):
    """float64 softmax_reg over the rows of x and the relative bound of softmax_reg_kernel's arithmetic: the rounding of x - m amplified by
    |x - m|, expf's 2 ulp, a block sum of depth ceil(L / 256) + 5 + 3, the add of expf(reg - m) and the division."""
    xd = x.double()
    m = xd.max(1, keepdim=True).values
    ex_all = None
    if reg is not None:
        reg32 = float(np.float32(reg))                                   # the kernels take reg in float32
        m = torch.clamp(m, min=reg32)
    e = torch.exp(xd - m)
    ex = U * (xd - m).abs() + 4 * U                                      # each exp(x - m): argument rounding and 2 ulp of expf
    ex_all = ex.max(1, keepdim=True).values
    den = e.sum(1, keepdim=True)
    if reg is not None:
        den = den + torch.exp(reg32 - m)
        ex_all = torch.maximum(ex_all, U * (reg32 - m).abs() + 4 * U)
    p = e / den
    D = -(-x.shape[1] // 256) + 8
    rel = ex + ex_all + R.gamma(D + 1) + U
    return p, 1.01 * rel * p


def _loc_params(pre, reg):
    from tracker_cases import DIMP50
    from pytracking_b200.tracker import make_params
    return make_params(**dict(DIMP50, score_preprocess=pre, softmax_reg=reg, target_not_found_threshold=-1.0, uncertain_threshold=-1.0,
                              hard_sample_threshold=-1.0))


def _localize(L, scores, params):
    from pytracking_b200 import _lib
    S = scores.shape[0]
    s = scores.cuda().contiguous()
    res = torch.zeros(16, dtype=torch.int32, device="cuda")
    n = np.full((S, 2), 3.0, np.float32)
    pv = np.zeros((S, 2), np.float32)
    _lib.check(L.b200trk_dimp_localize(_p(s), S, s.shape[1], s.shape[2], C.byref(params), n.ctypes.data_as(C.c_void_p),
                                       pv.ctypes.data_as(C.c_void_p), _p(res), _st()), "dimp_localize")
    return _lib.LocResult.from_buffer_copy(res.cpu().numpy().tobytes())


def test_localize_preprocessing_vs_softmax_reg_and_float64(L):
    from pytracking_b200 import ops
    g = torch.Generator().manual_seed(5)
    checked = 0
    for hw in (19, 23):
        for S in (1, 2, 3):
            for pre, reg in (("exp", None), ("softmax", None), ("softmax", 1.3)):
                for trial in range(4):
                    x = 2.0 * torch.rand(S, hw, hw, generator=g) - 1.0
                    for s in range(S):
                        for _ in range(1 + trial % 3):
                            x[s, int(torch.randint(0, hw, (1,), generator=g)), int(torch.randint(0, hw, (1,), generator=g))] = \
                                2.0 + 4.0 * float(torch.rand(1, generator=g))
                    out = _localize(L, x, _loc_params(pre, reg))
                    flat = x.reshape(S, -1)
                    if pre == "exp":
                        p64 = flat.double().exp()
                        bnd = (U * flat.double().abs() + 4 * U) * 1.01 * p64
                    else:
                        pk = ops.softmax_reg(flat.cuda(), reg).cpu()
                        p64, bnd = softmax_f64_bound(flat, reg)
                        assert (pk.double() - p64).abs().le(bnd).all(), ("softmax_reg", hw, S, reg)
                        si = out.scale_ind
                        for (r_, c_), v in (((out.r1, out.c1), out.score1), ((out.r1, out.c1), out.max_score), ((out.r2, out.c2), out.score2)):
                            assert np.float32(v).view(np.int32) == pk[si, r_ * hw + c_].numpy().view(np.int32), (pre, reg, hw, S, trial)
                    si = out.scale_ind
                    for (r_, c_), v in (((out.r1, out.c1), out.score1), ((out.r2, out.c2), out.score2)):
                        ref, b = float(p64[si, r_ * hw + c_]), float(bnd[si, r_ * hw + c_])
                        assert abs(float(np.float32(v)) - ref) <= b, (pre, reg, hw, S, trial, v, ref, b)
                    # the first cell: the float64 arg-max over every scale wherever the gap allows
                    b2 = 2 * float(bnd.max())
                    top2 = p64.reshape(-1).topk(2).values
                    if float(top2[0] - top2[1]) > b2:
                        j = int(p64.reshape(-1).argmax())
                        assert (out.scale_ind, out.r1 * hw + out.c1) == (j // (hw * hw), j % (hw * hw)), (pre, reg, hw, S, trial)
                        checked += 1
    assert checked >= 40, checked
    REPORT[("localize",)] = (0.0, checked, "localize pre-processing: exp / softmax / softmax_reg at S 1-3 on 19^2 and 23^2")


def test_zz_corr_features_reached():
    """Every plan feature was reached at this device's SM count; one report line per case."""
    sms = _sms()
    missing = R.required_features() - REACHED
    assert not missing, "plan features not reached at %d SMs: %s" % (sms, sorted(missing))
    print("\nstage-2 kernels vs float64 on %s (%d SMs)" % (torch.cuda.get_device_name(), sms))
    for key in sorted(REPORT, key=str):
        worst, exact, line = REPORT[key]
        print("  %s | worst err/bar %.4f | arg-max exact %d" % (line, worst, exact))
