"""CPU tier of tests/test_corr_f64_gpu.py: the float64 helper (tests/corr_ref.py) pinned to the reference goldens, its plan mirror pinned to
the kernels' own corr_plan (csrc/corr_kernels.cuh, exported by tests/cpu_emul/corr_emul.cpp) at 132, 114 and 148 SMs, and the GPU file's
small cases run on the kernel sources under the CPU emulator at 132 and 114 SMs: float, integer, call sequence, max2d and NaN."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import corr_ref as R
from pytracking_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SMS = (132, 114)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("corr_f64_emul")), "libcorr_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", "corr_emul.cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _run(emul, op, x, y, sms=132, want_max=False):
    x = np.ascontiguousarray(x.numpy(), np.float32)
    y = np.ascontiguousarray(y.numpy(), np.float32)
    n, c, h, _ = x.shape
    mv = mi = None
    if op == "adjoint":
        out = np.full((1, c, 4, 4), np.nan, np.float32)
        rc = emul.corr_emul_feat_transpose(_p(x), _p(y), _p(out), n, c, h, h, sms)
    else:
        crop = op == "same"
        out = np.full((n, 1, h + (not crop), h + (not crop)), np.nan, np.float32)
        if want_max:
            mv, mi = np.full(n, np.nan, np.float32), np.full((n, 2), -7, np.int64)
        rc = emul.corr_emul_apply_filter(_p(x), _p(y), _p(out), n, c, h, h, _p(mv), _p(mi), int(crop))
    assert rc == 0, (op, x.shape, rc)
    return out, mv, mi


def test_helper_matches_reference_goldens_and_permutations():
    g = np.load(os.path.join(GOLDEN, "corr.npz"))
    for tag, n, c, h in (("a", 3, 32, 18), ("b", 2, 64, 22)):
        feat = synth.make_clf_features(100 + ord(tag), n, c, h, h)
        w = torch.from_numpy(g[tag + "_w"])
        r = torch.from_numpy(g[tag + "_r"])[:, 0:1].contiguous()
        s = R.apply(feat, w)
        ref = g[tag + "_scores"].reshape(s.shape)
        assert np.abs(s.numpy() - ref).max() <= 1e-5 * np.abs(ref).max()
        gr = R.adjoint(feat, r)
        assert np.abs(gr.numpy() - g[tag + "_grad"]).max() <= 1e-5 * np.abs(g[tag + "_grad"]).max()
        # channels and samples permuted: the same sums in another order
        pc, ps = torch.randperm(c, generator=torch.Generator().manual_seed(1)), torch.randperm(n, generator=torch.Generator().manual_seed(2))
        s2 = R.apply(feat[ps][:, pc], w[:, pc])
        assert (s2 - s[ps]).abs().max() <= 1e-12 * s.abs().max()
        g2 = R.adjoint(feat[ps][:, pc], r[ps])
        assert (g2 - gr[:, pc]).abs().max() <= 1e-12 * gr.abs().max()
        assert torch.equal(R.apply(feat, w, crop=True), s[..., :h, :h])


def test_plan_mirror_matches_kernel_plan(emul):
    out = np.zeros(5, np.int32)
    shapes = {(op, FS, n, c) for op, FS, n, c in R.cases(132)}
    shapes |= {(op, FS, n, c) for op in ("apply", "adjoint") for FS in (18, 22) for n in (1, 2, 7, 15, 16, 17, 33, 50, 100, 250, 513, 1024)
               for c in (8, 16, 24, 40, 48, 64, 96, 128, 200, 256, 512, 1080, 2048, 8200)}
    for sms in (132, 114, 148):
        for op, FS, n, c in sorted(shapes):
            assert emul.corr_emul_plan(int(op == "adjoint"), n, c, FS, sms, _p(out)) == 0
            p = R.corr_plan(op, n, c, FS, sms)
            assert [p["passes"], p["nch"], p["ng"], p["spc_max"], p["slots"]] == out.tolist(), (op, FS, n, c, sms, p, out)


@pytest.mark.parametrize("sms", SMS)
def test_every_plan_feature_reachable(sms):
    missing = R.required_features() - R.all_features(sms)
    assert not missing, (sms, sorted(missing))


def _operands(FS, n, c, integer, seed):
    g = torch.Generator().manual_seed(seed)
    if integer:
        draw = lambda *s: torch.randint(-2, 3, s, generator=g).float()
        return draw(n, c, FS, FS), draw(1, c, 4, 4), draw(n, 1, FS + 1, FS + 1)
    return torch.randn(n, c, FS, FS, generator=g), 0.3 * torch.randn(1, c, 4, 4, generator=g), torch.randn(n, 1, FS + 1, FS + 1, generator=g)


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("op,FS,n,c", R.cases(132, small=True))
def test_kernel_sources_vs_float64(emul, sms, op, FS, n, c):
    from oracle import dimp_oracle as O
    plan = R.corr_plan(op, n, c, FS, sms)
    for integer in (False, True):
        x, w, r = _operands(FS, n, c, integer, 17 * n + c + FS)
        if op == "apply":
            s, mv, mi = _run(emul, "apply", x, w, want_max=True)
            sc, _, _ = _run(emul, "same", x, w)
            assert np.array_equal(_bits(sc), _bits(s[..., :FS, :FS]))
            v_ref, i_ref = O.max2d(torch.from_numpy(s)[:, 0])
            assert np.array_equal(mi, i_ref.numpy()) and np.array_equal(_bits(mv), _bits(v_ref.numpy()))
            ref = R.apply(x, w).numpy()
            k, mag = s, R.magnitude("apply", x, w).numpy()
        else:
            k, _, _ = _run(emul, "adjoint", x, r, sms)
            ref, mag = R.adjoint(x, r).numpy(), R.magnitude("adjoint", x, r).numpy()
        if integer:
            assert np.array_equal(k.astype(np.float64), ref), (op, FS, n, c, sms)
        else:
            bar = R.gamma(plan["depth"]) * mag + R.U * np.abs(k.astype(np.float64))
            assert (np.abs(k - ref) <= bar).all(), (op, FS, n, c, sms, float((np.abs(k - ref) / bar).max()))


def test_call_sequence_bitwise(emul):
    """Interleaved calls with the arrival counters kept across them (as in the library's workspace): every repeat equals its first run."""
    seq = [("apply", 18, 5, 64), ("adjoint", 18, 5, 64), ("same", 22, 3, 16), ("adjoint", 22, 3, 24), ("apply", 22, 17, 32),
           ("adjoint", 18, 17, 128), ("apply", 18, 1, 512), ("same", 18, 1, 48)]
    first = {}
    for rnd, order in enumerate((seq, seq[::-1])):
        for sms in SMS:
            for key in order:
                op, FS, n, c = key
                x, w, r = _operands(FS, n, c, True, n + c + FS)
                out = _run(emul, op, x, r if op == "adjoint" else w, sms, want_max=(op == "apply"))
                res = [out[0]] + ([out[1], out[2]] if op == "apply" else [])
                if key not in first:
                    ref = (R.adjoint(x, r) if op == "adjoint" else R.apply(x, w, crop=(op == "same"))).numpy()
                    assert np.array_equal(out[0].astype(np.float64), ref), key
                    first[key] = res
                else:
                    for a, b in zip(res, first[key]):
                        assert np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                              b.view(np.int32) if b.dtype == np.float32 else b), (rnd, sms, key)


@pytest.mark.parametrize("N,H,W", [(60, 1, 1), (60, 1, 37), (60, 41, 1), (60, 19, 19), (60, 23, 23), (10, 288, 288), (10, 289, 300)])
def test_max2d_kernel_source_bitwise_vs_dcf_max2d(emul, N, H, W):
    from oracle import dimp_oracle as O
    a = R.max2d_maps(N, H, W, 7 * H + W)
    mv, mi = np.full(N, np.nan, np.float32), np.full((N, 2), -7, np.int64)
    assert emul.corr_emul_max2d(_p(np.ascontiguousarray(a.numpy())), N, H, W, _p(mv), _p(mi)) == 0
    v_ref, i_ref = O.max2d(a)
    bad = np.nonzero((_bits(mv) != _bits(v_ref.numpy())) | (mi != i_ref.numpy()).any(1))[0].tolist()
    assert not bad, "max2d %dx%d differs from dcf.max2d on maps %s (classes %s)" % (H, W, bad[:8], sorted({b % 10 for b in bad}))


def test_fused_argmax_nan_kernel_source(emul):
    from oracle import dimp_oracle as O
    for FS, n, c in ((18, 4, 64), (22, 1, 32), (18, 20, 64)):
        x, w, _ = _operands(FS, n, c, False, 31 + FS)
        x[0, 5, 3, 7] = float("nan")
        if n > 1:
            x[1].fill_(float("nan"))
            x[2, 0, 17, 0] = float("nan")
        s, mv, mi = _run(emul, "apply", x, w, want_max=True)
        v_ref, i_ref = O.max2d(torch.from_numpy(s)[:, 0])
        assert torch.isnan(v_ref[0])
        assert np.array_equal(mi, i_ref.numpy()) and np.array_equal(_bits(mv), _bits(v_ref.numpy())), (FS, n, mi[:3], i_ref[:3])
