"""CPU tier of tests/test_atom_steps_f64_gpu.py: pins tests/atom_step_ref.py, then runs its bars on the CG kernel's own source.

  * the float64 steps equal a Gauss-Newton step built from autograd (J^T J p from torch.func.jvp / vjp of the residual function, M1
    applied for FactorizedConvProblem) at 1e-12, and central differences of the objective confirm the gradient b;
  * in float32 the helper's operands reproduce the reference classes' goldens (tests/golden/atom_cg.npz, atom_gn.npz);
  * `cg_plan` reproduces launch_cg's plans at 132 and 114 SMs;
  * csrc/atom_cg_kernel.cuh, built as host code with whole cooperative grids (tests/cpu_emul/cg_emul.cpp, fibers) and the pipeline depth
    launch_cg picks, meets the single-step bound and the k-iteration rule at 132 and 114 SMs for FS 18 and 22."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import atom_step_ref as R
from oracle import atom_oracle as A
from pytracking_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACT = {"none": 0, "relu": 1, "elu": 2, "mlu": 3}

PLANS = {(18, 16, 12): ((1, 1, 12, 1, 4), (1, 1, 12, 1, 4)),
         (18, 64, 40): ((1, 4, 33, 2, 4), (1, 4, 28, 2, 4)),
         (18, 64, 250): ((1, 4, 33, 8, 3), (2, 2, 57, 5, 4)),
         (18, 64, 330): ((2, 2, 66, 5, 4), (2, 2, 57, 6, 3)),
         (18, 64, 600): ((4, 1, 132, 5, 3), (4, 1, 114, 6, 3)),
         (22, 64, 40): ((1, 4, 33, 2, 3), (1, 4, 28, 2, 3)),
         (22, 64, 250): ((1, 4, 33, 8, 2), (2, 2, 57, 5, 2)),
         (18, 256, 250): ((4, 4, 33, 8, 3), None)}


def test_cg_plan_reproduces_the_launcher():
    for (fs, c, n), want in PLANS.items():
        for sms, w in zip((132, 114), want):
            p = R.cg_plan(n, c, fs, sms)
            got = None if p is None else (p["passes"], p["NCH"], p["NG"], p["spc"], p["NST"])
            assert got == w, (fs, c, n, sms, got, w)
    assert "NG < n, uneven groups" in R.plan_features(250, 64, 18, 132)          # 250 = 19 * 8 + 14 * 7
    assert "n = NG * CG_SPC_MAX" in R.plan_features(264, 64, 18, 132)


def _phi(s, act):
    return A.activation(s, act, 0.05)


@pytest.mark.parametrize("act", ["none", "elu", "mlu", "relu"])
def test_cg_step_equals_autograd_gauss_newton(act):
    x, y, sw = synth.make_atom_memory(3, 6, 16, 18, 18, n_filled=5)
    w = 0.05 * torch.randn(1, 16, 4, 4, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    prob = R.ConvProblem(x, y, sw, 0.1, act)
    X, Y, S = prob.X, prob.y, prob.sw.view(-1, 1, 1, 1)

    def f(wt):
        return torch.cat([(S.sqrt() * (_phi(A.conv_same(X, wt), act) - Y)).flatten(), 0.1 ** 0.5 * wt.flatten()])

    f0 = f(w)
    b = -torch.func.vjp(f, w)[1](f0)[0]
    Ab = torch.func.vjp(f, w)[1](torch.func.jvp(f, (w,), (b,))[1])[0]
    d = float((b * b).sum() / (b * Ab).sum()) * b
    assert float((prob.step(w, 1) - d).abs().max() / d.abs().max()) < 1e-12
    # the gradient b against central differences of the objective |f|^2 (b = -grad / 2)
    g = torch.Generator().manual_seed(5)
    for _ in range(3):
        v = torch.randn(w.shape, generator=g, dtype=torch.float64)
        h = 1e-6
        fd = (float((f(w + h * v) ** 2).sum()) - float((f(w - h * v) ** 2).sum())) / (2 * h)
        assert abs(fd + 2 * float((b * v).sum())) <= 1e-6 * abs(fd) + 1e-9


@pytest.mark.parametrize("act,fr", [("mlu", True), ("elu", False)])
def test_gn_step_equals_autograd_gauss_newton(act, fr):
    x, y, sw = synth.make_atom_memory(7, 4, 20, 18, 18)
    g = torch.Generator().manual_seed(8)
    w = 0.05 * torch.randn(1, 16, 4, 4, generator=g, dtype=torch.float64)
    P = torch.randn(16, 20, 1, 1, generator=g, dtype=torch.float64) / 4
    rw, rP = 0.1, 1e-2
    prob = R.FactorizedProblem(x, y, sw, rw, rP, act, 0.05, fr)
    X, Y, S = prob.X, prob.y, prob.sw.view(-1, 1, 1, 1)

    def f(wt, Pt):
        s = A.conv_same(A.conv1x1(X, Pt), wt)
        return torch.cat([(S.sqrt() * (_phi(s, act) - Y)).flatten(), rw ** 0.5 * wt.flatten(), rP ** 0.5 * Pt.flatten()])

    f0, vjp = torch.func.vjp(f, w, P)
    rw_, rP_ = [-t for t in vjp(f0)]
    zw, zP = rw_ / rw, rP_ / rP                                                      # M1
    Jz = torch.func.jvp(f, (w, P), (zw, zP))[1]
    qw, qP = vjp(Jz)
    alpha = float((rw_ * zw).sum() + (rP_ * zP).sum()) / float((zw * qw).sum() + (zP * qP).sum())
    dw, dP = prob.step(w, P, 1)
    assert float((dw - alpha * zw).abs().max() / dw.abs().max()) < 1e-12
    assert float((dP - alpha * zP).abs().max() / dP.abs().max()) < 1e-12
    h, v = 1e-6, torch.randn(P.shape, generator=g, dtype=torch.float64)
    fd = (float((f(w, P + h * v) ** 2).sum()) - float((f(w, P - h * v) ** 2).sum())) / (2 * h)
    assert abs(fd + 2 * float((rP_ * v).sum())) <= 1e-6 * abs(fd) + 1e-9


def _golden(name):
    return np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))


@pytest.mark.parametrize("tag,n,c,nf,it,fr,act,seed", [("n12_c16_pr_mlu", 12, 16, 12, 5, False, "mlu", 51), ("n9_c32_fr_none", 9, 32, 9, 4, True, "none", 53)])
def test_helper_float32_reproduces_reference_goldens(tag, n, c, nf, it, fr, act, seed):
    g = _golden("atom_cg")
    x, y, sw = synth.make_atom_memory(seed, n, c, 18, 18, n_filled=nf)
    w0 = torch.from_numpy(g[tag + "_w0"])
    prob = R.ConvProblem(x, y, sw, 0.1, act, 0.05, fr)
    d = A.atom_cg_filter(w0, prob.X32, prob.y32, prob.sw32, 0.1, it, act, 0.05, fr)[1]
    ref = g[tag + "_w"].astype(np.float64) - w0.double().numpy()
    assert np.abs(d.double().numpy() - ref).max() / np.abs(ref).max() < 1e-4
    assert float((prob.step(w0, it).numpy() - ref).__abs__().max() / np.abs(ref).max()) < 1e-4


def test_helper_float32_reproduces_gn_golden():
    g = _golden("atom_gn")
    tag, (n, cin, cc, ncg, ngn, fr, act, seed) = "n6_c32_16", (6, 32, 16, 3, 2, True, "mlu", 101)
    x, y, sw = synth.make_atom_memory(seed, n, cin, 18, 18)
    w0, P0 = torch.from_numpy(g[tag + "_w0"]), torch.from_numpy(g[tag + "_P0"])
    prob = R.FactorizedProblem(x, y, sw, 0.1, 1e-2, act, 0.05, fr)
    w, P = A.atom_gn_joint(w0, P0, prob.X32, prob.y32, prob.sw32, 0.1, 1e-2, ncg, ngn, act, 0.05, fr)
    assert float((w.numpy() - g[tag + "_w"]).__abs__().max() / np.abs(g[tag + "_w"]).max()) < 1e-4
    assert float((P.numpy() - g[tag + "_P"]).__abs__().max() / np.abs(g[tag + "_P"]).max()) < 1e-4


# ---- the kernel source under the bars ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cg_coop(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("cg_emul_coop")), "libcg_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    "-DB200_EMUL_COOP_FIBERS", os.path.join(ROOT, "tests", "cpu_emul", "cg_emul.cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


def _emul_cg(lib, w, x, y, sw, k, fr, act, sms):
    n, c, h = x.shape[0], x.shape[1], x.shape[-1]
    out = np.full((1, c, 4, 4), np.nan, np.float32)
    a = [np.ascontiguousarray(t.numpy(), dtype=np.float32) for t in (w, x, y, sw)]
    p = lambda z: z.ctypes.data_as(C.c_void_p)
    assert lib.cg_emul_atom_cg_filter(p(a[0]), p(out), p(a[1]), p(a[2]), p(a[3]), n, c, h, h, k, C.c_float(0.1), int(fr), ACT[act],
                                      C.c_float(0.05), sms) == 0
    return torch.from_numpy(out)


def check_kernel_steps(lib, fs, c, n, nf, act, fr, sms, ks=(1, 2, 3, 5)):
    """The GPU file's bars on the emulated kernel: the single step from w_0 and from the 5-iteration result, k iterations from w_0.
    Returns a list of failures (index of the first failing step first)."""
    x, y, sw = synth.make_atom_memory(300 + n + c + fs, n, c, fs, fs, n_filled=nf)
    w0 = 0.02 * torch.randn(1, c, 4, 4, generator=torch.Generator().manual_seed(n))
    prob = R.ConvProblem(x, y, sw, 0.1, act, 0.05, fr)
    depths = R.cg_depths(n, c, fs, sms)
    sb0 = prob.single_bound(w0, depths)
    cells0 = prob.kink_cells(w0)
    fails = []
    for k in ks:
        wk = _emul_cg(lib, w0, x, y, sw, k, fr, act, sms)
        ref = prob.step(w0, k)
        allow = prob.kink_allowance(w0, k, cells0, ref) + R.U * wk.double().abs()
        e = float(((wk.double() - w0.double() - ref).abs() - allow).clamp(min=0).max() / ref.abs().max())
        e32 = prob.e32(w0, k, ref)
        bar = sb0 if k == 1 else max(4 * e32, k * sb0)
        if not (e <= bar and e <= R.F32_FACTOR * e32):
            fails.append("k %d: e %.3e > bar %.3e or %d x e_f32 %.3e" % (k, e, bar, R.F32_FACTOR, e32))
    w5 = _emul_cg(lib, w0, x, y, sw, 5, fr, act, sms)
    w6 = _emul_cg(lib, w5, x, y, sw, 1, fr, act, sms)
    ref = prob.step(w5, 1)
    cells = prob.kink_cells(w5)
    allow = prob.kink_allowance(w5, 1, cells, ref) + R.U * w6.double().abs()
    e = float(((w6.double() - w5.double() - ref).abs() - allow).clamp(min=0).max() / ref.abs().max())
    if not (e <= prob.single_bound(w5, depths) and e <= R.F32_FACTOR * prob.e32(w5, 1, ref)):
        fails.append("single step from w_5: e %.3e" % e)
    return fails


# (FS, C, n, filled, act, FR): at 132 SMs 1/4/33/2/4 and 1/4/33/2/3 (FS 22), at 114 SMs 1/4/28/2/4 and 1/4/28/2/3
@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("fs,c,n,nf,act,fr", [(18, 64, 40, 25, "mlu", False), (22, 64, 40, 40, "relu", True), (18, 16, 12, 12, "elu", False)])
def test_cg_kernel_source_meets_the_step_bars(cg_coop, fs, c, n, nf, act, fr, sms):
    fails = check_kernel_steps(cg_coop, fs, c, n, nf, act, fr, sms)
    assert not fails, (R.cg_plan(n, c, fs, sms), fails)
