"""SURVEY 8 row f4 (ECO's Fourier-domain filter optimiser) on the CPU:
  * oracle/eco_oracle.py against tests/golden/eco_cg.npz (outputs of the UNMODIFIED reference FilterOptim, oracle/gen_eco_golden.py);
  * the CUDA kernel source itself (csrc/eco_cg_kernel.cuh) compiled as host code under tests/cpu_emul/cuda_shim.h -- one OS thread
    per CUDA thread, pthread barriers for bar.sync / shuffles / the grid barrier -- against the same golden vectors, over several
    decompositions (grid, block, lane groups per coefficient, resident / streamed slabs), and once under ThreadSanitizer (a missing
    barrier in the kernel is a data race between the emulating threads);
  * the launch plan at ECO's real block sizes (shared memory within the 227 KB a block may use, every slab resident where it fits);
  * the plug-in seam: FilterOptim.run falls through to the reference for CPU tensors.
"""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import eco_oracle as E

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpu_emul"))
from eco_emul_driver import run_emulated as _run_emulated, run_emulated_joint as _run_emulated_joint, rel as _rel  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "eco_cg.npz")
CASES = [(c, r, b) for c in ("pr_forget", "fr_reset") for r in range(3) for b in range(2)]


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("case,run,bi", CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_matches_reference_filter_optim(gold, case, run, bi, dtype):
    g = gold
    fr, sa, dff, pdp, prp = g[case + "/params"]
    k = "%s/run%d/b%d/" % (case, run, bi)
    T = lambda key: torch.from_numpy(g[key]).to(dtype)
    st = {}
    if int(g[k + "has_state"]):
        st = {"p": T(k + "p_in"), "rho": float(g[k + "rho_in"]), "r_prev": T(k + "r_prev_in") if (k + "r_prev_in") in g else None}
    en = T(k + "energy_in") if int(g[k + "has_energy"]) else None
    hf, en2, st2 = E.filter_optim_run(T(k + "hf_in"), T(k + "samples"), T("%s/b%d/yf" % (case, bi)), T(k + "sw"),
                                      T("%s/b%d/reg_filter" % (case, bi)), en, st, int(g[k + "num_iter"]), T(k + "new_xf"),
                                      float(g["%s/b%d/lr" % (case, bi)]), pdp, prp, bool(fr), bool(sa), dff)
    assert _rel(hf, g[k + "hf_out"]) < 2e-5
    assert _rel(en2, g[k + "energy_out"]) < 1e-6
    assert _rel(st2["p"], g[k + "p_out"]) < 2e-5
    assert abs(float(st2["rho"]) - float(g[k + "rho_out"])) < 2e-5 * abs(float(g[k + "rho_out"]))
    if (k + "r_prev_out") in g:
        assert _rel(st2["r_prev"], g[k + "r_prev_out"]) < 2e-5


# ---- the kernel source on the CPU ------------------------------------------------------------------------------------------------
def _build(tmp, tsan=False):
    out = os.path.join(tmp, "libeco_emul%s.so" % ("_tsan" if tsan else ""))
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-fno-gnu-unique", "-Wno-unknown-pragmas"] + \
          (["-fsanitize=thread"] if tsan else []) + [os.path.join(ROOT, "tests", "cpu_emul", "eco_emul.cpp"), "-o", out]
    subprocess.run(cmd, check=True, capture_output=True)
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return C.CDLL(_build(str(tmp_path_factory.mktemp("eco_emul"))))


@pytest.mark.parametrize("case,run,bi", CASES)
def test_emulated_kernel_matches_reference(emul, gold, case, run, bi):
    err, plan, _ = _run_emulated(emul, gold, case, run, bi, 3, 128, -1)
    assert err < 2e-5, (err, plan)


# (co-resident CTAs, threads per CTA, resident slabs forced) -> covers 1 / 2 / 4 / 8 lane groups per coefficient, a CTA per coefficient,
# one CTA for everything, every slab streamed from global memory, partial residency, 64 / 128 / 256 threads
# (at most ~3000 emulating OS threads per launch)
DECOMPOSITIONS = [(1, 64, -1), (5, 64, 0), (45, 64, -1), (10, 256, 1), (7, 256, 2), (1000, 32, -1)]


@pytest.mark.parametrize("max_ctas,block,force_res", DECOMPOSITIONS)
def test_emulated_kernel_is_decomposition_independent(emul, gold, max_ctas, block, force_res):
    seen = set()
    for case, run in (("pr_forget", 1), ("fr_reset", 2)):
        for bi in range(2):
            err, plan, _ = _run_emulated(emul, gold, case, run, bi, max_ctas, block, force_res)
            assert err < 2e-5, (case, run, bi, err, plan)
            seen.add(plan[3])
    assert seen                                                   # lane groups per coefficient actually used


def test_emulated_kernel_is_deterministic(emul, gold):
    a = _run_emulated(emul, gold, "pr_forget", 2, 1, 28, 64, -1)[2]
    b = _run_emulated(emul, gold, "pr_forget", 2, 1, 28, 64, -1)[2]
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_emulated_kernel_under_thread_sanitizer(gold, tmp_path):
    """Every cross-thread hand-over in the kernel is ordered by a barrier: no data race between the emulating threads."""
    tsan_rt = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(tsan_rt) or not os.path.exists(tsan_rt):
        pytest.skip("no ThreadSanitizer runtime")
    lib = _build(str(tmp_path), tsan=True)
    script = (
        "import sys, numpy as np, ctypes as C\n"
        "sys.path.insert(0, %r)\n"
        "from eco_emul_driver import run_emulated as _run_emulated\n"
        "g = np.load(%r)\n"
        "lib = C.CDLL(%r)\n"
        "for ctas, blk, fres in ((3, 64, 1), (28, 64, -1)):\n"
        "    for bi in range(2):\n"
        "        e, plan, _ = _run_emulated(lib, g, 'pr_forget', 1, bi, ctas, blk, fres)\n"
        "        assert e < 2e-5, (e, plan)\n"
        "print('EMUL_DONE')\n" % (os.path.join(ROOT, "tests", "cpu_emul"), GOLD, lib))
    env = dict(os.environ, LD_PRELOAD=tsan_rt, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0")
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, timeout=600, cwd=ROOT)
    if "EMUL_DONE" not in r.stdout and "ThreadSanitizer" not in r.stderr:
        pytest.skip("ThreadSanitizer could not run here: %s" % r.stderr[-300:])
    assert "EMUL_DONE" in r.stdout, r.stderr[-2000:]
    assert "data race" not in r.stderr, r.stderr[:4000]


def test_launch_plan_at_eco_block_sizes(emul):
    """ECO default (parameter/eco/default.py): memory 200, deep block 64 channels on ~15x8 coefficients, shallow block 16 channels on
    ~63x32; 148 SMs and the H100's 132, 256 threads."""
    out = (C.c_longlong * 8)()
    emul.eco_emul_plan(15, 8, 200, 64, 5, 148, 256, out)
    grid, G, CPL, GPP, res, npx_max, smem, ws = list(out)
    assert (grid, G, CPL, GPP, res, npx_max) == (120, 32, 2, 8, 1, 1) and smem <= 227 * 1024      # every slab resident, 8 warps per slab
    emul.eco_emul_plan(63, 32, 200, 16, 5, 148, 256, out)
    grid, G, CPL, GPP, res, npx_max, smem, ws = list(out)
    assert (grid, G, CPL, GPP, npx_max) == (148, 16, 1, 1, 14) and res == 8 and smem <= 227 * 1024  # 8 of <= 14 slabs resident
    emul.eco_emul_plan(31, 16, 250, 128, 5, 148, 256, out)                                          # a slab larger than shared memory
    assert out[4] == 0 and out[6] <= 227 * 1024
    # the launch an H100 makes (132 SMs): the deep block as above, the shallow block with <= 16 coefficients per CTA, 8 of them resident
    emul.eco_emul_plan(15, 8, 200, 64, 5, 132, 256, out)
    grid, G, CPL, GPP, res, npx_max, smem, ws = list(out)
    assert (grid, G, CPL, GPP, res, npx_max) == (120, 32, 2, 8, 1, 1) and smem <= 227 * 1024
    emul.eco_emul_plan(63, 32, 200, 16, 5, 132, 256, out)
    grid, G, CPL, GPP, res, npx_max, smem, ws = list(out)
    assert (grid, G, CPL, GPP, npx_max) == (132, 16, 1, 1, 16) and res == 8 and smem <= 227 * 1024
    emul.eco_emul_plan(31, 16, 250, 128, 5, 132, 256, out)
    assert out[4] == 0 and out[6] <= 227 * 1024


def test_plugin_seam_and_ops_wrapper_over_the_emulated_kernel(emul, gold, monkeypatch):
    """The host side above the C ABI (plugin.install()'s FilterOptim.run + ops.eco_filter_cg_) exercised on the CPU: the library
    entry point is replaced by the emulated kernel (same argument list), the device checks are relaxed to accept CPU tensors.  Three
    consecutive runs of the UNMODIFIED reference FilterOptim object: the CG state must travel through the reference's own attributes
    (p, rho, r_prev as TensorLists) exactly as the reference keeps it, and a later fall-through run must continue from it."""
    from baseline import ref_env
    if not ref_env.reference_available():
        pytest.skip("reference tree not staged (baseline/_ref)")
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking import TensorList
    from pytracking.tracker.eco.optim import FilterOptim
    from pytracking.utils import TrackerParams
    from pytracking_b200 import _lib, ops, plugin

    class FakeLib:
        calls = 0

        def b200trk_eco_filter_cg(self, *a):
            FakeLib.calls += 1
            a = [C.c_float(x) if isinstance(x, float) else x for x in a[:-1]]
            return emul.eco_emul_filter_cg(*a, 3, 64, -1, None)

    monkeypatch.setattr(_lib, "lib", lambda: FakeLib())
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops, "_dev", lambda t, name: t.contiguous())
    monkeypatch.setattr(plugin, "_inference", lambda *ts: all(isinstance(t, torch.Tensor) and t.dtype == torch.float32 for t in ts))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    g, case = gold, "pr_forget"
    fr, sa, dff, pdp, prp = g[case + "/params"]
    T = lambda k: torch.from_numpy(g[k].copy())
    params = TrackerParams()
    params.fletcher_reeves, params.standard_alpha, params.direction_forget_factor, params.debug = bool(fr), bool(sa), float(dff), 0
    params.precond_data_param, params.precond_reg_param = float(pdp), float(prp)
    params.precond_learning_rate = TensorList([float(g["%s/b%d/lr" % (case, b)]) for b in range(2)])
    k0 = [case + "/run0/b%d/" % b for b in range(2)]
    filt = TensorList([T(k + "hf_in") for k in k0])
    samples, sw = TensorList([T(k + "samples") for k in k0]), TensorList([T(k + "sw") for k in k0])
    reg = TensorList([T("%s/b%d/reg_filter" % (case, b)) for b in range(2)])
    opt = FilterOptim(params, reg.view(-1) @ reg.view(-1))
    opt.register(filt, samples, TensorList([T("%s/b%d/yf" % (case, b)) for b in range(2)]), sw, reg)
    plugin.install()
    served = plugin.stats.get("FilterOptim.run", 0)
    try:
        for run in range(3):
            ks = ["%s/run%d/b%d/" % (case, run, b) for b in range(2)]
            for b, k in enumerate(ks):                            # ECO.update_memory between the runs
                samples[b].copy_(T(k + "samples"))
                sw[b].copy_(T(k + "sw"))
            if run == 2:                                          # the last run on the reference implementation, from OUR state
                monkeypatch.setattr(plugin, "_inference", lambda *ts: False)
            opt.run(int(g[ks[0] + "num_iter"]), TensorList([T(k + "new_xf") for k in ks]))
            for b, k in enumerate(ks):
                assert _rel(filt[b].numpy(), g[k + "hf_out"]) < 5e-5, (run, b)
                assert _rel(opt.p[b].numpy(), g[k + "p_out"]) < 5e-5, (run, b)
                assert _rel(opt.r_prev[b].numpy(), g[k + "r_prev_out"]) < 5e-5, (run, b)
                assert _rel(opt.sample_energy[b].numpy(), g[k + "energy_out"]) < 1e-5
                assert abs(float(opt.rho[b]) - float(g[k + "rho_out"])) < 5e-5 * abs(float(g[k + "rho_out"]))
            for hf in filt:
                hf[:, :, :, 0, :] /= 2
        assert FakeLib.calls == 4 and plugin.stats.get("FilterOptim.run") == served + 2      # two blocks x two runs through the library
    finally:
        plugin.uninstall()


# ---- first-frame joint optimisation (FactorizedConvProblem + GaussNewtonCG, eco/optim.py:8-117) ---------------------------------------
JOINT_GOLD = os.path.join(ROOT, "tests", "golden", "eco_joint.npz")


@pytest.fixture(scope="module")
def jgold():
    return np.load(JOINT_GOLD)


@pytest.mark.parametrize("bi", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_joint_oracle_matches_reference_autograd(jgold, bi, dtype):
    """The explicit J / J^T of oracle/eco_oracle.py against the reference's GaussNewtonCG, which differentiates the residuals twice."""
    g, k = jgold, "b%d/" % bi
    T = lambda key: torch.from_numpy(g[key]).to(dtype)
    num_cg, num_gn, lam, pdp, prp, ppp = g["params"]
    hf, P, se = E.joint_gn_run(T(k + "hf_in"), T(k + "P_in"), T(k + "samples"), T(k + "yf"), T(k + "sample_weights"), T(k + "reg_filter"),
                               int(num_cg), int(num_gn), float(lam), float(pdp), float(prp), float(ppp))
    assert _rel(hf, g[k + "hf_out"]) < 5e-6 and _rel(P, g[k + "P_out"]) < 5e-6 and _rel(se, g[k + "sample_energy"]) < 2e-6
    dMh, dMP, _ = E.joint_precond(T(k + "samples"), T(k + "P_in"), T(k + "yf"), T(k + "reg_filter"), float(pdp), float(prp), float(ppp), float(lam))
    assert _rel(dMh, g[k + "diag_M_filter"]) < 2e-6 and abs(float(dMP) - float(g[k + "diag_M_proj"])) < 2e-6 * float(g[k + "diag_M_proj"])


JOINT_DECOMPOSITIONS = [(3, 64, -1), (1, 64, -1), (5, 64, 0), (45, 64, -1), (10, 256, 1), (7, 256, 2), (2, 32, -1)]


@pytest.mark.parametrize("max_ctas,block,force_res", JOINT_DECOMPOSITIONS)
def test_emulated_joint_kernel_matches_reference(emul, jgold, max_ctas, block, force_res):
    """csrc/eco_joint_kernel.cuh on the CPU: 3 GN x 4 CG iterations on both blocks; covers one CTA for everything, a CTA per coefficient,
    resident / streamed slabs, 1-16 coefficient splits per projection-gradient element and several tiles per CTA."""
    for bi in range(2):
        err, plan, _ = _run_emulated_joint(emul, jgold, bi, max_ctas, block, force_res)
        assert err < 5e-6, (bi, err, plan)


def test_emulated_joint_kernel_is_deterministic(emul, jgold):
    a = _run_emulated_joint(emul, jgold, 1, 28, 64, -1)[2]
    b = _run_emulated_joint(emul, jgold, 1, 28, 64, -1)[2]
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_emulated_joint_kernel_under_thread_sanitizer(jgold, tmp_path):
    tsan_rt = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(tsan_rt) or not os.path.exists(tsan_rt):
        pytest.skip("no ThreadSanitizer runtime")
    lib = _build(str(tmp_path), tsan=True)
    script = (
        "import sys, numpy as np, ctypes as C\n"
        "sys.path.insert(0, %r)\n"
        "from eco_emul_driver import run_emulated_joint\n"
        "g = np.load(%r)\n"
        "lib = C.CDLL(%r)\n"
        "for ctas, blk, fres in ((3, 64, 1), (28, 64, -1)):\n"
        "    for bi in range(2):\n"
        "        e, plan, _ = run_emulated_joint(lib, g, bi, ctas, blk, fres)\n"
        "        assert e < 5e-6, (e, plan)\n"
        "print('EMUL_DONE')\n" % (os.path.join(ROOT, "tests", "cpu_emul"), JOINT_GOLD, lib))
    env = dict(os.environ, LD_PRELOAD=tsan_rt, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0")
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, timeout=900, cwd=ROOT)
    if "EMUL_DONE" not in r.stdout and "ThreadSanitizer" not in r.stderr:
        pytest.skip("ThreadSanitizer could not run here: %s" % r.stderr[-300:])
    assert "EMUL_DONE" in r.stdout, r.stderr[-2000:]
    assert "data race" not in r.stderr, r.stderr[:4000]


def test_joint_seam_over_the_emulated_kernel(emul, jgold, monkeypatch):
    """plugin.install()'s GaussNewtonCG.run on the UNMODIFIED reference FactorizedConvProblem (two blocks, the tracker's permuted sample
    view, one-element sample weights) with the emulated kernel behind the library's entry point: same result as the reference's own
    autograd run recorded in the golden file; ATOM's problem of the same class name is not affected."""
    from baseline import ref_env
    if not ref_env.reference_available():
        pytest.skip("reference tree not staged (baseline/_ref)")
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking import TensorList
    from pytracking.libs.optimization import GaussNewtonCG
    from pytracking.tracker.eco.optim import FactorizedConvProblem
    from pytracking.utils import TrackerParams
    from pytracking_b200 import _lib, ops, plugin

    class FakeLib:
        calls = 0

        def b200trk_eco_joint_gn(self, *a):
            FakeLib.calls += 1
            a = [C.c_float(x) if isinstance(x, float) else x for x in a[:-1]]
            return emul.eco_emul_joint_gn(*a, 3, 64, -1, None)

    monkeypatch.setattr(_lib, "lib", lambda: FakeLib())
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops, "_dev", lambda t, name: t.contiguous())
    monkeypatch.setattr(plugin, "_inference", lambda *ts: all(isinstance(t, torch.Tensor) and t.dtype == torch.float32 for t in ts))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    g = jgold
    num_cg, num_gn, lam, pdp, prp, ppp = g["params"]
    params = TrackerParams()
    params.precond_data_param, params.precond_reg_param, params.precond_proj_param, params.projection_reg = float(pdp), float(prp), float(ppp), float(lam)
    T = lambda k: torch.from_numpy(g[k].copy())
    # eco.py:133: the problem gets a permuted VIEW of [N,Cin,H,Wh,2]
    X = TensorList([T("b%d/samples" % b).permute(2, 3, 0, 1, 4).contiguous().permute(2, 3, 0, 1, 4) for b in range(2)])
    hf = TensorList([T("b%d/hf_in" % b) for b in range(2)])
    P = TensorList([T("b%d/P_in" % b) for b in range(2)])
    n = X[0].shape[2]
    prob = FactorizedConvProblem(X, TensorList([T("b%d/yf" % b) for b in range(2)]), TensorList([T("b%d/reg_filter" % b) for b in range(2)]),
                                 P, params, TensorList([torch.ones(1) / n for _ in range(2)]))
    var = hf.concat(P)
    opt = GaussNewtonCG(prob, var, debug=False)
    plugin.install()
    served = plugin.stats.get("GaussNewtonCG.run[eco]", 0)
    try:
        opt.run(int(num_cg), int(num_gn))
    finally:
        plugin.uninstall()
    assert FakeLib.calls == 2 and plugin.stats.get("GaussNewtonCG.run[eco]", 0) == served + 1
    for b in range(2):
        assert _rel(var[b].numpy(), g["b%d/hf_out" % b]) < 5e-6 and _rel(var[2 + b].numpy(), g["b%d/P_out" % b]) < 5e-6
        assert var[b] is hf[b] and not var[b].requires_grad              # updated in place, detached as the reference leaves it


def test_joint_launch_plan_at_eco_block_sizes(emul):
    """ECO default first frame: 30 augmented samples; deep block 256 -> 64 channels on ~15x8 coefficients, shallow 96 -> 16 on ~63x32."""
    # the shared-memory arithmetic of eco_joint_plan, through the Python mirror the plug-in guard uses (pytracking_b200/eco_plan.py)
    from pytracking_b200 import eco_plan
    for n, cin, c in ((30, 256, 64), (30, 96, 16), (30, 512, 128)):
        fixed = 4 * eco_plan.ecoj_fixed_smem_floats(n, cin, c)
        assert eco_plan.eco_joint_fits(n, cin, c)
        slab = n * (cin + 1) * 8
        assert fixed <= 226 * 1024
        assert (227 * 1024 - 1024 - fixed) // slab >= 1                # at least one coefficient's slab resident per CTA


# The WHOLE launch of an H100 (132 CTAs x 256 threads) at ECO's default sizes runs in tests/test_eco_gpu_file_on_cpu.py: the `-m gpu` test file
# itself against the launchers' host code and these kernel sources.


def test_eco_kernels_under_address_sanitizer(tmp_path):
    """No access outside the launch's dynamic shared memory or a global buffer, at real per-CTA sizes and at ragged ones."""
    rt = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if shutil.which("g++") is None or not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no AddressSanitizer runtime")
    lib = str(tmp_path / "libeco_emul_asan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-fno-gnu-unique", "-Wno-unknown-pragmas", "-fsanitize=address",
                    os.path.join(ROOT, "tests", "cpu_emul", "eco_emul.cpp"), "-o", lib], check=True, capture_output=True)
    env = dict(os.environ, LD_PRELOAD=rt, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpu_emul", "eco_asan_sweep.py"), lib], capture_output=True, text=True, env=env,
                       timeout=900)
    if "EMUL_DONE" not in r.stdout and "AddressSanitizer" not in r.stderr:
        pytest.skip("AddressSanitizer could not run here: %s" % r.stderr[-300:])
    assert "AddressSanitizer" not in r.stderr, r.stderr[:4000]
    assert "EMUL_DONE" in r.stdout, r.stderr[-2000:]
