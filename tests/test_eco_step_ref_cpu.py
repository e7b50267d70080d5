"""CPU tier of tests/test_eco_steps_f64_gpu.py: pins tests/eco_step_ref.py, then runs the GPU file itself on the kernels' sources.

  * the helper's float64 steps reproduce the reference FilterOptim / GaussNewtonCG goldens (tests/golden/eco_cg.npz, eco_joint.npz)
    within their float32 spread, and the oracle really computes in float64: runs in other channel and sample orders agree to 1e-12;
  * `eco_plan` / `eco_joint_plan` (pytracking_b200/eco_plan.py) reproduce the kernels' own plan functions at 132, 114 and 148 SMs;
  * tests/test_eco_steps_f64_gpu.py runs in a subprocess with tests/cpu_emul/gpu_file_on_cpu_plugin.py -- the launchers and kernel
    sources built as host code, whole cooperative grids -- on its small cases at 132 and 114 SMs (every case and the score path with
    B200_ECO_STEPS_ON_CPU=1, which takes far longer)."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import eco_step_ref as R
from oracle import eco_oracle as E
from pytracking_b200.eco_plan import eco_joint_plan, eco_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FULL = os.environ.get("B200_ECO_STEPS_ON_CPU") == "1"


def _gold(name):
    return np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))


def _golden_call(g, case, run, bi):
    fr, sa, dff, pdp, prp = g[case + "/params"]
    k = "%s/run%d/b%d/" % (case, run, bi)
    T = lambda key: torch.from_numpy(np.ascontiguousarray(g[key]))
    state = None
    if int(g[k + "has_state"]):
        state = {"p": T(k + "p_in"), "r_prev": T(k + "r_prev_in") if (k + "r_prev_in") in g else None,
                 "rho": torch.tensor([float(g[k + "rho_in"])], dtype=torch.float32)}
    prob = R.FilterProblem(T(k + "samples"), T("%s/b%d/yf" % (case, bi)), T(k + "sw"), T("%s/b%d/reg_filter" % (case, bi)), bool(fr), bool(sa),
                           float(dff), float(g["%s/b%d/lr" % (case, bi)]), float(pdp), float(prp))
    en = T(k + "energy_in") if int(g[k + "has_energy"]) else None
    return prob, T(k + "hf_in"), en, state, int(g[k + "num_iter"]), T(k + "new_xf"), k


@pytest.mark.parametrize("case,run,bi", [(c, r, b) for c in ("pr_forget", "fr_reset") for r in range(3) for b in range(2)])
def test_helper_float64_steps_match_reference_goldens(case, run, bi):
    g = _gold("eco_cg")
    prob, hf, en, state, k, nx, key = _golden_call(g, case, run, bi)
    ref = prob.step(hf, en, state, k, nx)
    r32 = prob.run(hf, en, state, k, nx, torch.float32)
    gold = torch.from_numpy(g[key + "hf_out"]).double() - hf.double()
    spread = R.rel_err(r32["hf"].double() - hf.double(), ref["d"])
    assert R.rel_err(gold, ref["d"]) <= max(20 * spread, 1e-6), (R.rel_err(gold, ref["d"]), spread)
    assert R.rel_err(torch.from_numpy(g[key + "p_out"]), ref["p"]) <= max(20 * R.rel_err(r32["p"], ref["p"]), 1e-6)
    assert R.rel_err(float(g[key + "rho_out"]), float(ref["rho"])) <= max(20 * R.rel_err(float(r32["rho"]), float(ref["rho"])), 1e-6)
    assert float(((torch.from_numpy(g[key + "energy_out"]).double() - ref["energy"]).abs() / ref["energy"]).max()) <= 8 * R.U


@pytest.mark.parametrize("bi", [0, 1])
def test_helper_float64_joint_steps_match_reference_golden(bi):
    g, k = _gold("eco_joint"), "b%d/" % bi
    T = lambda key: torch.from_numpy(np.ascontiguousarray(g[key]))
    num_cg, num_gn, lam = int(g["params"][0]), int(g["params"][1]), float(g["params"][2])
    hf = T(k + "hf_in")
    dMh = T(k + "diag_M_filter").reshape(1, *hf.shape[1:4])
    prob = R.JointProblem(T(k + "samples"), T(k + "yf"), T(k + "sample_weights").sqrt(), T(k + "reg_filter"), dMh, float(g[k + "diag_M_proj"]), lam)
    h64, P64 = prob.run(hf, T(k + "P_in"), num_cg, num_gn)
    h32, P32 = prob.run(hf, T(k + "P_in"), num_cg, num_gn, torch.float32)
    for out, o32, ref in ((h64, h32, T(k + "hf_out")), (P64, P32, T(k + "P_out"))):
        spread = R.rel_err(o32, out)
        assert R.rel_err(ref, out) <= max(20 * spread, 1e-6), (R.rel_err(ref, out), spread)


def test_oracle_computes_in_float64():
    """A float64 run agrees with runs in other channel and sample orders to 1e-12: nothing inside rounds to float32 (which would show as
    ~1e-7).  Covers the carried state under Polak-Ribiere with a forget factor, the energy update, and the joint GN step."""
    g = torch.Generator().manual_seed(5)
    h, wh, n, c = 9, 5, 12, 16
    samples = torch.randn(h, wh, n, c, 2, generator=g)
    sw = torch.rand(n, generator=g) + 0.1
    yf = torch.rand(1, 1, h, wh, generator=g)
    reg = torch.rand(1, 1, 3, 3, generator=g) * 0.2
    prob = R.FilterProblem(samples, yf, sw / sw.sum(), reg, False, True, 0.7)
    hf = 0.01 * torch.randn(1, c, h, wh, 2, generator=g)
    nx = torch.randn(1, c, h, wh, 2, generator=g)
    en = torch.rand(1, c, h, wh, generator=g) + 0.1
    st = {"p": torch.randn(1, c, h, wh, 2, generator=g), "r_prev": torch.randn(1, c, h, wh, 2, generator=g), "rho": torch.tensor([3.0])}
    ref = prob.run(hf, en, st, 4, nx)
    for seed in (0, 1):
        gp = torch.Generator().manual_seed(seed)
        alt = prob.run(hf, en, st, 4, nx, torch.float64, (torch.randperm(c, generator=gp), torch.randperm(n, generator=gp)))
        for key in ("hf", "p", "r_prev", "energy"):
            assert R.rel_err(alt[key], ref[key]) < 1e-12, (key, R.rel_err(alt[key], ref[key]))
        assert R.rel_err(float(alt["rho"]), float(ref["rho"])) < 1e-12
    cin = 24
    X = torch.randn(h, wh, n, cin, 2, generator=g)
    P = torch.linalg.qr(torch.randn(cin, cin, generator=g))[0][:, :c].contiguous()
    dMh, dMP, _ = E.joint_precond(X, P, yf, reg, 0.3, 0.15, 35.0, 5e-8)
    jp = R.JointProblem(X, yf, torch.full((n,), n ** -0.5), reg, dMh.reshape(1, c, h, wh), float(dMP), 5e-8)
    h1, P1 = jp.run(hf, P, 5, 2)
    gp = torch.Generator().manual_seed(2)
    h2, P2 = jp.run(hf, P, 5, 2, torch.float64, (torch.randperm(c, generator=gp), torch.randperm(cin, generator=gp), torch.randperm(n, generator=gp)))
    assert R.rel_err(h2, h1) < 1e-12 and R.rel_err(P2, P1) < 1e-12


# ---- the plan mirrors ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("eco_emul_plan")), "libeco_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", "eco_emul.cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


CG_SHAPES = [(15, 8, 200, 64), (63, 32, 200, 16), (17, 9, 200, 32), (31, 16, 250, 128), (5, 3, 40, 16), (11, 6, 500, 64), (23, 12, 120, 32),
             (9, 5, 6, 16), (13, 7, 50, 128), (200, 101, 4000, 128)]
JOINT_SHAPES = [(63, 32, 30, 96, 16), (15, 8, 30, 256, 64), (15, 8, 30, 512, 128), (15, 8, 200, 256, 64), (5, 3, 20, 64, 16), (9, 5, 6, 32, 16)]


@pytest.mark.parametrize("sms", [132, 114, 148])
def test_plan_mirrors_reproduce_the_kernels(emul, sms):
    out = (C.c_longlong * 8)()
    for h, wh, n, c in CG_SHAPES:
        for it in (1, 5, 40):
            emul.eco_emul_plan(h, wh, n, c, it, sms, 256, out)
            p = eco_plan(h, wh, n, c, it, sms)
            assert list(out) == [p["grid"], p["G"], p["CPL"], p["GPP"], p["res_slabs"], p["npx_max"], p["smem_bytes"], p["ws_bytes"]], (h, wh, n, c, sms)
    # the joint plan as the emulated launch reports it (grid, res_slabs, npx_max, EPB, SPL, smem bytes), on the shapes whose whole launch
    # is quick on the CPU
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    for h, wh, n, cin, c in [s for s in JOINT_SHAPES if s[0] * s[1] <= 45]:
        X = torch.randn(h, wh, n, cin, 2, generator=torch.Generator().manual_seed(h + cin)).numpy()
        hf, P = np.zeros((1, c, h, wh, 2), np.float32), np.zeros((cin, c), np.float32)
        yf, sws, rf, dmh = np.ones((h, wh), np.float32), np.ones(n, np.float32), np.ones((1, 1, 1, 1), np.float32), np.ones((1, c, h, wh), np.float32)
        plan = (C.c_int * 6)()
        assert emul.eco_emul_joint_gn(ptr(hf), ptr(P), ptr(X), ptr(yf), ptr(sws), ptr(rf), 1, 1, ptr(dmh), C.c_float(1.0), C.c_float(1e-3),
                                      h, wh, n, cin, c, 1, 1, sms, 256, -1, plan) == 0
        p = eco_joint_plan(h, wh, n, cin, c, 1, 1, sms)
        assert list(plan) == [p["grid"], p["res_slabs"], p["npx_max"], p["EPB"], p["SPL"], p["smem_bytes"]], (h, wh, n, cin, c, sms)
    for h, wh, n, cin, c in JOINT_SHAPES:
        p = eco_joint_plan(h, wh, n, cin, c, 1, 1, sms)
        assert p["smem_bytes"] <= 227 * 1024 and p["EPB"] * p["SPL"] <= 256


def test_plan_features_are_reachable_on_other_sm_counts():
    for sms in (132, 114):
        reached = set()
        for h, wh, n, c in CG_SHAPES[:7]:
            reached |= R.plan_features(h, wh, n, c, sms)
        assert set(R.PLAN_FEATURES) <= reached, (sms, sorted(set(R.PLAN_FEATURES) - reached))
        reached = set()
        for s in JOINT_SHAPES[:5]:
            reached |= R.joint_plan_features(*s, sms)
        assert set(R.JOINT_PLAN_FEATURES) <= reached, (sms, sorted(set(R.JOINT_PLAN_FEATURES) - reached))


# ---- the GPU file on the kernel sources ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def abi_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    lib = os.path.join(str(tmp_path_factory.mktemp("eco_abi")), "libeco_abi_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-pthread", "-shared", "-fPIC", "-fno-gnu-unique", "-ffp-contract=off", "-Wno-unknown-pragmas",
                    "-DB200_EMUL_COOP_FIBERS", "-x", "c++", os.path.join(ROOT, "tests", "cpu_emul", "eco_abi_emul.cpp"), "-o", lib],
                   check=True, capture_output=True)
    return lib


SMALL = "5x3 or 23x12 or score"


@pytest.mark.parametrize("sms", ["132", "114"])
def test_steps_gpu_file_runs_on_the_kernel_sources(abi_lib, sms):
    env = dict(os.environ, B200_ECO_ABI_EMUL=abi_lib, B200_EMUL_SMS=sms,
               PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "tests", "cpu_emul"), os.path.join(ROOT, "tests"), ROOT, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_eco_steps_f64_gpu.py"), "-p", "gpu_file_on_cpu_plugin", "-q",
                        "-p", "no:cacheprovider", "-s", "-rs"] + ([] if FULL else ["-k", SMALL]),
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=3000)
    tail = r.stdout[-4000:] + r.stderr[-1500:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
    for line in r.stdout.split("\n"):
        if line.startswith("eco f64"):
            print(sms, "SMs:", line)
