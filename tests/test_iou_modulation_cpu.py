"""CPU tier of get_modulation's linear blocks (mod_linear_kernel of csrc/init_heads_kernels.cuh, built as host code under
tests/cpu_emul/cuda_shim.h with the launch shape of csrc/init_heads.cu): fc3_1r (1152 -> 256) and fc34_*r (256 + 256 -> 256) with ReLU
against float64 on seeded operands, boxes independent of each other bit for bit, and no data race under ThreadSanitizer."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from test_filter_init_cpu import _build, _p


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return C.CDLL(_build(os.path.join(str(tmp_path_factory.mktemp("mod_emul")), "libinit_heads_emul.so")))


def _linear(emul, xa, xb, W, b):
    R, D = xa.shape[0], W.shape[0]
    Kb = 0 if xb is None else xb.shape[1]
    out = np.full((R, D), np.nan, np.float32)
    assert emul.mod_emul_linear(_p(xa), xa.shape[1], None if xb is None else _p(xb), Kb, _p(W), _p(b), _p(out), D, R, D) == 0
    return out


@pytest.mark.parametrize("Ka,Kb,R", [(1152, 0, 1), (1152, 0, 5), (256, 256, 3)])
def test_linear_block_kernel_source_against_float64(emul, Ka, Kb, R):
    rng = np.random.RandomState(Ka + Kb + R)
    D = 256
    xa = np.ascontiguousarray(rng.randn(R, Ka).astype(np.float32))
    xb = np.ascontiguousarray(rng.randn(R, Kb).astype(np.float32)) if Kb else None
    W = np.ascontiguousarray(((rng.rand(D, Ka + Kb) * 2 - 1) / np.sqrt(Ka + Kb)).astype(np.float32))
    b = np.ascontiguousarray(0.05 * rng.randn(D).astype(np.float32))
    out = _linear(emul, xa, xb, W, b)
    x = xa.astype(np.float64) if xb is None else np.concatenate([xa, xb], 1).astype(np.float64)
    z = x @ W.astype(np.float64).T + b
    m = np.abs(x) @ np.abs(W.astype(np.float64)).T + np.abs(b)
    ref = np.maximum(z, 0)
    assert float((np.abs(out - ref) / m).max()) <= (Ka + Kb + 2) * 2.0 ** -23
    for r in range(R):         # a box's vector depends on that box only
        one = _linear(emul, np.ascontiguousarray(xa[r:r + 1]), None if xb is None else np.ascontiguousarray(xb[r:r + 1]), W, b)
        assert np.array_equal(one[0], out[r])


_SWEEP = r"""
import ctypes as C, sys
import numpy as np
L = C.CDLL(sys.argv[1])
P = lambda a: a.ctypes.data_as(C.c_void_p)
rng = np.random.RandomState(0)
xa, xb = rng.randn(3, 40).astype(np.float32), rng.randn(3, 24).astype(np.float32)
W, b, out = rng.randn(70, 64).astype(np.float32), rng.randn(70).astype(np.float32), np.zeros((3, 70), np.float32)
L.mod_emul_linear(P(xa), 40, P(xb), 24, P(W), P(b), P(out), 70, 3, 70)
print("EMUL_DONE")
"""


def test_linear_block_kernel_source_under_thread_sanitizer(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    rt = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no ThreadSanitizer runtime")
    lib = _build(str(tmp_path / "libmod_tsan.so"), ["-fsanitize=thread,alignment", "-Wno-tsan"])
    env = dict(os.environ, LD_PRELOAD=rt, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0", B200_EMUL_THREADS="1")
    r = subprocess.run([sys.executable, "-c", _SWEEP, lib], capture_output=True, text=True, env=env, timeout=600)
    if "EMUL_DONE" not in r.stdout and "ThreadSanitizer" not in r.stderr:
        pytest.skip("ThreadSanitizer could not run here: %s" % r.stderr[-300:])
    assert "EMUL_DONE" in r.stdout, r.stderr[-2000:]
    assert "data race" not in r.stderr, r.stderr[:4000]
    assert "runtime error" not in r.stderr, r.stderr[:4000]
