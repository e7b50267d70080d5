"""CPU tier of the learnt filter initialiser (FilterInitializerLinear, csrc/init_heads_kernels.cuh + prroi_kernels.cuh's forward):
  * the float64 restatement oracle/filter_init_oracle.py against tests/golden/filter_init.npz (the reference's own module, recorded by
    oracle/gen_filter_init_golden.py);
  * the kernel sources, built as host code under tests/cpu_emul/cuda_shim.h with the launch shapes of csrc/init_heads.cu, on the
    golden's cases from filter_conv's float64 output: within 1e-5 relative of the golden;
  * the same kernels under ThreadSanitizer (one OS thread per CUDA thread): no data race."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "filter_init.npz")
SRC = os.path.join(ROOT, "tests", "cpu_emul", "init_heads_emul.cpp")
PREFIX = "classifier.filter_initializer."


def golden_cases():
    """[(seed, S, H, filter_norm, pool_square, boxes [S,4], reference filter [1,512,4,4])] of the golden."""
    d = np.load(GOLDEN)
    out = []
    for i in range(int(d["num_cases"])):
        seed, S, H, norm, square = [int(v) for v in d["case_%d_meta" % i]]
        out.append((seed, S, H, norm, square, d["case_%d_boxes" % i], d["case_%d_filter" % i]))
    return out


def filter_conv_weights():
    from pytracking_b200 import synth
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    return sd[PREFIX + "filter_conv.weight"].float(), sd[PREFIX + "filter_conv.bias"].float()


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _build(out, flags=()):
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique",
                    "-Wno-unknown-pragmas"] + list(flags) + [SRC, "-o", out], check=True, capture_output=True)
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return C.CDLL(_build(os.path.join(str(tmp_path_factory.mktemp("init_heads_emul")), "libinit_heads_emul.so")))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_float64_restatement_matches_reference_golden():
    from oracle import filter_init_oracle as O
    from pytracking_b200 import synth
    w, b = filter_conv_weights()
    worst = 0.0
    for seed, S, H, norm, square, boxes, ref in golden_cases():
        feat = synth.make_clf_features(seed, S, 512, H, H)
        e = rel(O.filter_init(w, b, feat, boxes, filter_norm=norm, pool_square=square), ref)
        assert e <= 1e-5, (seed, S, H, norm, square, e)
        worst = max(worst, e)
    print("float64 restatement vs reference: worst relative difference %.2e" % worst)


def test_kernel_sources_match_reference_golden(emul):
    from pytracking_b200 import synth
    w, b = filter_conv_weights()
    for seed, S, H, norm, square, boxes, ref in golden_cases():
        feat = synth.make_clf_features(seed, S, 512, H, H)
        conv = np.ascontiguousarray(F.conv2d(feat.double(), w.double(), b.double(), padding=1).float().numpy())
        out = np.full((512, 4, 4), np.nan, np.float32)
        img = np.arange(S, dtype=np.int32)
        bx = np.ascontiguousarray(boxes, dtype=np.float32)
        assert emul.fi_emul_pool(_p(conv), S, 512, H, H, S, _p(img), _p(bx), 4, norm, square, _p(out)) == 0
        assert rel(out[None], ref) <= 1e-5, (seed, S, H, norm, square, rel(out[None], ref))


def test_nchw_import_kernel_source_is_a_transpose(emul):
    x = np.ascontiguousarray(np.random.RandomState(0).randn(3, 70, 22 * 22).astype(np.float32))
    y = np.full((3, 22 * 22, 70), np.nan, np.float32)
    assert emul.fi_emul_nchw_to_nhwc(_p(x), _p(y), 3, 22 * 22, 70) == 0
    assert np.array_equal(y, x.transpose(0, 2, 1))


_SWEEP = r"""
import ctypes as C, sys
import numpy as np
L = C.CDLL(sys.argv[1])
P = lambda a: a.ctypes.data_as(C.c_void_p)
rng = np.random.RandomState(0)
x, y = np.ascontiguousarray(rng.randn(2, 40, 81).astype(np.float32)), np.zeros((2, 81, 40), np.float32)
L.fi_emul_nchw_to_nhwc(P(x), P(y), 2, 81, 40)
conv = np.ascontiguousarray(rng.randn(3, 16, 9, 9).astype(np.float32))
boxes = np.array([[10, 12, 60, 40], [-5, 30, 50, 90], [100, 3, 2.5, 70]], np.float32)
img, out = np.array([2, 0, 1], np.int32), np.zeros((16, 4, 4), np.float32)
L.fi_emul_pool(P(conv), 3, 16, 9, 9, 3, P(img), P(boxes), 4, 1, 1, P(out))
print("EMUL_DONE")
"""


def test_kernel_sources_under_thread_sanitizer(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    rt = subprocess.run(["g++", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no ThreadSanitizer runtime")
    lib = _build(str(tmp_path / "libfilter_init_tsan.so"), ["-fsanitize=thread,alignment", "-Wno-tsan"])
    env = dict(os.environ, LD_PRELOAD=rt, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 exitcode=0", B200_EMUL_THREADS="1")
    r = subprocess.run([sys.executable, "-c", _SWEEP, lib], capture_output=True, text=True, env=env, timeout=600)
    if "EMUL_DONE" not in r.stdout and "ThreadSanitizer" not in r.stderr:
        pytest.skip("ThreadSanitizer could not run here: %s" % r.stderr[-300:])
    assert "EMUL_DONE" in r.stdout, r.stderr[-2000:]
    assert "data race" not in r.stderr, r.stderr[:4000]
    assert "runtime error" not in r.stderr, r.stderr[:4000]
