"""The fp32 CUDA-core kernels of stage 1 (csrc/conv_fp32_kernels.cuh, SURVEY 8 rows S1.1 / S1.2): `NetWithBackbone.preprocess_image`, the
7x7 stem + folded BN + ReLU, max-pool 3x3/2, the generic implicit-GEMM convolution with the fused (bias + residual + ReLU) epilogue and the
deterministic split-K path (the engine's exact-fp32 `precision=1` path), NHWC -> NCHW export and `InstanceL2Norm` -- executed ON THE CPU: the
same source file the CUDA build compiles (per-function `cuobjdump -sass` identical before and after the kernels moved into the header),
built as host code under tests/cpu_emul/cuda_shim.h with the launch arithmetic of csrc/conv_fp32.cu, against plain PyTorch (float64).
With tests/test_dimp_kernels_cpu.py and tests/test_corr_kernels_cpu.py every kernel of a tracked DiMP frame except the two wgmma ones
(`conv_tc_kernel`, `sd_tc_kernel`) also runs in the CPU tier."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp("c32_emul")), "libc32_emul.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", "conv_fp32_emul.cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _nhwc(t):
    return np.ascontiguousarray(t.permute(0, 2, 3, 1).numpy())


def test_preprocess_stem_maxpool_kernel_sources(emul):
    """uint8-range crop -> (x/255 - mean)/std in NHWC4 -> conv 7x7/2 + bias + ReLU -> max-pool 3x3/2 (resnet.py:182-186), odd sizes."""
    g = torch.Generator().manual_seed(0)
    S, H, W = 2, 37, 50
    crop = torch.rand(S, 3, H, W, generator=g) * 255
    pre = np.full((S, H, W, 4), np.nan, np.float32)
    assert emul.c32_emul_preprocess(_p(np.ascontiguousarray(crop.numpy())), _p(pre), S, H, W) == 0
    mean, std = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1), torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    ref = (crop / 255 - mean) / std                                   # net_wrappers.py:55-69, same operation order
    assert np.array_equal(pre[..., :3], _nhwc(ref)) and not pre[..., 3].any()
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    b = torch.randn(64, generator=g) * 0.1
    wt = np.ascontiguousarray(w.permute(2, 3, 1, 0).reshape(49, 3, 64).numpy())      # [tap][cin][cout]
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    stem = np.full((S, Ho, Wo, 64), np.nan, np.float32)
    assert emul.c32_emul_stem(_p(pre), _p(wt), _p(b.numpy()), _p(stem), S, H, W) == 0
    stem_ref = torch.relu(F.conv2d(ref.double(), w.double(), b.double(), stride=2, padding=3))
    assert _rel(stem, _nhwc(stem_ref)) < 2e-6
    Hp, Wp = (Ho - 1) // 2 + 1, (Wo - 1) // 2 + 1
    pool = np.full((S, Hp, Wp, 64), np.nan, np.float32)
    assert emul.c32_emul_maxpool(_p(stem), _p(pool), S, Ho, Wo, 64) == 0
    pool_ref = F.max_pool2d(torch.from_numpy(stem).permute(0, 3, 1, 2), 3, 2, 1)
    assert np.array_equal(pool, _nhwc(pool_ref))


@pytest.mark.parametrize("S,Hin,Cin,Cout,k,stride,pad,bias,res,relu,sms", [
    (1, 12, 64, 64, 3, 1, 1, True, True, 1, 1),          # basic-block second conv: bias + residual + ReLU fused, one K split
    (2, 9, 128, 128, 1, 1, 0, True, False, 0, 148),      # 1x1, few CTAs on many SMs: split-K + separate epilogue
    (1, 13, 48, 20, 3, 2, 1, True, False, 1, 148),       # stride 2, partial tiles in M and N, split-K
    (1, 7, 16, 8, 3, 1, 1, False, False, 0, 0),          # no bias, fused path
])
def test_conv_igemm_kernel_source(emul, S, Hin, Cin, Cout, k, stride, pad, bias, res, relu, sms):
    g = torch.Generator().manual_seed(Cin + Cout)
    x = torch.randn(S, Cin, Hin, Hin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) if bias else None
    ref = F.conv2d(x.double(), w.double(), b.double() if bias else None, stride=stride, padding=pad)
    r = torch.randn(ref.shape, generator=g) if res else None
    if res:
        ref = ref + r.double()
    if relu:
        ref = torch.relu(ref)
    wk = np.ascontiguousarray(w.permute(0, 2, 3, 1).numpy())                      # [cout][kh][kw][cin]
    out = np.full(tuple(_nhwc(ref).shape), np.nan, np.float32)
    splits = C.c_int(0)
    rc = emul.c32_emul_conv(_p(_nhwc(x)), _p(wk), _p(out), S, Hin, Hin, Cin, Cout, k, stride, pad, _p(b.numpy()) if bias else None,
                            _p(_nhwc(r)) if res else None, relu, sms, C.byref(splits))
    assert rc == 0
    assert _rel(out, _nhwc(ref)) < 2e-6, splits.value
    assert (splits.value > 1) == (sms == 148)                      # both the fused and the split-K path are exercised


def test_export_and_instance_l2norm_kernel_sources(emul):
    """NHWC -> NCHW, and InstanceL2Norm (ltr/models/layers/normalization.py:15-20): x * scale * sqrt(C*H*W / (sum x^2 + eps))."""
    g = torch.Generator().manual_seed(3)
    for (S, C_, H) in ((2, 40, 7), (1, 512, 18)):
        x = torch.randn(S, C_, H, H, generator=g)
        out = np.full((S, C_, H, H), np.nan, np.float32)
        assert emul.c32_emul_export(_p(_nhwc(x)), _p(out), S, H * H, C_, 0, C.c_float(1.0), C.c_float(0.0)) == 0
        assert np.array_equal(out, x.numpy())
        scale, eps = 0.05, 1e-5
        assert emul.c32_emul_export(_p(_nhwc(x)), _p(out), S, H * H, C_, 1, C.c_float(scale), C.c_float(eps)) == 0
        xd = x.double()
        ref = xd * (scale * ((C_ * H * H) / ((xd * xd).reshape(S, -1).sum(1).view(S, 1, 1, 1) + eps)).sqrt())
        assert _rel(out, ref.numpy()) < 2e-6
