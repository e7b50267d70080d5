"""CPU: pins tests/tomp_step_ref.py, the float64 reference and error bounds the ToMP head's device checks use
(tests/test_tomp_steps_f64_gpu.py).

* Composed launch by launch in `launch_plan` order, the step functions reproduce oracle/tomp_oracle.transformer_forward (float64 both)
  and the reference module's outputs recorded in tests/golden/transformer.npz; the token and tower steps reproduce the reference
  FilterPredictor tokens and DenseBoxRegressor output of tests/golden/iou_tomp_ref.npz.
* Every bound holds for the kernel sources themselves, run on the CPU under tests/cpu_emul/cuda_shim.h at the shapes of
  tests/test_transformer_kernels_cpu.py and tests/test_tomp_kernels_cpu.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import tomp_step_ref as R
from pytracking_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TRANSFORMER_CASES = {"small": (64, 2, 128, 2, 2, 40, 2, 91, True), "tomp_l72": (256, 8, 2048, 6, 6, 72, 2, 92, True),
                     "tomp_l48_nomask": (256, 8, 2048, 6, 6, 48, 1, 93, False)}


def _inputs(d, L, B, seed, use_mask):
    """The inputs of tests/test_gpu_parity.py::test_transformer_golden."""
    g = torch.Generator().manual_seed(seed + 1)
    src = torch.randn(L, B, d, generator=g)
    pos = torch.randn(L, 1, d, generator=g) * 0.5
    qe = torch.randn(1, d, generator=g)
    mask = None
    if use_mask:
        mask = torch.zeros(B, L, dtype=torch.bool)
        mask[B - 1, L // 3: L // 2] = True
    return src, pos, qe, mask


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


def test_launch_plan_matches_the_forward_pass():
    """9 launches per encoder layer, 1 memory add_pos, 13 per decoder layer, the final norm; each writes a buffer it does not read."""
    for ne, nd in ((6, 6), (1, 1), (2, 3)):
        P = R.launch_plan(ne, nd)
        assert len(P) == 9 * ne + 1 + 13 * nd + 1
        for e in P:
            assert e["out"] not in e["ins"] and e["out"] != e.get("res"), e
        assert sum(e["kind"] == "gemm" for e in P) == 5 * ne + 2 * nd


def test_composed_steps_reproduce_the_oracle():
    from oracle import tomp_oracle as T
    d, nh, ff, ne, nd, L, B, seed, _ = TRANSFORMER_CASES["small"]
    sd = {k: v.double() for k, v in synth.make_transformer_state_dict(seed, d, nh, ff, ne, nd).items()}
    src, pos, qe, mask = _inputs(d, L, B, seed, True)
    for m in (mask, None):
        hs, mem = R.compose(sd, src.double(), pos.double(), m, qe.double(), nh, ne, nd)
        with torch.no_grad():
            hs_o, mem_o = T.transformer_forward(sd, src.double(), m, qe.double(), pos.double(), nh, ne, nd)
        assert _rel(mem, mem_o) < 1e-12 and _rel(hs, hs_o.reshape(B, d)) < 1e-12


@pytest.mark.parametrize("tag", sorted(TRANSFORMER_CASES))
def test_composed_steps_reproduce_the_reference_module(tag):
    g = np.load(os.path.join(GOLD, "transformer.npz"))
    d, nh, ff, ne, nd, L, B, seed, use_mask = TRANSFORMER_CASES[tag]
    sd = synth.make_transformer_state_dict(seed, d, nh, ff, ne, nd)
    src, pos, qe, mask = _inputs(d, L, B, seed, use_mask)
    hs, mem = R.compose(sd, src, pos, mask, qe, nh, ne, nd)
    assert _rel(mem, torch.from_numpy(g[tag + "_memory"]).reshape(mem.shape)) < 1e-5
    assert _rel(hs, torch.from_numpy(g[tag + "_hs"]).reshape(hs.shape)) < 1e-5


def test_token_step_reproduces_the_reference_filter_predictor():
    from ref_weights import GOLDEN, token_inputs, token_state_dict
    from pytracking_b200.transformer_engine import TokenBuilder
    gold = np.load(GOLDEN)
    train_feat, test_feat, label, ltrb = token_inputs()
    for use_test in (0, 1):
        tb = TokenBuilder(token_state_dict(gold, use_test), device="cpu")
        st = R.tokens(train_feat[:, 0], test_feat[:, 0], label[:, 0], ltrb[:, 0], tb.fg, tb.test if use_test else None, tb.w1, tb.b1,
                      tb.w2t, tb.b2, tb.w3t, tb.b3, 2)
        name = "tok%d_feat" % use_test
        assert tuple(st.ref.shape) == tuple(gold[name + "_shape"])
        a = st.ref.reshape(-1)[torch.from_numpy(gold[name + "_idx"])]
        assert float((a - torch.from_numpy(gold[name]).double()).abs().max() / float(gold[name + "_amax"])) < 1e-6


def test_tower_steps_reproduce_the_reference_box_regressor():
    from ref_weights import GOLDEN, tower_inputs, tower_state_dict
    gold = np.load(GOLDEN)
    sd = tower_state_dict(gold)
    feat, filt = tower_inputs()
    fp = (filt.reshape(1, 256) @ sd["linear.weight"].t() + sd["linear.bias"]).reshape(1, 256, 1, 1)
    att = R.conv1x1(feat[0], fp.reshape(1, 256)).ref[:, 0]
    sd = {k: v.double() for k, v in sd.items()}
    x = R.import_scaled(feat[0].double(), att).ref
    for i in range(4):
        x = R.conv3x3(x, sd["tower.%d.weight" % (3 * i)], sd["tower.%d.bias" % (3 * i)]).ref
        x = R.groupnorm_relu(x, sd["tower.%d.weight" % (3 * i + 1)], sd["tower.%d.bias" % (3 * i + 1)]).ref
    y = R.export_exp(R.conv3x3(x, sd["bbreg_layer.weight"], sd["bbreg_layer.bias"]).ref).ref
    assert _rel(y, torch.from_numpy(gold["tower_out"])) < 1e-5


# ---- the bounds against the kernel sources on the CPU -------------------------------------------------------------------------------
def _emul(tmp_path_factory, name):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    out = os.path.join(str(tmp_path_factory.mktemp(name)), "lib%s.so" % name)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-fno-gnu-unique", "-Wno-unknown-pragmas",
                    os.path.join(ROOT, "tests", "cpu_emul", name + ".cpp"), "-o", out], check=True, capture_output=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def tr(tmp_path_factory):
    return _emul(tmp_path_factory, "transformer_emul")


@pytest.fixture(scope="module")
def tomp(tmp_path_factory):
    return _emul(tmp_path_factory, "tomp_emul")


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _np(t):
    return np.ascontiguousarray(t.numpy())


@pytest.mark.parametrize("L,B,H,use_mask", [(72, 2, 2, True), (130, 1, 3, False), (17, 3, 1, True)])
def test_attention_bounds_hold_for_the_kernel_sources(tr, L, B, H, use_mask):
    g = torch.Generator().manual_seed(L)
    D = H * 32
    qk, v = torch.randn(L, B, 2 * D, generator=g) * 2, torch.randn(L, B, D, generator=g)
    mask = None
    if use_mask:
        mask = torch.zeros(B, L, dtype=torch.bool)
        mask[B - 1, L // 3: L // 2] = True
    scale = 1.0 / 32 ** 0.5
    qkn, vn = _np(qk), _np(v)
    m8 = _np(mask.to(torch.uint8)) if mask is not None else None
    out = np.full((L, B, D), np.nan, np.float32)
    kptr = C.c_void_p(qkn.ctypes.data + D * 4)
    assert tr.tr_emul_attention(_p(qkn), kptr, _p(vn), _p(m8), _p(out), L, L, B, H, 2 * D, 2 * D, D, D, C.c_float(scale)) == 0
    R.check(torch.from_numpy(out), R.attention(qk, v, mask, H, scale), "attention")
    q1 = torch.randn(B, D, generator=g) * 2
    o1 = np.full((B, D), np.nan, np.float32)
    assert tr.tr_emul_attention_q1(_p(_np(q1)), kptr, _p(vn), _p(m8), _p(o1), L, B, H, D, 2 * D, D, D, C.c_float(scale)) == 0
    R.check(torch.from_numpy(o1), R.attention_q1(q1, qk[..., D:], v, mask, H, scale), "attention_q1")


def test_layernorm_add_pos_small_linear_bounds_hold_for_the_kernel_sources(tr):
    g = torch.Generator().manual_seed(1)
    T, D = 37, 256
    x, gam, bet = torch.randn(T, D, generator=g) * 3 + 1, torch.rand(D, generator=g) + 0.5, torch.randn(D, generator=g)
    y = np.full((T, D), np.nan, np.float32)
    assert tr.tr_emul_layernorm(_p(_np(x)), _p(_np(gam)), _p(_np(bet)), _p(y), T, D) == 0
    R.check(torch.from_numpy(y), R.layernorm(x, gam, bet), "layernorm")
    L, B = 9, 2
    for Bp in (1, 2):
        src, pos = torch.randn(L, B, D, generator=g), torch.randn(L, Bp, D, generator=g)
        out = np.full((L, B, D), np.nan, np.float32)
        assert tr.tr_emul_add_pos(_p(_np(src)), _p(_np(pos)), _p(out), L, B, Bp, D) == 0
        assert torch.equal(torch.from_numpy(out), R.add_pos(src, pos).r32)
    M, K, N = 2, 256, 96
    xm, W, b, res = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / 16, torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    for relu, r in ((0, res), (1, None)):
        out = np.full((M, N), np.nan, np.float32)
        assert tr.tr_emul_small_linear(_p(_np(xm)), _p(_np(W)), _p(_np(b)), _p(_np(r)) if r is not None else None, _p(out), M, K, N, relu) == 0
        R.check(torch.from_numpy(out), R.small_linear(xm, W, b, r, bool(relu)), "small_linear")


@pytest.mark.parametrize("D,D1,n_train,n_test,hw,B,use_test_token", [(256, 64, 2, 1, 6, 2, False), (64, 16, 1, 2, 5, 1, True)])
def test_token_bound_holds_for_the_kernel_source(tomp, D, D1, n_train, n_test, hw, B, use_test_token):
    g = torch.Generator().manual_seed(D)
    trf, tef = torch.randn(n_train, D, hw, hw, generator=g), torch.randn(n_test, D, hw, hw, generator=g)
    label, ltrb = torch.rand(n_train, hw, hw, generator=g), torch.rand(n_train, 4, hw, hw, generator=g)
    fg, tt = torch.randn(D, generator=g), torch.randn(D, generator=g)
    w1, b1 = torch.randn(D1, 4, generator=g), torch.randn(D1, generator=g)
    w2, b2 = torch.randn(D, D1, generator=g) / D1 ** 0.5, torch.randn(D, generator=g)
    w3, b3 = torch.randn(D, D, generator=g) / D ** 0.5, torch.randn(D, generator=g)
    out = np.full(((n_train + n_test) * hw * hw, B, D), np.nan, np.float32)
    assert tomp.tomp_emul_tokens(_p(_np(trf)), _p(_np(tef)), _p(_np(label)), _p(_np(ltrb)), _p(_np(fg)), _p(_np(tt)) if use_test_token else None,
                                 _p(_np(w1)), _p(_np(b1)), _p(_np(w2.t())), _p(_np(b2)), _p(_np(w3.t())), _p(_np(b3)), _p(out), n_train, n_test,
                                 hw, hw, D, D1, B) == 0
    st = R.tokens(trf, tef, label, ltrb, fg, tt if use_test_token else None, w1, b1, w2.t().contiguous(), b2, w3.t().contiguous(), b3, B)
    R.check(torch.from_numpy(out), st, "tokens")


def test_tower_kernel_bounds_hold_for_the_kernel_sources(tomp):
    g = torch.Generator().manual_seed(2)
    S, Cc, hw = 2, 40, 7
    HW = hw * hw
    feat, att = torch.randn(S, Cc, hw, hw, generator=g), torch.rand(S, hw, hw, generator=g)
    out = np.full((S, HW, Cc), np.nan, np.float32)
    assert tomp.tomp_emul_import_scaled(_p(_np(feat)), _p(_np(att)), _p(out), S, HW, Cc) == 0
    assert torch.equal(torch.from_numpy(out).reshape(S, hw, hw, Cc), R.import_scaled(feat, att).r32)
    x = torch.randn(S, hw, hw, Cc, generator=g) * 2 + 0.5
    gam, bet = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g)
    xn = _np(x).copy()
    assert tomp.tomp_emul_groupnorm1_relu(_p(xn), _p(_np(gam)), _p(_np(bet)), S, HW, Cc) == 0
    R.check(torch.from_numpy(xn), R.groupnorm_relu(x, gam, bet), "groupnorm_relu")
    y = torch.randn(S, hw, hw, 4, generator=g)
    e = np.full((S, 4, HW), np.nan, np.float32)
    assert tomp.tomp_emul_export_exp(_p(_np(y)), _p(e), S, HW, 4) == 0
    R.check(torch.from_numpy(e).reshape(S, 4, hw, hw), R.export_exp(y), "export_exp")
