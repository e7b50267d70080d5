"""-m gpu: the ToMP head on the device, launch by launch, against float64 (tests/tomp_step_ref.py).

Each transformer case runs `Transformer.forward` once per launch of its fixed sequence, stopped right after that launch
(`b200trk_transformer_debug_stop_after`); every launch writes a buffer it does not read, so one stopped run holds the launch's inputs
and its output (`b200trk_transformer_debug_buffer`).  The output is then held to the float64 reference of the same operation on those
inputs:
  * token GEMMs (wgmma, 3xTF32): e <= e_TF32 / 16 and e <= (K + 2) 2^-23 + 2^-20, e = max |y - ref| / mag;
  * add_pos: bitwise equal to torch's float32 add;
  * attention, single-query attention, LayerNorm, small_linear: every entry within max(4 e_32, bound), and the case's worst e within
    20 x its worst e_32 + 64 ulp of the magnitude term (`yardstick`).
The tower (import, 3x3 convolutions, GroupNorm + ReLU, exp export) is checked the same way through `b200trk_tower_debug_*`, the token
assembly and the 1x1 correlation (`ops.conv1x1`) on their outputs.  Each case prints its GEMM plans and the worst ratios per kind; the
last test asserts the plans the cases were chosen to reach.  Bitwise properties: batch permutation, an all-False mask row against no
mask, identical batch entries, repeats, and a stopped run's buffers against the full run's."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import tomp_step_ref as R
from pytracking_b200 import _lib, ops, synth
from pytracking_b200.transformer_engine import BoxTower, TokenBuilder, TransformerEngine

pytestmark = pytest.mark.gpu

MAX_L_H100 = 57792          # (232448 B opt-in - 256 B static) / 4 - 256: the largest L the decoder's attention holds on an H100
PLANS = []                  # (case, gemm info) of every transformer case, for test_zz_plan_coverage
WORST = {}                  # kind -> [worst e / bar, worst yardstick ratio]


def _note(kind, ratio_bar, yard):
    w = WORST.setdefault(kind, [0.0, 0.0])
    w[0], w[1] = max(w[0], ratio_bar), max(w[1], yard)


def _inputs(L, B, Bp, d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(L, B, d, generator=g), torch.randn(L, Bp, d, generator=g) * 0.5, torch.randn(1, d, generator=g)


def _buf(eng, i):
    n = C.c_longlong()
    _lib.check(_lib.lib().b200trk_transformer_debug_buffer(eng.handle, i, None, C.byref(n), None), "debug_buffer")
    t = torch.empty(n.value, device="cuda")
    _lib.check(_lib.lib().b200trk_transformer_debug_buffer(eng.handle, i, C.c_void_p(t.data_ptr()), None, None), "debug_buffer")
    torch.cuda.synchronize()
    if i <= R.K:
        return t.reshape(eng.L, eng.B, -1)
    return t.reshape(eng.B, -1)


def _stop(eng, k):
    _lib.check(_lib.lib().b200trk_transformer_debug_stop_after(eng.handle, k), "debug_stop_after")


def _gemms(eng, n):
    out = []
    for g in range(n):
        info = (C.c_int * 15)()
        _lib.check(_lib.lib().b200trk_transformer_debug_gemm(eng.handle, g, C.byref(info)), "debug_gemm")
        out.append(list(info))
    return out


def _run(eng, src, mask, qe, pos):
    hs, mem = eng.forward(src, mask, qe, pos)
    torch.cuda.synchronize()
    return hs.reshape(eng.B, -1), mem


def check_transformer(name, L, B, d=256, H=8, FF=2048, ne=6, nd=6, Bp=1, mask=None, seed=0, rows=None):
    """Every launch of one forward pass against float64; returns (hs, memory) of the full run."""
    sd = synth.make_transformer_state_dict(seed + 90, d, H, FF, ne, nd)
    src, pos, qe = _inputs(L, B, Bp, d, seed)
    src, pos, qe = src.cuda(), pos.cuda(), qe.cuda()
    m = mask.cuda() if mask is not None else None
    sdc = {k: v.cuda() for k, v in sd.items()}
    eng = TransformerEngine(sd, L, B, d, H, FF, ne, nd)
    try:
        plan = R.launch_plan(ne, nd)
        assert _lib.lib().b200trk_transformer_debug_num_launches(eng.handle) == len(plan)
        hs, mem = _run(eng, src, m, qe, pos)
        hs2, mem2 = _run(eng, src, m, qe, pos)
        assert torch.equal(hs, hs2) and torch.equal(mem, mem2), "%s: repeats differ" % name
        infos = _gemms(eng, 5 * ne + 2 * nd)
        for g, info in enumerate(infos):
            PLANS.append((name, info))
            print("%s gemm %2d  %3d->%3d res %2d relu %d  image %4dx%-3d K %4d N %4d  grid %s BN %d red %d tile %dx%d" % (
                name, g, info[0], info[1], info[2], info[3], info[4], info[5], info[6], info[7], info[8:11], info[11], info[12], info[13],
                info[14]))
        gi, worst = 0, {}
        for k, e in enumerate(plan):
            _stop(eng, k)
            _run(eng, src, m, qe, pos)
            bufs = {i: _buf(eng, i) for i in set(e["ins"]) | ({e["res"]} if e.get("res") is not None else set())}
            out = hs if e["out"] == R.HS else _buf(eng, e["out"])
            if k == len(plan) - 1:
                assert torch.equal(out, hs), "%s: the stopped run's hs differs from the full run's" % name
            if e["kind"] == "add_pos" and e["out"] == R.MEM_POS:
                assert torch.equal(bufs[R.SRC], mem), "%s: src after the encoder differs from the full run's memory" % name
            what = "%s launch %d (%s %s)" % (name, k, e["kind"], e.get("p", ""))
            kind = e["kind"]
            if kind in ("add_pos", "add_query_pos"):
                st = R.run_step(e, bufs, sdc, pos, m, H)
                assert torch.equal(out, st.r32), what
                continue
            if kind == "gemm":
                st = R.run_step(e, bufs, sdc, pos, m, H)
                ee, et = R.check_gemm(out, st, infos[gi][6], what)
                gi += 1
                w = worst.setdefault("gemm", [0.0, 0.0])
                w[0], w[1] = max(w[0], ee), max(w[1], ee / max(et, 1e-30))
                _note("gemm e/e_tf32", ee / max(et, 1e-30), 0.0)
                continue
            if kind == "attention" and rows is not None:
                st = R.attention(bufs[R.QK], bufs[R.V], m, H, 1.0 / math.sqrt(32.0), rows=rows)
                out = out[rows]
            else:
                st = R.run_step(e, bufs, sdc, pos, m, H)
            rb, yd, _ = R.check(out, st, what)
            assert yd <= 1.0, "%s: worst e %.3g x the yardstick (20 e_32 + 64 ulp)" % (what, yd)
            w = worst.setdefault(kind, [0.0, 0.0])
            w[0], w[1] = max(w[0], rb), max(w[1], yd)
            _note(kind, rb, yd)
        assert gi == len(infos)
        for kind, (a, b) in sorted(worst.items()):
            if kind == "gemm":
                print("%s: gemm worst e %.3e, worst e / e_tf32 %.4f" % (name, a, b))
            else:
                print("%s: %-13s worst e / bar %.3f, worst e / yardstick %.3f" % (name, kind, a, b))
        _stop(eng, -1)
        return hs, mem
    finally:
        eng.close()


def _mask(B, L, spans):
    m = torch.zeros(B, L, dtype=torch.bool)
    for b, a, z in spans:
        m[b, a:z] = True
    return m


def test_tomp_l648_one_training_frame():
    check_transformer("l648", 648, 2, mask=_mask(2, 648, []), seed=1)


def test_tomp_l972_masked_run_inside_a_key_tile():
    check_transformer("l972", 972, 2, mask=_mask(2, 972, [(1, 324, 648)]), seed=2)


def test_prime_token_count_one_wide_plan():
    check_transformer("prime1009", 1009, 1, ne=2, nd=2, mask=_mask(1, 1009, [(0, 5, 70)]), seed=3)        # L B = 1009, prime


def test_mask_edges_tile_and_single_live_key():
    L = 203                                                                                                # not a multiple of 16 or 64
    m = _mask(3, L, [(0, 64, 128), (1, 0, 100), (1, 101, L)])                                              # a whole key tile; one live key
    check_transformer("edges", L, 3, ne=2, nd=2, mask=m, seed=4)


def test_no_mask_pos_per_batch_b8():
    check_transformer("b8_bp8", 100, 8, ne=2, nd=2, Bp=8, seed=5)


def test_small_d64():
    check_transformer("d64", 40, 2, d=64, H=2, FF=128, ne=2, nd=2, mask=_mask(2, 40, [(1, 13, 20)]), seed=6)


def test_b1_l11969_runs():
    """The first L whose single-query attention needs more than 48 KB of shared memory (failed to launch before create opted in)."""
    check_transformer("l11969", 11969, 1, ne=1, nd=1, mask=_mask(1, 11969, [(0, 100, 4000)]), seed=7,
                      rows=torch.arange(0, 11969, 47))


def test_largest_accepted_l_and_the_next_refused():
    L = MAX_L_H100
    if torch.cuda.get_device_properties(0).shared_memory_per_block_optin != 232448:
        pytest.skip("limit pinned for an H100's 227 KB opt-in shared memory")
    check_transformer("lmax", L, 1, ne=1, nd=1, mask=_mask(1, L, [(0, 1000, 30000)]), seed=8, rows=torch.arange(0, L, 229))
    sd = synth.make_transformer_state_dict(98, 256, 8, 2048, 1, 1)
    free0 = torch.cuda.mem_get_info()[0]
    with pytest.raises(RuntimeError, match="L <= %d" % L):
        TransformerEngine(sd, L + 1, 1, 256, 8, 2048, 1, 1)
    assert torch.cuda.mem_get_info()[0] >= free0 - (64 << 20), "a refused create kept device memory"


def test_bitwise_batch_permutation_mask_rows_and_identical_entries():
    d, H, FF, ne, nd, L = 256, 8, 2048, 2, 2, 324
    sd = synth.make_transformer_state_dict(99, d, H, FF, ne, nd)
    src, pos, qe = (t.cuda() for t in _inputs(L, 2, 2, d, 9))
    mask = _mask(2, L, [(0, 100, 200)]).cuda()
    eng = TransformerEngine(sd, L, 2, d, H, FF, ne, nd)
    try:
        hs, mem = _run(eng, src, mask, qe, pos)
        p = [1, 0]
        hs_p, mem_p = _run(eng, src[:, p].contiguous(), mask[p].contiguous(), qe, pos[:, p].contiguous())
        assert torch.equal(hs_p, hs[p]) and torch.equal(mem_p, mem[:, p]), "permuting the batch does not permute the outputs"
        hs_n, mem_n = _run(eng, src, None, qe, pos)
        assert torch.equal(hs_n[1], hs[1]) and torch.equal(mem_n[:, 1], mem[:, 1]), "an all-False mask row differs from no mask"
        same = src[:, :1].expand(L, 2, d).contiguous()
        hs_s, mem_s = _run(eng, same, torch.zeros(2, L, dtype=torch.bool, device="cuda"), qe, pos[:, :1].contiguous())
        assert torch.equal(hs_s[0], hs_s[1]) and torch.equal(mem_s[:, 0], mem_s[:, 1]), "identical batch entries differ"
    finally:
        eng.close()


# ---- the tower ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
def test_tower_steps(precision):
    from ref_weights import GOLDEN, tower_state_dict
    sd = tower_state_dict(np.load(GOLDEN))
    sdc = {k: v.cuda() for k, v in sd.items()}
    tw = BoxTower(sd, 18, 18, max_batch=4, precision=precision)
    L = _lib.lib()
    try:
        n = L.b200trk_tower_debug_num_launches(tw.handle)
        nconv = (n - 1) // 2
        for S in (1, 2, 3, 4):
            g = torch.Generator().manual_seed(20 + S)
            feat = (torch.randn(S, 256, 18, 18, generator=g) * 0.3).cuda()
            att = torch.rand(S, 18, 18, generator=g).cuda()
            full = tw.forward(feat, att)
            assert torch.equal(full, tw.forward(feat, att)), "tower repeats differ"

            def buf(i, C_):
                t = torch.empty(S, 18, 18, C_, device="cuda")
                _lib.check(L.b200trk_tower_debug_buffer(tw.handle, i, S, C.c_void_p(t.data_ptr()), None), "tower_debug_buffer")
                torch.cuda.synchronize()
                return t
            for k in range(n):
                _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k), "tower_debug_stop_after")
                out = tw.forward(feat, att)
                torch.cuda.synchronize()
                what = "tower p%d S=%d launch %d" % (precision, S, k)
                if k == 0:
                    assert torch.equal(buf(0, 256), R.import_scaled(feat, att).r32), what
                    continue
                ci, is_gn = (k - 1) // 2, (k - 1) % 2 == 1
                info = (C.c_int * 10)()
                _lib.check(L.b200trk_tower_debug_conv(tw.handle, min(ci, nconv - 1), C.byref(info)), "tower_debug_conv")
                if k == n - 1:
                    x = buf(info[9], 4)
                    rb, yd, _ = R.check(full, R.export_exp(x), what)
                    assert torch.equal(out, full)
                    _note("export_exp", rb, yd)
                    continue
                cout = info[1]
                key = "bbreg_layer" if ci == nconv - 1 else "tower.%d" % (3 * ci)
                if not is_gn:
                    _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k - 1), "tower_debug_stop_after")
                    tw.forward(feat, att)
                    torch.cuda.synchronize()
                    x = buf(ci, 256)                                  # the input as the convolution read it (after the previous GN)
                    _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k), "tower_debug_stop_after")
                    tw.forward(feat, att)
                    torch.cuda.synchronize()
                    y = buf(ci + 1, cout)
                    st = R.conv3x3(x, sdc[key + ".weight"], sdc[key + ".bias"])
                    print("%s conv %d tc %d grid %s BN %d red %d tile_w %d" % (what, ci, info[2], list(info[3:6]), info[6], info[7], info[8]))
                    if info[2]:
                        ee, et = R.check_gemm(y, st, 9 * 256, what)
                        _note("tower conv e/e_tf32", ee / max(et, 1e-30), 0.0)
                    else:
                        ee = float(((y.double() - st.ref).abs() / st.mag).max())
                        assert ee <= R.gemm_bound_rel(9 * 256), "%s: e %.3e above the fp32 summation bound" % (what, ee)
                        e32 = float(((st.r32.double() - st.ref).abs() / st.mag).max())
                        yd = ee / (R.YARD * e32 + R.FLOOR)
                        assert yd <= 1.0, "%s: e %.3e vs e_32 %.3e" % (what, ee, e32)
                        _note("tower conv fp32 yardstick", yd, yd)
                else:
                    _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k - 1), "tower_debug_stop_after")
                    tw.forward(feat, att)
                    torch.cuda.synchronize()
                    x = buf(ci + 1, 256)                              # GroupNorm's input exists only between the two launches
                    _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, k), "tower_debug_stop_after")
                    tw.forward(feat, att)
                    torch.cuda.synchronize()
                    y = buf(ci + 1, 256)
                    gn = "tower.%d" % (3 * ci + 1)
                    rb, yd, _ = R.check(y, R.groupnorm_relu(x, sdc[gn + ".weight"], sdc[gn + ".bias"]), what)
                    assert yd <= 1.0, "%s: yardstick %.3f" % (what, yd)
                    _note("groupnorm_relu", rb, yd)
            _lib.check(L.b200trk_tower_debug_stop_after(tw.handle, -1), "tower_debug_stop_after")
    finally:
        tw.close()


# ---- tokens and the 1x1 correlation -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_train", [1, 2])
@pytest.mark.parametrize("use_test", [0, 1])
def test_token_assembly_steps(n_train, use_test):
    from ref_weights import GOLDEN, token_state_dict
    tb = TokenBuilder(token_state_dict(np.load(GOLDEN), use_test))
    g = torch.Generator().manual_seed(30 + n_train)
    trf, tef = torch.randn(n_train, 256, 18, 18, generator=g).cuda(), torch.randn(1, 256, 18, 18, generator=g).cuda()
    label, ltrb = torch.rand(n_train, 18, 18, generator=g).cuda(), (torch.rand(n_train, 4, 18, 18, generator=g) * 2).cuda()
    out = tb.build(trf, tef, label, ltrb, B=2, use_test_token=bool(use_test))
    torch.cuda.synchronize()
    st = R.tokens(trf, tef, label, ltrb, tb.fg, tb.test if use_test else None, tb.w1, tb.b1, tb.w2t, tb.b2, tb.w3t, tb.b3, 2)
    rb, yd, _ = R.check(out, st, "tokens n_train=%d test=%d" % (n_train, use_test))
    assert yd <= 1.0
    assert torch.equal(out[:, 0], out[:, 1])
    _note("tokens", rb, yd)


@pytest.mark.parametrize("S", [1, 2])
def test_conv1x1_correlation_steps(S):
    g = torch.Generator().manual_seed(40 + S)
    x = torch.randn(S, 256, 18, 18, generator=g).cuda()
    P = (torch.randn(1, 256, generator=g) * 0.1).cuda()
    y = ops.conv1x1(x, P.reshape(1, 256, 1, 1))
    torch.cuda.synchronize()
    rb, yd, _ = R.check(y, R.conv1x1(x, P), "conv1x1 S=%d" % S)
    assert yd <= 1.0
    _note("conv1x1", rb, yd)


def test_zz_plan_coverage():
    """The GEMM plans the transformer cases were chosen to reach (and the per-kind worst ratios of the whole file)."""
    for kind, (a, b) in sorted(WORST.items()):
        print("worst over the file: %-26s e / bar %.4f   yardstick %.4f" % (kind, a, b))
    if not PLANS:
        pytest.skip("no transformer case ran")
    infos = [i for _, i in PLANS]
    assert any(i[5] == 1 for i in infos), "no 1-wide token image (L B prime)"
    assert any(i[4] % i[14] != 0 for i in infos), "no partial last row tile"
    assert any(i[12] == 1 for i in infos), "no split-K through the cluster"
    assert any(i[12] == 2 for i in infos), "no split-K through the workspace"
    assert {64, 128} <= {i[11] for i in infos}, "BN 64 and 128 not both reached"
