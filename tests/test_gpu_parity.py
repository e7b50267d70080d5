"""GPU parity tests: the CUDA path (through the C ABI) against the oracle and the committed golden vectors.
Tolerances: score maps / filter weights <= 1e-4 relative (fp32), indices bit-exact."""
import os

import numpy as np
import pytest
import torch

from pytracking_b200 import synth

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture(scope="module")
def G(golden_dir):
    return {n: np.load(os.path.join(golden_dir, n + ".npz")) for n in ("corr", "labels", "dimp_sd", "prdimp_sd", "backbone")}


@pytest.fixture(scope="module")
def ops():
    from pytracking_b200 import ops as o
    return o


@pytest.mark.parametrize("tag,n,c,h", [("a", 3, 32, 18), ("b", 2, 64, 22)])
def test_apply_filter_golden(G, ops, tag, n, c, h):
    g = G["corr"]
    feat = synth.make_clf_features(100 + ord(tag), n, c, h, h).cuda()
    w = torch.from_numpy(g[tag + "_w"]).cuda()
    s, mv, mi = ops.apply_filter(feat, w, return_max=True)
    assert _rel(s, g[tag + "_scores"].reshape(s.shape)) < 1e-5
    assert np.array_equal(mi.cpu().numpy(), g[tag + "_maxidx"])
    assert _rel(mv, g[tag + "_maxval"]) < 1e-5
    r = torch.from_numpy(g[tag + "_r"])[:, 0:1].cuda()
    gt = ops.apply_feat_transpose(feat, r, 4)
    assert _rel(gt, g[tag + "_grad"]) < 1e-5


@pytest.mark.parametrize("n,c,h", [(1, 512, 18), (5, 512, 18), (50, 512, 18), (17, 256, 18), (3, 512, 22), (33, 64, 22)])
def test_apply_filter_oracle(ops, n, c, h):
    from oracle import dimp_oracle as O
    feat = synth.make_clf_features(7 * n + c, n, c, h, h)
    w = torch.randn(1, c, 4, 4, generator=torch.Generator().manual_seed(n)) * 0.3
    s_ref = O.apply_filter(feat, w)
    s, mv, mi = ops.apply_filter(feat.cuda(), w.cuda(), return_max=True)
    assert _rel(s, s_ref) < 1e-5
    mv_ref, mi_ref = O.max2d(s.cpu()[:, 0])          # arg-max of the engine's own map must follow the reference rule
    assert torch.equal(mi.cpu(), mi_ref) and torch.equal(mv.cpu(), mv_ref)
    r = torch.randn(n, 1, h + 1, h + 1, generator=torch.Generator().manual_seed(n + 1))
    g_ref = O.apply_feat_transpose(feat, r, 4)
    g = ops.apply_feat_transpose(feat.cuda(), r.cuda(), 4)
    assert _rel(g, g_ref) < 1e-5
    # adjointness: <A w, r> == <w, A^T r>
    lhs = float((s.cpu().double() * r.double()).sum())
    rhs = float((w.double() * g.cpu().double()).sum())
    assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs))


def test_max2d_ties(ops):
    a = torch.zeros(3, 19, 19)
    a[0, 3, 1] = 1.0; a[0, 1, 3] = 1.0
    a[1, 4, 2] = 2.0; a[1, 2, 2] = 2.0
    a[2] = -1.0; a[2, 18, 18] = -0.5
    mv, mi = ops.max2d(a.cuda())
    assert mi.cpu().tolist() == [[3, 1], [2, 2], [18, 18]]
    assert mv.cpu().tolist() == [1.0, 2.0, -0.5]


@pytest.mark.parametrize("tag,n,c,h,it,use_sw,seed", [("n15_it10", 15, 512, 18, 10, True, 21), ("n50_it2", 50, 512, 18, 2, True, 22),
                                                      ("n4_c64", 4, 64, 18, 3, False, 23), ("n7_22", 7, 128, 22, 4, True, 24)])
def test_dimp_sd_golden(G, ops, tag, n, c, h, it, use_sw, seed):
    g = G["dimp_sd"]
    p = synth.make_dimp_optimizer_params(seed=seed)
    feat = synth.make_clf_features(seed, n, c, h, h).cuda()
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda()
    sw = torch.from_numpy(g[tag + "_sw"]).cuda() if use_sw else None
    step = float(torch.exp(p["log_step_length"]))
    reg = max(float(p["filter_reg"]) ** 2, 1e-3 ** 2)
    w, its, losses = ops.dimp_sd_gn(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, sw,
                                    p["label_map_predictor.weight"].cuda(), p["target_mask_predictor.0.weight"].cuda(),
                                    p["spatial_weight_predictor.weight"].cuda(), it, step, reg,
                                    return_iterates=True, compute_losses=True)
    assert _rel(its[1], g[tag + "_w1"][0]) < 1e-4
    assert _rel(w, g[tag + "_wfinal"]) < 1e-4
    assert _rel(its[-1], g[tag + "_wfinal"][0]) < 1e-4
    assert np.allclose(losses.cpu().numpy(), g[tag + "_losses"], rtol=1e-4)
    # run-to-run bitwise determinism (fixed summation order)
    w2, _, _ = ops.dimp_sd_gn(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, sw,
                              p["label_map_predictor.weight"].cuda(), p["target_mask_predictor.0.weight"].cuda(),
                              p["spatial_weight_predictor.weight"].cuda(), it, step, reg)
    assert torch.equal(w, w2)


def test_dimp_sd_full_size_properties(ops):
    """BASELINE size (n=50, C=512, 10 iterations): loss decreases monotonically; zero iterations is the identity."""
    p = synth.make_dimp_optimizer_params(seed=3)
    feat = synth.make_clf_features(77, 50, 512, 18, 18).cuda()
    bb = synth.make_boxes(78, 50).cuda()
    sw = torch.full((50,), 1.0 / 50).cuda()
    luts = [p[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
    w0 = torch.zeros(1, 512, 4, 4).cuda()
    w, its, losses = ops.dimp_sd_gn(w0, feat, bb, sw, *luts, 10, 0.9, 0.01, return_iterates=True, compute_losses=True)
    l = losses.cpu().numpy()
    assert np.all(np.diff(l) < 0), l
    w_id, _, _ = ops.dimp_sd_gn(w, feat, bb, sw, *luts, 0, 0.9, 0.01)
    assert torch.equal(w_id, w)
    # the carried score maps (linear recurrence) must agree with a fresh correlation of the final filter
    from oracle import dimp_oracle as O
    w_ref, _, l_ref = O.dimp_sd_gn(w0.cpu(), feat.cpu(), bb.cpu(), sw.cpu(), p, 10, min_filter_reg=0.1)
    assert _rel(w, w_ref) < 1e-4
    assert np.allclose(l, [float(x) for x in l_ref], rtol=1e-4)


@pytest.mark.parametrize("tag,n,c,h,it,seed,sreg,lthr", [("n15_22", 15, 512, 22, 10, 31, None, 0.0), ("n6_18", 6, 64, 18, 3, 32, -2.0, 0.05)])
def test_prdimp_sd_golden(G, ops, tag, n, c, h, it, seed, sreg, lthr):
    g = G["prdimp_sd"]
    feat = synth.make_clf_features(seed, n, c, h, h).cuda()
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda()
    w, its, losses = ops.prdimp_sd_newton(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, torch.from_numpy(g[tag + "_sw"]).cuda(),
                                          it, float(g[tag + "_sigma"]), 1.0, 0.05 ** 2, alpha_eps=0.05, softmax_reg=sreg,
                                          label_threshold=lthr, normalize_label=True,
                                          label_shrink=0.0 if sreg is None else 0.1, return_iterates=True, compute_losses=True)
    assert _rel(its[1], g[tag + "_w1"][0]) < 1e-4
    assert _rel(w, g[tag + "_wfinal"]) < 1e-4
    assert np.allclose(losses.cpu().numpy(), g[tag + "_losses"], rtol=1e-4)


@pytest.mark.parametrize("arch,size,seed,precision", [("resnet50", 96, 42, 1), ("resnet18", 96, 42, 1), ("resnet50", 288, 41, 1),
                                                      ("resnet50", 96, 42, 0), ("resnet18", 96, 42, 0), ("resnet50", 288, 41, 0)])
def test_backbone_golden(G, arch, size, seed, precision):
    from pytracking_b200.engine import BackboneEngine
    g = G["backbone"]
    sd = synth.make_dimp_state_dict(arch, seed=0, lut_seed=3)
    eng = BackboneEngine(sd, arch=arch, max_batch=2, crop_size=size, precision=precision)
    im = synth.make_crop(seed, 1, size).cuda()
    out = eng.forward(im)
    tag = "%s_%d_" % (arch, size)
    l2 = out["layer2"] if size == 96 else out["layer2"][:, ::8]
    assert _rel(l2, g[tag + "layer2"]) < 1e-4
    assert _rel(out["layer3"], g[tag + "layer3"]) < 1e-4
    assert _rel(out["classification"], g[tag + "clf"]) < 1e-4
    # a batch of two different crops: row 0 is the golden crop, row 1 another crop's batch-1 pass (a kernel that read one sample for
    # every row, or mixed rows, fails one of the two)
    im1 = synth.make_crop(seed + 1, 1, size).cuda()
    one = eng.forward(im1)
    out2 = eng.forward(torch.cat([im, im1]))
    assert _rel(out2["layer2"][0] if size == 96 else out2["layer2"][0:1, ::8], g[tag + "layer2"]) < 1e-4
    assert _rel(out2["layer3"][0], g[tag + "layer3"][0]) < 1e-4
    assert _rel(out2["classification"][0], g[tag + "clf"][0]) < 1e-4
    for name in ("layer2", "layer3", "classification"):
        assert _rel(out2[name][1], one[name][0]) < 1e-4, name
    eng.close()


def test_prroi_known_answer(ops):
    """The reference's only known-answer test (PreciseRoIPooling/pytorch/tests/test_prroi_pooling2d.py:21-35):
    on integer-aligned RoIs with spatial_scale 0.5, PrRoIPool 7x7 equals avg_pool2d(k=2, s=1) slices."""
    import torch.nn.functional as F
    feat = torch.rand(4, 16, 24, 32, generator=torch.Generator().manual_seed(0)).cuda()
    rois = torch.tensor([[0, 0, 0, 14, 14], [1, 14, 14, 28, 28]], dtype=torch.float32).cuda()
    out = ops.prroi_pool_forward(feat, rois, 7, 7, 0.5)
    ref = F.avg_pool2d(feat, kernel_size=2, stride=1)
    assert torch.allclose(out[0], ref[0, :, :7, :7], atol=1e-6)
    assert torch.allclose(out[1], ref[1, :, 7:14, 7:14], atol=1e-6)


ATOM_CG_CASES = {"n12_c16_pr_mlu": (12, 16, 12, 5, False, "mlu", 51), "n40_c64_pr_mlu": (40, 64, 25, 5, False, "mlu", 52),
                 "n9_c32_fr_none": (9, 32, 9, 4, True, "none", 53), "n20_c64_pr_relu": (20, 64, 20, 3, False, "relu", 54)}


@pytest.mark.parametrize("tag", sorted(ATOM_CG_CASES))
def test_atom_cg_golden(golden_dir, ops, tag):
    """ATOM ConjugateGradient.run on ConvProblem against the outputs of the reference classes (two consecutive runs)."""
    g = np.load(os.path.join(golden_dir, "atom_cg.npz"))
    n, c, nf, it, fr, act, seed = ATOM_CG_CASES[tag]
    x, y, sw = synth.make_atom_memory(seed, n, c, 18, 18, n_filled=nf)
    x, y, sw = x.cuda(), y.cuda(), sw.cuda()
    w1 = ops.atom_cg_filter(torch.from_numpy(g[tag + "_w0"]).cuda(), x, y, sw, 0.1, it, act, 0.05, fr)
    assert _rel(w1, g[tag + "_w"]) < 1e-4
    w2 = ops.atom_cg_filter(w1, x, y, sw, 0.1, it, act, 0.05, fr)
    assert _rel(w2, g[tag + "_w2"]) < 1e-4
    w1b = ops.atom_cg_filter(torch.from_numpy(g[tag + "_w0"]).cuda(), x, y, sw, 0.1, it, act, 0.05, fr)
    assert torch.equal(w1, w1b)                      # fixed summation order: bitwise reproducible


def test_atom_cg_full_size(ops):
    """BASELINE size (ATOM memory 250 x 64 x 18 x 18, 5 PR-CG iterations, mlu 0.05): equals the oracle run on the filled
    slots (zero-weight slots contribute nothing), zero iterations is the identity, and the GN objective decreases."""
    from oracle import atom_oracle as A
    x, y, sw = synth.make_atom_memory(77, 250, 64, 18, 18, n_filled=24)
    w0 = torch.randn(1, 64, 4, 4, generator=torch.Generator().manual_seed(5)) * 0.02
    w = ops.atom_cg_filter(w0.cuda(), x.cuda(), y.cuda(), sw.cuda(), 0.1, 5, "mlu", 0.05, False)
    w_ref, _, _ = A.atom_cg_filter(w0, x[:24], y[:24], sw[:24], 0.1, 5, "mlu", 0.05, False)
    assert _rel(w, w_ref) < 1e-4
    assert torch.equal(ops.atom_cg_filter(w0.cuda(), x.cuda(), y.cuda(), sw.cuda(), 0.1, 0).cpu(), w0)

    def loss(wt):
        s = A.conv_same(x[:24], wt)
        r = sw[:24].view(-1, 1, 1, 1) * (A.activation(s, "mlu", 0.05) - y[:24]) ** 2
        return float(r.sum() + 0.1 * (wt ** 2).sum())
    assert loss(w.cpu()) < loss(w0)


def test_atom_stage2_ops(golden_dir, ops):
    """S1.3 / S2.2 / S2.3: feature normalisation, conv1x1 projection, conv2d 'same', Fourier upsampling."""
    from oracle import atom_oracle as A
    g = torch.Generator().manual_seed(9)
    x = torch.randn(5, 256, 18, 18, generator=g)
    xn = ops.feature_normalize_(x.clone().cuda(), 2.0)
    assert _rel(xn, A.feature_normalize(x, 2.0)) < 1e-5
    P = torch.randn(64, 256, 1, 1, generator=g) * 0.05
    proj = ops.conv1x1(xn, P.cuda())
    proj_ref = A.conv1x1(A.feature_normalize(x, 2.0), P)
    assert _rel(proj, proj_ref) < 1e-5
    w = torch.randn(1, 64, 4, 4, generator=g) * 0.1
    s = ops.conv2d_same(proj, w.cuda())
    assert s.shape == (5, 1, 18, 18)
    assert _rel(s, A.conv_same(proj_ref, w)) < 1e-5
    x22 = torch.randn(2, 32, 22, 22, generator=g)
    w22 = torch.randn(1, 32, 4, 4, generator=g)
    assert _rel(ops.conv2d_same(x22.cuda(), w22.cuda()), A.conv_same(x22, w22)) < 1e-5
    gf = np.load(os.path.join(golden_dir, "fourier.npz"))
    for tag, (S, H, ksz, osz) in {"s18_k4": (3, 18, 4, 288), "s18_k4_o72": (2, 18, 4, 72), "s17_k5": (2, 17, 5, 64), "s22_k4": (1, 22, 4, 352)}.items():
        up = ops.fourier_interp(torch.from_numpy(gf[tag + "_scores"]).cuda(), (ksz, ksz), (osz, osz))
        assert _rel(up, gf[tag + "_up"]) < 1e-4, tag
    # ATOM localisation at BASELINE size: 5 scales, arg-max on the 288x288 grid must agree with the oracle's arg-max
    up = ops.fourier_interp(s, (4, 4), (288, 288))
    up_ref = A.fourier_interp(A.conv_same(proj_ref, w), (4, 4), (288, 288))
    assert _rel(up, up_ref) < 1e-4
    mv, mi = ops.max2d(up[:, 0])
    from oracle import dimp_oracle as O
    mv_ref, mi_ref = O.max2d(up.cpu()[:, 0])
    assert torch.equal(mi.cpu(), mi_ref)


@pytest.mark.parametrize("B,C,H,W,R,ph,pw,scale,seed", [(2, 16, 18, 18, 6, 4, 4, 1.0 / 16, 1), (1, 32, 36, 36, 10, 5, 5, 1.0 / 8, 2),
                                                       (3, 8, 9, 11, 4, 3, 1, 0.9, 3)])
def test_prroi_all_three_kernels(ops, B, C, H, W, R, ph, pw, scale, seed):
    """PrRoIPool forward / backward / coordinate backward against the CPU restatement of the reference kernels."""
    from oracle import prroi_oracle as P
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, C, H, W, generator=g)
    ext_w, ext_h = W / scale, H / scale
    x1 = torch.rand(R, generator=g) * ext_w * 0.5
    y1 = torch.rand(R, generator=g) * ext_h * 0.5
    bw = (0.15 + 0.45 * torch.rand(R, generator=g)) * ext_w
    bh = (0.15 + 0.45 * torch.rand(R, generator=g)) * ext_h
    rois = torch.stack([torch.randint(0, B, (R,), generator=g).float(), x1, y1, x1 + bw, y1 + bh], 1).contiguous()
    rois[0, 3] = ext_w + 5.0                       # a box leaving the feature map: zero padding outside
    og = torch.randn(R, C, ph, pw, generator=g)
    out = ops.prroi_pool_forward(feat.cuda(), rois.cuda(), ph, pw, scale)
    out_ref = P.forward(feat.numpy(), rois.numpy(), ph, pw, scale)
    assert _rel(out, out_ref) < 1e-5
    fg = ops.prroi_pool_backward(feat.cuda(), rois.cuda(), out, og.cuda(), ph, pw, scale)
    assert _rel(fg, P.backward(feat.numpy(), rois.numpy(), og.numpy(), ph, pw, scale)) < 1e-5
    rg = ops.prroi_pool_coor_backward(feat.cuda(), rois.cuda(), out, og.cuda(), ph, pw, scale)
    rg_ref = P.coor_backward(feat.numpy(), rois.numpy(), out_ref, og.numpy(), ph, pw, scale)
    assert _rel(rg, rg_ref) < 1e-4
    # degenerate RoI (zero area): zero output and zero gradients, as the reference (win_size == 0)
    z = torch.tensor([[0, 5.0, 5.0, 5.0, 9.0]])
    assert float(ops.prroi_pool_forward(feat.cuda(), z.cuda(), ph, pw, scale).abs().max()) == 0.0


@pytest.mark.parametrize("tag,n,c,h,it,use_sw,thr,seed", [("n8_c64", 8, 64, 18, 4, True, 0.05, 71), ("n5_c32_22", 5, 32, 22, 3, False, -999.0, 72)])
def test_dimp_l2_sd_golden(golden_dir, ops, tag, n, c, h, it, use_sw, thr, seed):
    """DiMPL2SteepestDescentGN against the reference module's outputs (zero initial filter included: relu'(0) = 0)."""
    g = np.load(os.path.join(golden_dir, "dimp_l2_sd.npz"))
    feat = synth.make_clf_features(seed, n, c, h, h).cuda()
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda()
    sw = torch.from_numpy(g[tag + "_sw"]).cuda() if use_sw else None
    w, its, losses = ops.dimp_l2_sd_gn(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, sw, it, 1.3, thr, 0.9, max(0.1 ** 2, 1e-6),
                                       alpha_eps=0.01, return_iterates=True, compute_losses=True)
    assert _rel(its[1], g[tag + "_w1"][0]) < 1e-4
    assert _rel(w, g[tag + "_wfinal"]) < 1e-4
    assert np.allclose(losses.cpu().numpy(), g[tag + "_losses"], rtol=1e-4)


@pytest.mark.parametrize("tag,n,c,h,it,use_sw,thr,leak,act,seed", [("relu_n6_c64", 6, 64, 18, 4, True, 0.05, 0.0, "relu", 81),
                                                                  ("bent_n4_c32_22", 4, 32, 22, 3, False, 0.1, 0.1, "bentpar", 82)])
def test_gn_sd_hinge_golden(golden_dir, ops, tag, n, c, h, it, use_sw, thr, leak, act, seed):
    g = np.load(os.path.join(golden_dir, "gn_sd_hinge.npz"))
    feat = synth.make_clf_features(seed, n, c, h, h).cuda()
    sw = torch.from_numpy(g[tag + "_sw"]).cuda() if use_sw else None
    w, its, losses = ops.gn_sd_hinge(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, torch.from_numpy(g[tag + "_label"]).unsqueeze(1).cuda(),
                                     sw, it, 0.1, thr, leak, act, 0.7, 0.02, return_iterates=True, compute_losses=True)
    assert _rel(its[1], g[tag + "_w1"][0]) < 1e-4
    assert _rel(w, g[tag + "_wfinal"]) < 1e-4
    assert np.allclose(losses.cpu().numpy(), g[tag + "_losses"], rtol=1e-4)


TRANSFORMER_CASES = {"small": (64, 2, 128, 2, 2, 40, 2, 91, True), "tomp_l72": (256, 8, 2048, 6, 6, 72, 2, 92, True),
                     "tomp_l48_nomask": (256, 8, 2048, 6, 6, 48, 1, 93, False)}


def _transformer_inputs(d, L, B, seed, use_mask):
    g = torch.Generator().manual_seed(seed + 1)
    src = torch.randn(L, B, d, generator=g)
    pos = torch.randn(L, 1, d, generator=g) * 0.5
    qe = torch.randn(1, d, generator=g)
    mask = None
    if use_mask:
        mask = torch.zeros(B, L, dtype=torch.bool)
        mask[B - 1, L // 3: L // 2] = True
    return src, pos, qe, mask


@pytest.mark.parametrize("tag", sorted(TRANSFORMER_CASES))
def test_transformer_golden(golden_dir, tag):
    """ToMP Transformer.forward (6+6 post-norm layers) against the reference module's outputs."""
    from pytracking_b200.transformer_engine import TransformerEngine
    g = np.load(os.path.join(golden_dir, "transformer.npz"))
    d, nh, ff, ne, nd, L, B, seed, use_mask = TRANSFORMER_CASES[tag]
    sd = synth.make_transformer_state_dict(seed, d, nh, ff, ne, nd)
    src, pos, qe, mask = _transformer_inputs(d, L, B, seed, use_mask)
    eng = TransformerEngine(sd, L, B, d, nh, ff, ne, nd)
    hs, mem = eng.forward(src.cuda(), None if mask is None else mask.cuda(), qe.cuda(), pos.cuda())
    assert _rel(mem, g[tag + "_memory"]) < 1e-4
    assert _rel(hs, g[tag + "_hs"]) < 1e-4
    eng.close()


def test_transformer_tomp_size():
    """BASELINE ToMP size: 972 tokens x batch 2 ({cls, bbreg} stacked with the bbreg key-padding mask), d 256, 8 heads, FF 2048."""
    from oracle import tomp_oracle as T
    from pytracking_b200.transformer_engine import TransformerEngine
    d, nh, ff, ne, nd, L, B = 256, 8, 2048, 6, 6, 972, 2
    sd = synth.make_transformer_state_dict(95, d, nh, ff, ne, nd)
    g = torch.Generator().manual_seed(96)
    src = torch.randn(L, B, d, generator=g)
    pos = torch.randn(L, 1, d, generator=g) * 0.5
    qe = torch.randn(1, d, generator=g)
    mask = torch.zeros(B, L, dtype=torch.bool)
    mask[1, 324:648] = True                                  # filter_predictor.py:134-136 (one ground-truth frame)
    eng = TransformerEngine(sd, L, B, d, nh, ff, ne, nd)
    hs, mem = eng.forward(src.cuda(), mask.cuda(), qe.cuda(), pos.cuda())
    with torch.no_grad():
        hs_ref, mem_ref = T.transformer_forward(sd, src, mask, qe, pos, nh, ne, nd)
    assert _rel(mem, mem_ref) < 1e-4
    assert _rel(hs, hs_ref) < 1e-4
    hs2, mem2 = eng.forward(src.cuda(), mask.cuda(), qe.cuda(), pos.cuda())
    assert torch.equal(mem, mem2) and torch.equal(hs, hs2)
    eng.close()


ATOM_GN_CASES = {"n6_c32_16": (6, 32, 16, 3, 2, True, "mlu", 101), "n10_c64_32_pr": (10, 64, 32, 4, 3, False, "relu", 102)}


@pytest.mark.parametrize("tag", sorted(ATOM_GN_CASES))
def test_atom_gn_joint_golden(golden_dir, ops, tag):
    """ATOM first-frame joint optimisation (GaussNewtonCG on FactorizedConvProblem) against the reference classes' outputs."""
    g = np.load(os.path.join(golden_dir, "atom_gn.npz"))
    n, cin, cc, ncg, ngn, fr, act, seed = ATOM_GN_CASES[tag]
    x, y, sw = synth.make_atom_memory(seed, n, cin, 18, 18)
    w = torch.from_numpy(g[tag + "_w0"]).cuda().contiguous()
    P = torch.from_numpy(g[tag + "_P0"]).cuda().contiguous()
    ops.atom_gn_joint_(w, P, x.cuda(), y.cuda(), sw.cuda(), 0.1, 1e-2, ncg, ngn, act, 0.05, fr)
    assert _rel(w, g[tag + "_w"]) < 1e-4
    assert _rel(P, g[tag + "_P"]) < 1e-4


def test_atom_gn_joint_baseline_size(ops):
    """ATOM default init: 30 augmented samples x 256 channels -> 64, 6 GN x 10 CG iterations (atom/default.py:27-28)."""
    from oracle import atom_oracle as A
    x, y, sw = synth.make_atom_memory(111, 30, 256, 18, 18)
    g = torch.Generator().manual_seed(112)
    P0 = torch.randn(64, 256, 1, 1, generator=g) * (1.0 / 16)
    w0 = torch.zeros(1, 64, 4, 4)
    w, P = w0.clone().cuda(), P0.clone().cuda()
    ops.atom_gn_joint_(w, P, x.cuda(), y.cuda(), sw.cuda(), 0.1, 1e-4, 10, 6, "mlu", 0.05, True)
    w_ref, P_ref = A.atom_gn_joint(w0, P0, x, y, sw, 0.1, 1e-4, 10, 6, "mlu", 0.05, True)
    # (30 samples: well conditioned -- float32 oracle vs float64 oracle 8e-7; the kernel is 3e-6 from the float64 solution)
    w64, P64 = A.atom_gn_joint(w0.double(), P0.double(), x.double(), y.double(), sw.double(), 0.1, 1e-4, 10, 6, "mlu", 0.05, True)
    assert _rel(w, w64) < 2e-5 and _rel(P, P64) < 2e-5, (_rel(w, w64), _rel(P, P64))
    assert _rel(w, w_ref) < 2e-5 and _rel(P, P_ref) < 2e-5

    def loss(wt, Pt):
        s = A.conv_same(A.conv1x1(x, Pt), wt)
        return float((sw.view(-1, 1, 1, 1) * (A.activation(s, "mlu", 0.05) - y) ** 2).sum() + 0.1 * (wt ** 2).sum() + 1e-4 * (Pt ** 2).sum())
    l_gpu, l_ref, l0 = loss(w.cpu(), P.cpu()), loss(w_ref, P_ref), loss(w0, P0)
    assert l_gpu < 0.5 * l0 and abs(l_gpu - l_ref) < 1e-3 * l_ref


def test_plugin_mirror_reads_like_the_reference(golden_dir):
    """pytracking_b200.plugin: the reference call signatures (5-D feat, (weights, iterates, losses) returns) over the C ABI."""
    from pytracking_b200 import plugin
    g = np.load(os.path.join(golden_dir, "dimp_sd.npz"))
    tag, n, c, h, it, seed = "n15_it10", 15, 512, 18, 10, 21
    p = synth.make_dimp_optimizer_params(seed=seed)
    feat = synth.make_clf_features(seed, n, c, h, h).cuda().unsqueeze(1)                 # (images, sequences=1, C, H, W)
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda().unsqueeze(1)     # (images, sequences=1, 4)
    sw = torch.from_numpy(g[tag + "_sw"]).cuda().reshape(n, 1)
    opt = plugin.DiMPSteepestDescentGN(p["label_map_predictor.weight"], p["target_mask_predictor.0.weight"],
                                       p["spatial_weight_predictor.weight"], p["log_step_length"], p["filter_reg"], num_iter=5)
    weights, iterates, losses = opt(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, sample_weight=sw, num_iter=it, compute_losses=True)
    assert len(iterates) == it + 1 and len(losses) == it + 1 and iterates[0].shape == weights.shape
    assert _rel(weights, g[tag + "_wfinal"]) < 1e-4
    scores = plugin.apply_filter(feat, weights)
    assert scores.shape == (n, 1, 19, 19)
    mv, mi = plugin.max2d(scores[:, 0])
    assert mi.shape == (n, 2)
    gt = plugin.apply_feat_transpose(feat, scores, (4, 4), training=False)
    assert gt.shape == (1, c, 4, 4)
    with pytest.raises(NotImplementedError):
        plugin.apply_filter(torch.cat([feat, feat], 1), torch.cat([weights, weights], 0))      # two sequences: not claimed
    # ATOM optimiser objects update their variable in place, like the reference's run()
    x, y, swa = synth.make_atom_memory(52, 40, 64, 18, 18, n_filled=25)
    ga = np.load(os.path.join(golden_dir, "atom_cg.npz"))
    filt = torch.from_numpy(ga["n40_c64_pr_mlu_w0"]).cuda().contiguous()
    cg = plugin.ConjugateGradient(x.cuda(), y.cuda(), 0.1, swa.cuda(), filt, ("mlu", 0.05), fletcher_reeves=False)
    cg.run(5)
    assert _rel(filt, ga["n40_c64_pr_mlu_w"]) < 1e-4
    cg.run(5)
    assert _rel(filt, ga["n40_c64_pr_mlu_w2"]) < 1e-4


def test_dimp_tracker_trajectory_replay(golden_dir):
    """End to end inside a real tracker run: tests/golden/dimp_track.npz is a 12-frame trajectory of the UNMODIFIED reference
    DiMP tracker (oracle/gen_track_golden.py: dimp50 parameters, CPU, seeded random-init DiMP-50, no IoUNet). The frames are
    regenerated here, cropped with the bit-exact mirror of the reference's sample_patch, pushed through the host-buffer frame
    calls of the C ABI, and compared frame by frame: score maps (1e-4), arg-max cell (exact), filter after every online update."""
    from oracle import dimp_oracle as O
    from oracle import preprocessing_ref as pre
    from pytracking_b200.frame_engine import DiMPFrameEngine, SampleWeights
    g = np.load(os.path.join(golden_dir, "dimp_track.npz"))
    frames, init_bbox = synth.make_sequence(0, num_frames=12)
    assert np.allclose(init_bbox, g["init_bbox"])
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    eng = DiMPFrameEngine(sd, arch="resnet50", filter_size=4, memory_size=50, max_batch=1, crop_size=288, precision=0)
    sz = torch.from_numpy(g["img_sample_sz"])
    # ---- DiMP.initialize: one un-augmented sample, zero filter, net_opt_iter SD iterations ----
    im0 = pre.numpy_to_torch(frames[0])
    crop0 = pre.sample_init_patch(im0, torch.from_numpy(g["init_pos"]), float(g["init_scale"]), sz, float(g["aug_expansion_factor"]))
    eng.filter.zero_()
    eng.localize(crop0.contiguous().pin_memory())
    eng.update(0, 0, g["init_target_box"], np.array([1.0], dtype=np.float32), 1, int(g["init_num_iter"]))
    torch.cuda.synchronize()
    assert _rel(eng.filter, g["init_filter"]) < 1e-4
    swm = SampleWeights(50, 1, learning_rate=0.01, init_samples_minimum_weight=0.25)
    worst_s = worst_f = drift = 0.0
    prev_filter = g["init_filter"]
    for t in range(1, 13):
        k = "f%02d_" % t
        im = pre.numpy_to_torch(frames[t])
        crop, _ = pre.sample_patch_multiscale(im, torch.from_numpy(g[k + "crop_pos"]), [float(s) for s in g[k + "crop_scale"]], sz)
        # closed loop (our own evolving filter): the arg-max cell -- hence the tracker's box -- must be the reference's
        scores_cl, _, mi = eng.localize(crop.contiguous().pin_memory())
        ref = g[k + "scores"]
        _, mi_ref = O.max2d(torch.from_numpy(ref).reshape(1, 19, 19))
        assert mi.tolist() == mi_ref.tolist(), "frame %d: arg-max cell differs" % t
        drift = max(drift, _rel(scores_cl, ref.reshape(scores_cl.shape)))
        own_filter = eng.filter.clone()
        # open loop (the reference's filter of the previous frame): per-frame error of the hot path, free of the
        # frame-to-frame amplification of rounding noise that the CPU oracle shows as well (2e-5 -> 1.5e-3 over 12 frames)
        eng.filter.copy_(torch.from_numpy(prev_filter).cuda())
        scores, mv, _ = eng.localize(crop.contiguous().pin_memory())
        worst_s = max(worst_s, _rel(scores, ref.reshape(scores.shape)))
        if int(g[k + "updated"]):
            lr = float(g[k + "lr"])
            r = swm.step(None if lr < 0 else lr)
            n = int(g[k + "n_stored"])
            assert r == int(g[k + "replace_ind"]) and n == swm.num_stored
            assert np.allclose(swm.w[:n], g[k + "sample_weights"], rtol=1e-6, atol=1e-9)
            num_iter = 1 if lr >= 0 else 2
            eng.update(0, r, g[k + "target_box"].reshape(4), g[k + "sample_weights"], n, num_iter)
            torch.cuda.synchronize()
            worst_f = max(worst_f, _rel(eng.filter, g[k + "filter"]))
            prev_filter = g[k + "filter"]
            # continue the closed loop from our own filter
            from pytracking_b200 import ops as _ops
            luts = [sd["classifier.filter_optimizer." + q].cuda() for q in ("label_map_predictor.weight", "target_mask_predictor.0.weight",
                                                                           "spatial_weight_predictor.weight")]
            _ops.dimp_sd_gn(own_filter, eng.memory[:n], eng.boxes[:n], eng.sample_weights[:n], *luts, num_iter, eng.step_length,
                            eng.reg_weight, out=eng.filter)
    assert worst_s < 1e-4 and worst_f < 1e-4, (worst_s, worst_f)
    assert drift < 1e-2, drift
    eng.close()


def test_atom_tracker_trajectory_replay(golden_dir, ops):
    """BASELINE configs[0]: the UNMODIFIED reference ATOM tracker (ResNet-18, 5 scales, no IoUNet; oracle/gen_atom_track_golden.py)
    replayed through the engine: first-frame joint GN-CG optimisation, then per frame backbone -> p-norm -> projection -> conv 'same'
    -> Fourier upsampling -> arg-max, memory update and the CG filter update; open loop from the reference's previous filter."""
    from oracle import dimp_oracle as O
    from oracle import preprocessing_ref as pre
    from pytracking_b200.engine import BackboneEngine
    g = np.load(os.path.join(golden_dir, "atom_track.npz"))
    frames, init_bbox = synth.make_sequence(1, num_frames=8)
    assert np.allclose(init_bbox, g["init_bbox"])
    sd = synth.make_backbone_state_dict("resnet18", seed=5)
    sz = torch.from_numpy(g["img_sample_sz"])
    crop = int(sz[0])
    eng = BackboneEngine(sd, arch="resnet18", max_batch=5, crop_size=crop, precision=0, head=False)
    freg, preg = float(g["filter_reg"]), float(g["projection_reg"])
    osz = [int(v) for v in g["output_sz"]]

    def features(crops):
        x = eng.forward(crops.cuda().contiguous(), want=("layer3",))["layer3"]
        return ops.feature_normalize_(x, 2.0)

    # ---- ATOM.initialize: joint optimisation of filter and projection matrix on the un-augmented first-frame sample ----
    im0 = pre.numpy_to_torch(frames[0])
    crop0 = pre.sample_init_patch(im0, torch.from_numpy(g["init_pos"]), float(g["init_scale"]), sz, float(g["aug_expansion_factor"]))
    x0 = features(crop0)
    w = torch.from_numpy(g["init_w0"]).cuda().contiguous()
    P = torch.from_numpy(g["init_P0"]).cuda().contiguous()
    y0 = torch.from_numpy(g["init_y"]).cuda()
    ops.atom_gn_joint_(w, P, x0, y0, torch.ones(1, device="cuda"), freg, preg, int(g["init_num_cg"]), int(g["init_num_gn"]), "mlu", 0.05, True)
    # This single-sample, 60-iteration joint problem is ill-conditioned: in float64 a 1e-6 relative perturbation of the input features
    # moves the solution by 1.7e-3, the float32 oracle is 1e-2 away from the float64 oracle and the reference's own float32 autograd run
    # (the golden) 6e-3.  The bar is therefore the exact (float64) solution at the accuracy float32 itself reaches on this problem:
    # the GPU result must be as close to it as the two float32 references are, within a factor of 4 (same order of magnitude).
    from oracle import atom_oracle as AO
    x0c, w0c, P0c, y0c = x0.cpu(), torch.from_numpy(g["init_w0"]), torch.from_numpy(g["init_P0"]), y0.cpu()
    ncg0, ngn0 = int(g["init_num_cg"]), int(g["init_num_gn"])
    w64, P64 = AO.atom_gn_joint(w0c.double(), P0c.double(), x0c.double(), y0c.double(), torch.ones(1).double(), freg, preg, ncg0, ngn0, "mlu", 0.05, True)
    w32, P32 = AO.atom_gn_joint(w0c, P0c, x0c, y0c, torch.ones(1), freg, preg, ncg0, ngn0, "mlu", 0.05, True)
    fp32_w = max(_rel(w32, w64), _rel(g["init_w"], w64))
    fp32_P = max(_rel(P32, P64), _rel(g["init_P"], P64))
    print("ATOM first-frame GN-CG vs float64: GPU w %.2e P %.2e; float32 oracle / reference golden w %.2e P %.2e" %
          (_rel(w, w64), _rel(P, P64), fp32_w, fp32_P))
    assert _rel(w, w64) < 4 * fp32_w and _rel(P, P64) < 4 * fp32_P, (_rel(w, w64), fp32_w, _rel(P, P64), fp32_P)
    P_ref = torch.from_numpy(g["init_P"]).cuda()
    mem = torch.zeros(250, 64, 18, 18, device="cuda")
    ymem = torch.zeros(250, 1, 18, 18, device="cuda")
    mem[0] = ops.conv1x1(x0, P_ref)[0]
    ymem[0] = y0[0]
    prev_filter = torch.from_numpy(g["init_w"]).cuda()
    from oracle import atom_oracle as A
    worst_s = worst_f = worst_m = worst_l = worst_ref = 0.0
    per_frame = []
    for t in range(1, 9):
        k = "f%02d_" % t
        im = pre.numpy_to_torch(frames[t])
        crops, _ = pre.sample_patch_multiscale(im, torch.from_numpy(g[k + "crop_pos"]), [float(s) for s in g[k + "crop_scales"]], sz)
        proj = ops.conv1x1(features(crops), P_ref)
        scores = ops.conv2d_same(proj, prev_filter)
        worst_s = max(worst_s, _rel(scores, g[k + "scores_raw"]))
        up = ops.fourier_interp(scores, (4, 4), osz)
        mv, mi = ops.max2d(up[:, 0])
        assert np.array_equal(mi.cpu().numpy(), g[k + "up_maxidx"]), "frame %d: arg-max on the upsampled grid differs" % t
        worst_m = max(worst_m, _rel(mv, g[k + "up_maxval"]))
        scale_ind = int(np.argmax(g[k + "up_maxval"]))
        assert int(torch.argmax(mv)) == scale_ind
        if int(g[k + "updated"]):
            r = int(g[k + "replace_ind"])
            mem[r] = proj[scale_ind]
            ymem[r] = torch.from_numpy(g[k + "train_y"]).cuda()[0]
        sw = torch.from_numpy(g[k + "sample_weights"]).cuda() if int(g[k + "updated"]) else sw
        f = ops.atom_cg_filter(prev_filter, mem, ymem, sw, freg, int(g[k + "cg_iters"]), "mlu", 0.05, False)
        # With 2..9 stored samples and the MLU response the 5-step Polak-Ribiere CG of this trajectory is numerically unstable (its
        # rho sequence is not monotone; a 1e-5 relative perturbation of the samples moves the result by 1e-2).  As for the first-frame
        # problem the bar is the float64 solution at the accuracy float32 reaches: the kernel must be at least as close to it as
        # the float32 oracle and the reference's own float32 run (the golden) are, within a factor of 4.
        nz = torch.nonzero(sw > 0).reshape(-1)
        args64 = (prev_filter.double().cpu(), mem[nz].double().cpu(), ymem[nz].double().cpu(), sw[nz].double().cpu())
        f64 = A.atom_cg_filter(*args64, freg, int(g[k + "cg_iters"]), "mlu", 0.05, False)[0]
        f32 = A.atom_cg_filter(*[a.float() for a in args64], freg, int(g[k + "cg_iters"]), "mlu", 0.05, False)[0]
        e_gpu, e_ref = _rel(f, f64), max(_rel(f32, f64), _rel(g[k + "filter"], f64))
        per_frame.append((t, e_gpu, e_ref))
        worst_f = max(worst_f, e_gpu)
        worst_ref = max(worst_ref, e_ref)
        idx = torch.nonzero(sw > 0).reshape(-1)

        def objective(wt):
            sres = A.conv_same(mem[idx].cpu(), wt.cpu())
            return float((sw[idx].cpu().view(-1, 1, 1, 1) * (A.activation(sres, "mlu", 0.05) - ymem[idx].cpu()) ** 2).sum() + freg * (wt.cpu() ** 2).sum())
        l_ours, l_ref = objective(f), objective(torch.from_numpy(g[k + "filter"]))
        worst_l = max(worst_l, abs(l_ours - l_ref) / l_ref)
        prev_filter = torch.from_numpy(g[k + "filter"]).cuda()
    print("ATOM replay: scores %.1e, upsampled maxima %.1e; CG filter vs float64: GPU %.1e, float32 references %.1e; objective %.1e" %
          (worst_s, worst_m, worst_f, worst_ref, worst_l))
    print("  per frame (GPU vs f64, f32 references vs f64):", [(t, "%.1e" % a, "%.1e" % b) for t, a, b in per_frame])
    assert worst_s < 1e-4 and worst_m < 1e-4 and worst_l < 6e-2, (worst_s, worst_m, worst_l, worst_f)
    # per update: within a factor of 4 of that update's float32 references, or at least no worse than their worst over the trajectory
    assert all(a <= max(4 * b, worst_ref) + 1e-5 for _, a, b in per_frame) and worst_f <= 4 * worst_ref, per_frame
    eng.close()


def test_small_stage2_ops(ops):
    """softmax_reg (PrDiMP score pre-processing) and the 1x1 apply_filter path of the ToMP classifier."""
    from oracle import dimp_oracle as O
    from pytracking_b200 import plugin
    g = torch.Generator().manual_seed(3)
    s = torch.randn(5, 23 * 23, generator=g) * 3
    assert _rel(ops.softmax_reg(s.cuda(), None), torch.softmax(s, -1)) < 1e-5
    assert _rel(ops.softmax_reg(s.cuda(), -1.5), O.softmax_reg(s.reshape(5, 23, 23), -1.5).reshape(5, -1)) < 1e-5
    feat = torch.randn(3, 1, 256, 18, 18, generator=g)
    filt = torch.randn(1, 256, 1, 1, generator=g)
    ref = torch.matmul(filt.reshape(1, 1, 1, 256), feat.reshape(1, 3, 256, -1)).reshape(3, 1, 18, 18)     # filter.py:82-88
    assert _rel(plugin.apply_filter(feat.cuda(), filt.cuda()), ref) < 1e-5


@pytest.mark.parametrize("mode,n,c,h,it", [("dimp", 40, 128, 18, 3), ("prdimp", 9, 256, 22, 3), ("l2", 6, 128, 22, 3), ("hinge_relu", 7, 128, 18, 3),
                                           ("hinge_bent", 35, 256, 18, 2), ("dimp", 1, 512, 18, 2)])
def test_sd_tensor_core_kernel_matches_cuda_core_kernel(ops, monkeypatch, mode, n, c, h, it):
    """The tensor-core optimiser kernel (sd_tc.cu, B200TRK_SD_TC=1) and the CUDA-core kernel (sd_optimizer.cu, =0) implement the same four
    reference optimisers; the golden cases with C % 128 != 0 only reach the latter, so every mode is also compared kernel against kernel."""
    from pytracking_b200 import _lib
    g = torch.Generator().manual_seed(100 + n)
    feat = synth.make_clf_features(90 + n, n, c, h, h).cuda()
    bb = synth.make_boxes(91 + n, n, center=(h * 16) / 2 - 25).cuda()
    sw = torch.rand(n, generator=g) + 0.5
    sw = (sw / sw.sum()).cuda()
    w0 = (torch.randn(1, c, 4, 4, generator=g) * 0.01).cuda()
    p = synth.make_dimp_optimizer_params(seed=5)
    luts = [p[k].cuda() for k in ("label_map_predictor.weight", "target_mask_predictor.0.weight", "spatial_weight_predictor.weight")]
    lab = torch.rand(n, 1, h + 1, h + 1, generator=g).cuda()

    def run():
        if mode == "dimp":
            return ops.dimp_sd_gn(w0, feat, bb, sw, *luts, it, 0.9, 0.01, return_iterates=True, compute_losses=True)
        if mode == "prdimp":
            return ops.prdimp_sd_newton(w0, feat, bb, sw, it, 0.25, 1.0, 0.05 ** 2, alpha_eps=0.05, softmax_reg=-1.0, label_threshold=0.05,
                                        normalize_label=True, label_shrink=0.1, return_iterates=True, compute_losses=True)
        if mode == "l2":
            return ops.dimp_l2_sd_gn(w0, feat, bb, sw, it, 1.3, 0.05, 0.9, 0.01, alpha_eps=0.01, return_iterates=True, compute_losses=True)
        return ops.gn_sd_hinge(w0, feat, lab, sw, it, 0.1, 0.1, 0.1, "relu" if mode == "hinge_relu" else "bentpar", 0.7, 0.02,
                               return_iterates=True, compute_losses=True)

    res = {}
    for tag, tc in (("cuda", "0"), ("tc", "1")):
        monkeypatch.setenv("B200TRK_SD_TC", tc)
        w, its, losses = run()
        torch.cuda.synchronize()
        assert int(_lib.lib().b200trk_sd_last_kernel()) == (0 if tc == "0" else 1)
        res[tag] = (w.clone(), [x.clone() for x in its], losses.clone())
        w2, _, _ = run()
        assert torch.equal(w, w2), "%s: not deterministic" % tag
    for tag in ("tc",):
        assert _rel(res[tag][0], res["cuda"][0]) < 2e-5
        for a, b in zip(res[tag][1], res["cuda"][1]):
            assert _rel(a, b) < 2e-5
        assert np.allclose(res[tag][2].cpu().numpy(), res["cuda"][2].cpu().numpy(), rtol=2e-5)


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_softmax_reg_golden(golden_dir, ops, tag):
    g = np.load(os.path.join(golden_dir, "softmax_reg.npz"))
    x = torch.from_numpy(g[tag + "_x"])
    reg = None if np.isnan(g[tag + "_reg"][0]) else float(g[tag + "_reg"][0])
    y = ops.softmax_reg(x.reshape(x.shape[0], -1).cuda(), reg)
    assert _rel(y, g[tag + "_y"].reshape(x.shape[0], -1)) < 1e-5


def test_apply_filter_1x1_golden(G):
    """The reference's own 1x1 apply_filter output (ltr/models/layers/filter.py:60-88, corr.npz case c) through the plug-in mirror."""
    from pytracking_b200 import plugin
    g = G["corr"]
    feat = synth.make_clf_features(100 + ord("c"), 2, 32, 18, 18, filter_size=1)
    s = plugin.apply_filter(feat.unsqueeze(1).cuda(), torch.from_numpy(g["c_w"]).cuda())
    assert _rel(s, g["c_scores"].reshape(s.shape)) < 1e-5


# ---- parity holes named by the round-1 review ---------------------------------------------------------------------------------
def _rel_elem(a, b, floor=1e-3):
    """Element-wise relative error |a-b| / max(|b|, floor * max|b|) -- next to the global-norm `_rel` (north_star words the bar
    element-wise; entries far below the tensor's scale are compared against the floor, not against themselves)."""
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float(((a - b).abs() / b.abs().clamp(min=floor * float(b.abs().max()))).max())


def test_prdimp_sd_full_size_on_tensor_core_kernel_vs_oracle(ops, monkeypatch):
    """PrDiMP-50 at BASELINE configs[2] size (n = 50, C = 512, 22x22 features, 23x23 scores, 10 Newton iterations) on the tensor-core
    kernel against the CPU oracle (round 1 only compared the two CUDA kernels with each other at this size)."""
    from oracle import dimp_oracle as O
    monkeypatch.setenv("B200TRK_SD_TC", "1")
    feat = synth.make_clf_features(91, 50, 512, 22, 22)
    bb = synth.make_boxes(92, 50, center=(22 * 16) / 2 - 25)
    sw = torch.rand(50, generator=torch.Generator().manual_seed(93)) + 0.2
    sw = sw / sw.sum()
    w0 = 0.01 * torch.randn(1, 512, 4, 4, generator=torch.Generator().manual_seed(94))
    sigma = 0.25 * 22 / 5        # output_sigma_factor * feature_sz / search_area_scale (ltr/train_settings/dimp/prdimp50.py)
    kw = dict(alpha_eps=0.05, softmax_reg=None, label_threshold=0.0, normalize_label=True, label_shrink=0.0)
    w, its, losses = ops.prdimp_sd_newton(w0.cuda(), feat.cuda(), bb.cuda(), sw.cuda(), 10, sigma, 1.0, 0.05 ** 2,
                                          return_iterates=True, compute_losses=True, **kw)
    from pytracking_b200 import _lib
    assert _lib.lib().b200trk_sd_last_kernel() == 1
    w_ref, its_ref, l_ref = O.prdimp_sd_newton(w0, feat, bb, sw, torch.zeros(1), torch.tensor([0.05]), 10, sigma, min_filter_reg=0.05,
                                               alpha_eps=0.05, softmax_reg_val=None, label_threshold=0.0, normalize_label=True,
                                               label_shrink=0.0)
    assert _rel(w, w_ref) < 1e-4, _rel(w, w_ref)
    assert _rel_elem(w, w_ref) < 1e-3, _rel_elem(w, w_ref)
    assert _rel(its[1], its_ref[1]) < 1e-4
    assert np.allclose(losses.cpu().numpy(), [float(x) for x in l_ref], rtol=1e-4)


@pytest.mark.parametrize("precision", [0, 1])
def test_backbone_resnet101_vs_oracle(precision):
    """ResNet-101 to layer3 (the ToMP-101 backbone, ltr/models/backbone/resnet.py:281-291): declared in round 1, never run."""
    from oracle import dimp_oracle as O
    from pytracking_b200.engine import BackboneEngine
    sd = synth.make_backbone_state_dict("resnet101", seed=4)
    im = synth.make_crop(9, 1, 96)
    eng = BackboneEngine(sd, arch="resnet101", max_batch=1, crop_size=96, precision=precision, head=False)
    out = eng.forward(im.cuda(), want=("layer2", "layer3"))
    with torch.no_grad():
        ref = O.resnet_forward(sd, O.preprocess_image(im), "resnet101")
    for l in ("layer2", "layer3"):
        assert _rel(out[l], ref[l]) < 1e-4, (l, _rel(out[l], ref[l]))
        assert _rel_elem(out[l], ref[l], 1e-2) < 1e-3, (l, _rel_elem(out[l], ref[l], 1e-2))
    assert abs(eng.flops / 2 / 1e6 - 11555.2 * (96 / 288) ** 2) < 0.02 * 11555.2 * (96 / 288) ** 2       # SURVEY 8(a): 11 555.2 MMAC @ 288^2
    eng.close()


def test_elementwise_relative_error_of_the_frame_stages(ops):
    """The element-wise form of the 1e-4 / 1e-3 bar on the three stages at BASELINE configs[1] size (global-norm checks above)."""
    from oracle import dimp_oracle as O
    from pytracking_b200.engine import BackboneEngine
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    im = synth.make_crop(21, 1, 288)
    eng = BackboneEngine(sd, arch="resnet50", max_batch=1, crop_size=288)
    clf = eng.forward(im.cuda(), want=("classification",))["classification"]
    with torch.no_grad():
        clf_ref = O.clf_head_dimp50(sd, O.resnet_forward(sd, O.preprocess_image(im), "resnet50", output_layers=("layer3",))["layer3"])
    e_clf = _rel_elem(clf, clf_ref, 1e-2)
    w = 0.02 * torch.randn(1, 512, 4, 4, generator=torch.Generator().manual_seed(5))
    s = ops.apply_filter(clf, w.cuda())
    e_s = _rel_elem(s, O.apply_filter(clf_ref, w), 1e-2)
    print("element-wise relative error (floor 1e-2 of the max): clf features %.2e, score map %.2e" % (e_clf, e_s))
    assert e_clf < 1e-3 and e_s < 1e-3
    eng.close()
