"""How `pytracking_b200.plugin.install()` binds its seams: exactly the attributes below, each restored to the identical object by
`uninstall()`; `skip=` in both forms; a second `install()` is a no-op; an optional module that does not import leaves every other
seam bound; a call the CUDA path does not claim reaches the reference with the caller's own arguments; the DiMP-L2 optimiser seam
builds its mirror from the reference module.  Only the last test needs a GPU."""
import importlib
import inspect
import os
import sys
import types

import numpy as np
import pytest
import torch

from baseline import ref_env

pytestmark = pytest.mark.skipif(not ref_env.reference_available(), reason="reference tree not staged (baseline/_ref)")

_PRROI = "ltr.external.PreciseRoIPooling.pytorch.prroi_pool.functional"
# (module, owner class or None for the module itself, attribute), in binding order
BOUND = [
    ("ltr.models.layers.filter", None, "apply_filter"),
    ("ltr.models.layers.filter", None, "apply_feat_transpose"),
    ("pytracking.libs.dcf", None, "max2d"),
    ("ltr.models.target_classifier.optimizer", "DiMPSteepestDescentGN", "forward"),
    ("ltr.models.target_classifier.optimizer", "PrDiMPSteepestDescentNewton", "forward"),
    ("ltr.models.target_classifier.optimizer", "DiMPL2SteepestDescentGN", "forward"),
    ("ltr.models.meta.steepestdescent", "GNSteepestDescent", "forward"),
    ("pytracking.features.net_wrappers", "NetWithBackbone", "extract_backbone"),
    ("ltr.models.tracking.dimpnet", "DiMPnet", "extract_classification_feat"),
    ("ltr.models.transformer.heads", "Head", "extract_head_feat"),
    ("ltr.models.transformer.heads", "DenseBoxRegressor", "forward"),
    ("ltr.models.transformer.filter_predictor", "FilterPredictor", "predict_cls_bbreg_filters_parallel"),
    ("ltr.models.bbreg.atom_iou_net", "AtomIoUNet", "get_iou_feat"),
    ("ltr.models.bbreg.atom_iou_net", "AtomIoUNet", "predict_iou"),
    (_PRROI, None, "_prroi_pooling"),
    (_PRROI, None, "_import_prroi_pooling"),
    ("pytracking.libs.operation", None, "conv2d"),
    ("pytracking.libs.operation", None, "conv1x1"),
    ("pytracking.libs.optimization", "ConjugateGradient", "run"),
    ("pytracking.libs.optimization", "GaussNewtonCG", "run"),
    ("pytracking.tracker.eco.optim", "FilterOptim", "run"),
    ("pytracking.tracker.eco.eco", "ECO", "apply_filter"),
    ("pytracking.tracker.eco.eco", "ECO", "preprocess_sample"),
    ("pytracking.tracker.eco.eco", None, "fourier"),
    ("ltr.models.transformer.transformer", "Transformer", "forward"),
]


def _owner(module, owner):
    m = importlib.import_module(module)
    return getattr(m, owner) if owner else m


def _value(module, owner, name):
    o = _owner(module, owner)
    return vars(o)[name] if isinstance(o, type) else getattr(o, name)


def _name(module, owner, name):
    return "%s.%s" % (owner or module, name)


@pytest.fixture()
def plugin():
    from oracle import ref_shims
    ref_shims.install(prroi_cpu=False)
    from pytracking_b200 import plugin as p
    p.uninstall()
    yield p
    p.uninstall()


def test_install_binds_exactly_these_attributes_and_uninstall_restores_each(plugin):
    before = [_value(*b) for b in BOUND]
    assert plugin.install() == [_name(*b) for b in BOUND]
    for b, orig in zip(BOUND, before):
        new = _value(*b)
        assert new is not orig, b
        if b[1] is not None:                                  # bound on a class: a real function, so that it binds as a method
            assert inspect.isfunction(new), b
    plugin.uninstall()
    for b, orig in zip(BOUND, before):
        assert _value(*b) is orig, b


def test_skip_in_both_forms_and_install_twice(plugin):
    skip = ("predict_iou", "DiMPSteepestDescentGN.forward", "ltr.models.layers.filter.apply_filter")
    kept = [BOUND[0], BOUND[3], BOUND[13]]
    before = {b: _value(*b) for b in kept}
    names = plugin.install(skip=skip)
    assert names == [_name(*b) for b in BOUND if b not in kept]
    for b in kept:
        assert _value(*b) is before[b], b
    bound = [_value(*b) for b in BOUND]
    assert plugin.install() == names                          # no rebinding, whatever the arguments
    assert all(_value(*b) is v for b, v in zip(BOUND, bound))


@pytest.mark.parametrize("module", ["pytracking.tracker.eco.optim", "pytracking.tracker.eco.eco", "ltr.models.meta.steepestdescent"])
def test_an_optional_module_that_does_not_import_leaves_every_other_seam_bound(plugin, monkeypatch, module):
    plugin.install()                                          # every module imported once, so that only `module` fails below
    plugin.uninstall()
    monkeypatch.setitem(sys.modules, module, None)            # `import module` raises ImportError
    assert plugin.install() == [_name(*b) for b in BOUND if b[0] != module]


def test_fall_through_hands_the_reference_the_callers_arguments(plugin, monkeypatch):
    calls = []

    def recorder(*args, **kwargs):
        calls.append((args, kwargs))
        return "reference"

    targets = [("ltr.models.layers.filter", None, "apply_filter"), ("pytracking.libs.dcf", None, "max2d"),
               ("pytracking.libs.operation", None, "conv2d"), ("pytracking.libs.optimization", "GaussNewtonCG", "run"),
               ("ltr.models.transformer.transformer", "Transformer", "forward"), ("ltr.models.transformer.heads", "Head", "extract_head_feat")]
    for b in targets:
        monkeypatch.setattr(_owner(*b[:2]), b[2], recorder)
    plugin.install()
    try:
        _call_unclaimed(plugin, calls)
    finally:
        plugin.uninstall()                                    # before monkeypatch puts the originals back


def _call_unclaimed(plugin, calls):
    import ltr.models.layers.filter as fl
    import ltr.models.transformer.heads as hd
    import ltr.models.transformer.transformer as tr
    import pytracking.libs.dcf as dcf
    import pytracking.libs.operation as op
    import pytracking.libs.optimization as oz
    feat, filt = torch.zeros(3, 1, 32, 18, 18), torch.zeros(1, 32, 4, 4)          # CPU tensors: not claimed
    not_claimed = types.SimpleNamespace(training=True, problem=object())
    served = dict(plugin.stats)
    cases = [(fl.apply_filter, (feat, filt), {"dilation_factors": None}),
             (dcf.max2d, (feat[:, 0, 0],), {}),
             (op.conv2d, (feat[:, 0], filt), {"mode": "same"}),
             (oz.GaussNewtonCG.run, (not_claimed, 3), {"num_gn_iter": 2}),
             (tr.Transformer.forward, (not_claimed, feat, None), {"query_embed": filt, "pos_embed": None}),
             (hd.Head.extract_head_feat, (not_claimed, feat[:, 0]), {"num_sequences": 1})]
    for fn, args, kwargs in cases:
        calls.clear()
        assert fn(*args, **kwargs) == "reference"
        assert len(calls) == 1 and len(calls[0][0]) == len(args) and all(a is b for a, b in zip(calls[0][0], args))
        assert calls[0][1].keys() == kwargs.keys() and all(calls[0][1][k] is v for k, v in kwargs.items())
    assert plugin.stats == served


def test_head_feature_memo(plugin, monkeypatch):
    """Head.extract_head_feat of a tensor the CUDA path would claim: the first call runs the reference (not counted), later calls on
    the unchanged tensor return the kept feature (counted under "(cached)"), a changed tensor runs the reference again."""
    calls = []

    def reference(self, feat, num_sequences=None):
        calls.append(num_sequences)
        out = feat * 2
        return out if num_sequences is None else out.reshape(-1, num_sequences, *out.shape[-3:])

    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    plugin.install()
    head, feat = type("Head", (), {"training": False})(), torch.ones(4, 8, 3, 3)           # weakly referenceable, as a module is
    before = plugin.stats.get("Head.extract_head_feat(cached)", 0)
    with torch.no_grad():
        first = plugin.head_extract_head_feat(reference, head, feat, num_sequences=2)
        again = plugin.head_extract_head_feat(reference, head, feat)
        feat.add_(1)
        changed = plugin.head_extract_head_feat(reference, head, feat, 2)
    assert calls == [2, 2] and plugin.stats.get("Head.extract_head_feat(cached)", 0) == before + 1
    assert first.shape == (2, 2, 8, 3, 3) and torch.equal(again, first.reshape(4, 8, 3, 3)) and torch.equal(changed.reshape(4, 8, 3, 3), 2 * feat)


def test_dimp_l2_mirror_is_built_from_the_reference_module(plugin):
    import ltr.models.target_classifier.optimizer as opt
    m = opt.DiMPL2SteepestDescentGN(num_iter=3, feat_stride=8, init_step_length=0.9, gauss_sigma=1.3, hinge_threshold=0.05,
                                    init_filter_reg=0.1, min_filter_reg=1e-3, alpha_eps=0.01)
    mirror = plugin.DiMPL2SteepestDescentGN.from_module(m)
    assert mirror.step_length == pytest.approx(0.9, rel=1e-6) and mirror.reg_weight == pytest.approx(0.01, rel=1e-6)
    assert (mirror.num_iter, mirror.feat_stride, mirror.gauss_sigma, mirror.hinge_threshold, mirror.alpha_eps) == (3, 8, 1.3, 0.05, 0.01)
    m = opt.DiMPL2SteepestDescentGN(init_filter_reg=1e-4, min_filter_reg=1e-3)
    assert plugin.DiMPL2SteepestDescentGN.from_module(m).reg_weight == pytest.approx(1e-6, rel=1e-6)      # clamp(min=min_filter_reg**2)
    m.detach_length = 0
    with pytest.raises(NotImplementedError):
        plugin.DiMPL2SteepestDescentGN.from_module(m)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu().reshape(-1), torch.as_tensor(b).double().cpu().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("tag,n,c,h,it,use_sw,thr,seed", [("n8_c64", 8, 64, 18, 4, True, 0.05, 71), ("n5_c32_22", 5, 32, 22, 3, False, -999.0, 72)])
def test_reference_dimp_l2_module_above_the_engine(plugin, golden_dir, tag, n, c, h, it, use_sw, thr, seed):
    """The reference DiMPL2SteepestDescentGN module on CUDA with `install()` in place is served by the library and matches the
    reference's own outputs (tests/golden/dimp_l2_sd.npz, oracle/gen_golden.py) at the bars of test_gpu_parity's golden test."""
    import ltr.models.target_classifier.optimizer as opt
    from pytracking_b200 import synth
    g = np.load(os.path.join(golden_dir, "dimp_l2_sd.npz"))
    m = opt.DiMPL2SteepestDescentGN(num_iter=it, feat_stride=16, init_step_length=0.9, gauss_sigma=1.3, hinge_threshold=thr,
                                    init_filter_reg=0.1, min_filter_reg=1e-3, alpha_eps=0.01).cuda().eval()
    feat = synth.make_clf_features(seed, n, c, h, h).cuda().unsqueeze(1)
    bb = synth.make_boxes(seed + 1, n, center=(h * 16) / 2 - 25).cuda().unsqueeze(1)
    sw = torch.from_numpy(g[tag + "_sw"]).cuda().unsqueeze(1) if use_sw else None
    plugin.install()
    before = plugin.stats.get("DiMPL2SteepestDescentGN.forward", 0)
    with torch.no_grad():
        w, its, losses = m(torch.from_numpy(g[tag + "_w0"]).cuda(), feat, bb, sample_weight=sw, num_iter=it, compute_losses=True)
    assert plugin.stats.get("DiMPL2SteepestDescentGN.forward", 0) == before + 1
    assert _rel(its[1], g[tag + "_w1"]) < 1e-4
    assert _rel(w, g[tag + "_wfinal"]) < 1e-4
    assert np.allclose(torch.stack(losses).cpu().numpy(), g[tag + "_losses"], rtol=1e-4)
