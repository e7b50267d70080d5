"""TEST INFRASTRUCTURE ONLY -- records what the IoUNet and ToMP-head parity tests compare against, from the UNMODIFIED reference
modules run on the CPU with seeded weights and inputs (tests/ref_weights.py):

    python -m oracle.gen_iou_tomp_golden       (needs a reference checkout: baseline/_ref or PYTRACKING_REFERENCE)

-> tests/golden/iou_tomp_ref.npz:
  iou_keys / iou_shapes, tower_keys / tower_shapes, tok{0,1}_keys / _shapes   module layouts (AtomIoUNet, DenseBoxRegressor, FilterPredictor)
  feat_c3 / feat_c4 (+ _idx, _amax)      AtomIoUNet.get_iou_feat on the layer2 / layer3 features of two synthetic crops (sampled)
  piou_<seed>_iou / _grad                 predict_iou and its autograd box gradient (oracle PrRoIPool), seeds 0 / 1 / 2
  refine_<iters>_<rel>_boxes / _iou       DiMP.optimize_boxes (default / relative space) for the iteration counts the tests run
  tower_out                               DenseBoxRegressor.forward
  tok<use_test>_feat (+ _idx, _amax), tok<use_test>_mask   the tokens FilterPredictor hands to its transformer (sampled)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

REFINE = ((5, 1.0, False), (10, 2.5e-3, True), (3, 1.0, False), (4, 5e-3, True))     # (iterations, step length, relative space)


def _sampled(rec, name, t):
    a = t.detach().double().numpy().reshape(-1)
    idx = ref_weights.sample_index(a.size)
    rec[name] = a[idx].astype(np.float32)
    rec[name + "_idx"] = idx
    rec[name + "_amax"] = np.float64(np.abs(a).max())


def main():
    from oracle import ref_shims
    ref_shims.install()
    torch.set_num_threads(8)
    from baseline import ref_tracker
    from pytracking import TensorList
    from pytracking.tracker.dimp.dimp import DiMP
    from pytracking.utils import TrackerParams
    import ltr.models.transformer.filter_predictor as fp
    import ltr.models.transformer.heads as heads
    from pytracking_b200 import synth
    rec = {}

    # ---- IoUNet ----
    net = ref_tracker.build_dimp_net("resnet50", seed=0)
    rec["iou_keys"], rec["iou_shapes"] = ref_weights.layout_arrays(net.bb_regressor.state_dict())
    missing, unexpected = net.load_state_dict(ref_weights.iou_state_dict(rec), strict=False)
    assert not unexpected and all(k.startswith(("feature_extractor.layer4", "feature_extractor.fc")) for k in missing), (missing, unexpected)
    net.eval()
    im = synth.make_crop(3, 2, 288)
    with torch.no_grad():
        x = (im / 255 - torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)) / torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
        bf = net.extract_backbone_features(x)
        c3, c4 = net.bb_regressor.get_iou_feat([bf["layer2"], bf["layer3"]])
    _sampled(rec, "feat_c3", c3)
    _sampled(rec, "feat_c4", c4)
    for seed, R in ((0, 10), (1, 1), (2, 16)):
        mod, feat, boxes = ref_weights.iou_inputs(seed, R)
        bb = boxes.clone().requires_grad_(True)
        iou = net.bb_regressor.predict_iou(mod, feat, bb)
        iou.backward(gradient=torch.ones_like(iou))
        rec["piou_%d_iou" % seed], rec["piou_%d_grad" % seed] = iou.detach().numpy(), bb.grad.numpy()
    for iters, step, relative in REFINE:
        mod, feat, boxes = ref_weights.iou_inputs(7, 10)
        p = TrackerParams()
        p.device = "cpu"
        p.box_refinement_iter, p.box_refinement_step_length, p.box_refinement_step_decay = iters, step, 1
        p.box_refinement_space = "relative" if relative else "default"
        trk = DiMP.__new__(DiMP)
        trk.params = p
        trk.net = type("N", (), {"bb_regressor": net.bb_regressor})()
        trk.iou_modulation = TensorList(mod)
        b, i = trk.optimize_boxes(TensorList(feat), boxes.reshape(-1, 4).clone())
        rec["refine_%d_%d_boxes" % (iters, relative)], rec["refine_%d_%d_iou" % (iters, relative)] = b.numpy(), i.numpy()

    # ---- ToMP box-regression tower ----
    m = heads.DenseBoxRegressor(num_channels=256).eval()
    rec["tower_keys"], rec["tower_shapes"] = ref_weights.layout_arrays(m.state_dict())
    m.load_state_dict(ref_weights.tower_state_dict(rec))
    feat, filt = ref_weights.tower_inputs()
    with torch.no_grad():
        rec["tower_out"] = m(feat, filt)[0].numpy()                                  # [1, 4, 18, 18]

    # ---- ToMP token assembly ----
    for use_test in (0, 1):
        captured = {}

        class FakeTransformer(torch.nn.Module):
            d_model = 256

            def forward(self, feat, mask=None, query_embed=None, pos_embed=None):
                captured["feat"], captured["mask"] = feat.clone(), mask
                return torch.zeros(1, 1, feat.shape[1], 256), torch.zeros_like(feat)
        m = fp.FilterPredictor(FakeTransformer(), feature_sz=18, use_test_frame_encoding=bool(use_test)).eval()
        keys, shapes = ref_weights.layout_arrays(m.state_dict())
        rec["tok%d_keys" % use_test], rec["tok%d_shapes" % use_test] = keys, shapes
        m.load_state_dict(ref_weights.token_state_dict(rec, use_test))
        train_feat, test_feat, label, ltrb = ref_weights.token_inputs()
        with torch.no_grad():
            m.predict_cls_bbreg_filters_parallel(train_feat, test_feat, label, 1, ltrb)
        _sampled(rec, "tok%d_feat" % use_test, captured["feat"])                    # [972, 2, 256]
        rec["tok%d_feat_shape" % use_test] = np.array(captured["feat"].shape)
        rec["tok%d_mask" % use_test] = captured["mask"].numpy()

    np.savez_compressed(ref_weights.GOLDEN, **rec)
    print(ref_weights.GOLDEN, os.path.getsize(ref_weights.GOLDEN), "bytes")


import ref_weights  # noqa: E402  (tests/ on sys.path above)

if __name__ == "__main__":
    main()
