"""Seeded weights and inputs shared by the IoUNet / ToMP parity tests and the recorder of their reference outputs
(oracle/gen_iou_tomp_golden.py -> tests/golden/iou_tomp_ref.npz).  The module layouts (state-dict keys and shapes of the reference's
AtomIoUNet, DenseBoxRegressor and FilterPredictor) are stored in the golden file, so the tests rebuild the exact weights the reference
ran with, without the reference."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "iou_tomp_ref.npz")


def layout_arrays(sd):
    """{key: tensor} -> (keys, shapes) arrays for the golden file (shapes padded with -1 to rank 4)."""
    keys = sorted(sd)
    shapes = np.full((len(keys), 4), -1, dtype=np.int64)
    for i, k in enumerate(keys):
        s = tuple(sd[k].shape)
        shapes[i, :len(s)] = s
    return np.array(keys), shapes


def seeded_state_dict(keys, shapes, seed, prefix=""):
    """Weights for a (keys, shapes) layout from one seeded generator, in key order: weights of rank >= 2 ~ U(-1, 1) / sqrt(fan_in) (the
    default initialisation of torch's convolution and linear layers, which the reference's constructors use), rank-1
    `weight` (BatchNorm / GroupNorm scale) U[0.8, 1.2], `bias` 0.05 N(0, 1), `running_mean` 0.05 N(0, 1), `running_var` U[0.7, 1.3]."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, s in zip(keys, shapes):
        k = str(k)
        shape = tuple(int(v) for v in s if v >= 0)
        if k.endswith("num_batches_tracked"):
            sd[prefix + k] = torch.tensor(0, dtype=torch.long)
        elif len(shape) >= 2:
            fan_in = int(np.prod(shape[1:]))
            sd[prefix + k] = (2 * torch.rand(shape, generator=g) - 1) / fan_in ** 0.5
        elif k.endswith("running_var"):
            sd[prefix + k] = 0.7 + 0.6 * torch.rand(shape, generator=g)
        elif k.endswith("weight"):
            sd[prefix + k] = 0.8 + 0.4 * torch.rand(shape, generator=g)
        else:
            sd[prefix + k] = 0.05 * torch.randn(shape, generator=g)
    return sd


def iou_state_dict(gold):
    """The DiMP-50 network the IoUNet tests run: the synthetic backbone + classifier of pytracking_b200.synth and a seeded IoUNet
    (`bb_regressor.*`), its predictor scaled so that box gradients are O(1e-2) and the refinement loops move boxes by pixels."""
    from pytracking_b200 import synth
    sd = synth.make_dimp_state_dict("resnet50", seed=0, lut_seed=3)
    sd.update(seeded_state_dict(gold["iou_keys"], gold["iou_shapes"], 5, prefix="bb_regressor."))
    sd["bb_regressor.iou_predictor.weight"] = sd["bb_regressor.iou_predictor.weight"] * 20.0
    return sd


def iou_inputs(seed, R):
    """Modulation vectors, IoU features (layer2-like 36x36, layer3-like 18x18) and R proposal boxes [1, R, 4] (x, y, w, h)."""
    g = torch.Generator().manual_seed(seed)
    f3 = torch.relu(torch.randn(1, 256, 36, 36, generator=g))
    f4 = torch.relu(torch.randn(1, 256, 18, 18, generator=g))
    mod = [torch.randn(1, 256, 1, 1, generator=g).abs(), torch.randn(1, 256, 1, 1, generator=g).abs()]
    c = torch.tensor([120.0, 130.0]) + 30 * (torch.rand(R, 2, generator=g) - 0.5)
    sz = torch.tensor([70.0, 55.0]) * (0.6 + 0.8 * torch.rand(R, 2, generator=g))
    return mod, [f3, f4], torch.cat([c - sz / 2, sz], 1).reshape(1, R, 4)


def token_state_dict(gold, use_test):
    """FilterPredictor weights; `query_embed_fg_decoder` is the same parameter as `query_embed_fg` in the module, so its key gets the
    same value."""
    sd = seeded_state_dict(gold["tok%d_keys" % use_test], gold["tok%d_shapes" % use_test], 8 + use_test)
    sd["query_embed_fg_decoder.weight"] = sd["query_embed_fg.weight"]
    return sd


def tower_state_dict(gold):
    sd = seeded_state_dict(gold["tower_keys"], gold["tower_shapes"], 4)
    sd["bbreg_layer.weight"] = sd["bbreg_layer.weight"] * 0.3
    return sd


def tower_inputs():
    g = torch.Generator().manual_seed(14)
    return torch.randn(1, 1, 256, 18, 18, generator=g) * 0.3, torch.randn(1, 256, 1, 1, generator=g) * 0.2


def token_inputs():
    g = torch.Generator().manual_seed(18)
    return (torch.randn(2, 1, 256, 18, 18, generator=g), torch.randn(1, 1, 256, 18, 18, generator=g), torch.rand(2, 1, 18, 18, generator=g),
            torch.rand(2, 1, 4, 18, 18, generator=g))


def sample_index(n, count=16384, seed=0):
    """A fixed, sorted sample of flat indices into an array of n elements (all of them when n <= count)."""
    if n <= count:
        return np.arange(n)
    return np.sort(np.random.RandomState(seed).choice(n, count, replace=False))
