"""TEST INFRASTRUCTURE ONLY -- a restatement of FilterInitializerLinear.forward (ltr/models/target_classifier/initializer.py:9-44,
118-173) in float64 (or float32), pinned to tests/golden/filter_init.npz by tests/test_filter_init_cpu.py:
    weights = mean_i PrRoIPool_{k x k, 1/16}( conv_{k_c x k_c, pad k_c // 2}(feat_i) + bias, box_i )   [/ (C k k) with filter_norm]
with PrRoIPool from oracle/prroi_oracle.py (float64) and pool_square's square box of equal area around the box centre."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import prroi_oracle


def rois(boxes, images=None, pool_square=False):
    """boxes [n,4] (x, y, w, h) -> PrRoIPool RoIs [n,5] (image, x0, y0, x1, y1), float64."""
    b = np.asarray(boxes, dtype=np.float64).reshape(-1, 4).copy()
    if pool_square:
        s = np.sqrt(b[:, 2] * b[:, 3])
        b[:, 0] += b[:, 2] / 2 - s / 2
        b[:, 1] += b[:, 3] / 2 - s / 2
        b[:, 2] = b[:, 3] = s
    img = np.arange(b.shape[0]) if images is None else np.asarray(images)
    return np.stack([img.astype(np.float64), b[:, 0], b[:, 1], b[:, 0] + b[:, 2], b[:, 1] + b[:, 3]], 1)


def filter_init(weight, bias, feat, boxes, images=None, filter_size=4, filter_norm=False, pool_square=False, dtype=torch.float64):
    """weight [C,C,k,k], bias [C], feat [S,C,H,W] (torch), boxes [n,4] -> filter [1,C,filter_size,filter_size] float64 numpy.  dtype is
    the precision of the convolution; the pooling and the mean are float64."""
    k = weight.shape[-1]
    x = F.conv2d(feat.to(dtype), weight.to(dtype), bias.to(dtype), padding=k // 2)
    pooled = prroi_oracle.forward(x.double().numpy(), rois(boxes, images, pool_square), filter_size, filter_size, 1.0 / 16)
    w = pooled.mean(0, keepdims=True)
    if filter_norm:
        w = w / (w.shape[1] * filter_size * filter_size)
    return w
