"""Restatement of the first-frame augmentation DiMP.initialize applies (pytracking/features/augmentation.py; generate_init_samples,
pytracking/tracker/dimp/dimp.py:331-398) in numpy, without cv2 -- what csrc/augment_kernels.cuh must reproduce.

Images are float32 [C, H, W] (the expanded patch).  Every transform ends with Transform.crop_to_output, F.pad(..., 'replicate')
with pads floor / ceil((out - in) / 2) -/+ shift: a crop whose indices are clamped to the image.
  * rotate: cv.warpAffine(HWC image, [R, c - R c], BORDER_REPLICATE) as cv2 executes it on float32 images -- the matrix inverted in
    double, coordinates in fixed point with 1/32-pixel fractions, the four clamped neighbours weighted by exact products and summed
    ((S00 w00 + S01 w01) + S10 w10) + S11 w11 in float32.  Bit for bit with cv2 (tests/golden/augment.npz).
  * blur: the separable zero-padded convolution, each pass summed in tap order in float32 (blur), or in float64 with exact taps
    (blur64) for error bounds.  torch's conv2d sums in another order, so the reference's blurred crops agree to blur_bound only.
"""
import math

import numpy as np

KINDS = {"identity": 0, "translation": 1, "fliplr": 2, "blur": 3, "rotate": 4, "scale": 5}


def crop_index(out, inn, shift):
    """Source index of every output index of crop_to_output along one axis."""
    pad = math.floor((out - inn) / 2) + int(shift)
    return np.clip(np.arange(out) - pad, 0, inn - 1)


def crop(img, out_hw, shift):
    r, c = crop_index(out_hw[0], img.shape[1], shift[0]), crop_index(out_hw[1], img.shape[2], shift[1])
    return np.ascontiguousarray(img[:, r][:, :, c])


def warp_matrix(angle, h, w):
    """The inverse map cv2.warpAffine interpolates with, for augmentation.Rotate(angle) on an h x w image: the reference's numpy
    matrix [R, c - R c] (c = (shape[:2] - 1) / 2, rows first) inverted as imgwarp.cpp does."""
    a = math.pi * angle / 180
    c = (np.expand_dims(np.array([h, w]), 1) - 1) / 2
    R = np.array([[math.cos(a), math.sin(a)], [-math.sin(a), math.cos(a)]])
    M = [float(v) for v in np.concatenate([R, c - R @ c], 1).reshape(-1)]
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0] = A11; M[1] *= -D; M[3] *= -D; M[4] = A22
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return np.array(M).reshape(2, 3)


def rotate(img, angle):
    """augmentation.Rotate before its crop: [C,H,W] float32 -> [C,H,W] float32."""
    C, H, W = img.shape
    M = warp_matrix(angle, H, W)
    ys, xs = np.mgrid[0:H, 0:W]
    X0 = np.rint((M[0, 1] * ys + M[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((M[1, 1] * ys + M[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0 + np.rint(M[0, 0] * xs * 1024).astype(np.int64)) >> 5
    Y = (Y0 + np.rint(M[1, 0] * xs * 1024).astype(np.int64)) >> 5
    x0, y0 = X >> 5, Y >> 5
    fx, fy = (X & 31).astype(np.float32) / np.float32(32), (Y & 31).astype(np.float32) / np.float32(32)
    one = np.float32(1)
    w00, w01, w10, w11 = (one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx
    xa, xb = np.clip(x0, 0, W - 1), np.clip(x0 + 1, 0, W - 1)
    ya, yb = np.clip(y0, 0, H - 1), np.clip(y0 + 1, 0, H - 1)
    out = np.empty_like(img)
    for ch in range(C):
        P = img[ch]
        out[ch] = ((P[ya, xa] * w00 + P[ya, xb] * w01) + P[yb, xa] * w10) + P[yb, xb] * w11
    return out


def blur_taps(sigma, exact=False):
    """Normalised Gaussian taps exp(-x^2 / (2 sigma^2)), x = -ceil(2 sigma) .. ceil(2 sigma): evaluated in double and rounded once to
    float32 (what the kernel uses), or the double values themselves (exact=True)."""
    h = math.ceil(2 * sigma)
    g = [math.exp(-(float(i * i)) / (2.0 * sigma * sigma)) for i in range(-h, h + 1)]
    s = 0.0
    for v in g:
        s += v
    t = np.array([v / s for v in g], np.float64)
    return t if exact else t.astype(np.float32)


def _pass(img, taps, axis):
    h = (len(taps) - 1) // 2
    n = img.shape[axis]
    pad = [(0, 0)] * img.ndim
    pad[axis] = (h, h)
    p = np.pad(img, pad)
    acc = np.zeros_like(img)
    for k in range(len(taps)):
        sl = [slice(None)] * img.ndim
        sl[axis] = slice(k, k + n)
        acc = acc + p[tuple(sl)] * taps[k]
    return acc


def blur(img, sigma):
    """augmentation.Blur before its crop, each pass summed in tap order in float32 (the rows pass rounded to float32)."""
    s0, s1 = (sigma, sigma) if np.isscalar(sigma) else sigma
    return _pass(_pass(img.astype(np.float32), blur_taps(s0), 1), blur_taps(s1), 2)


def blur64(img, sigma):
    s0, s1 = (sigma, sigma) if np.isscalar(sigma) else sigma
    return _pass(_pass(img.astype(np.float64), blur_taps(s0, True), 1), blur_taps(s1, True), 2)


def blur_bound(img, sigma):
    """Bound on |float32 blur - blur64| for any tap-order or torch float32 evaluation: the rounding of taps (the reference's float32
    exp / sum / divide included), products, sums and the intermediate, relative to the largest |pixel|."""
    s0, s1 = (sigma, sigma) if np.isscalar(sigma) else sigma
    n = len(blur_taps(s0)) + len(blur_taps(s1))
    return (2 * n + 16) * 2.0 ** -24 * float(np.abs(img).max())


def transform(img, kind, shift, param, out_hw):
    """One transform of generate_init_samples on the expanded patch img [C,H,W], cropped to out_hw."""
    kind = KINDS[kind] if isinstance(kind, str) else kind
    if kind in (0, 1):
        src = img
    elif kind == 2:
        src = img[:, :, ::-1]
    elif kind == 3:
        src = blur(img, param)
    elif kind == 4:
        src = rotate(img, param)
    else:
        raise NotImplementedError("augmentation kind %r" % kind)
    return crop(src, out_hw, shift)


def transform_list(augmentation, img_sample_sz, rand_shift=None):
    """(kind, shift (row, col), param) of every transform generate_init_samples builds from params.augmentation, in its order.
    rand_shift() gives the flip / blur / rotate shifts (the reference's get_rand_shift; None = no random shift)."""
    rs = rand_shift or (lambda: (0, 0))
    out = [("identity", (0, 0), None)]
    for s in augmentation.get("shift", []):
        out.append(("translation", (int(s[0]), int(s[1])), None))
    for s in augmentation.get("relativeshift", []):
        out.append(("translation", tuple(int(v) for v in np.trunc(np.float32(s) * (np.float32(img_sample_sz) / np.float32(2)))), None))
    if augmentation.get("fliplr"):
        out.append(("fliplr", tuple(rs()), None))
    for s in augmentation.get("blur", []):
        out.append(("blur", tuple(rs()), s if isinstance(s, (tuple, list)) else (s, s)))
    if "scale" in augmentation:
        raise NotImplementedError("augmentation 'scale'")
    for a in augmentation.get("rotate", []):
        out.append(("rotate", tuple(rs()), a))
    return out
