"""Float64 reference of the IoUNet box refinement chain, error bounds for its float32 kernels, and the reference's own float32 error.

PrRoIPool (`forward`, `backward`, `coor_backward`) is evaluated in float64 in its separable form: for bin (i, j) of RoI r,
    out[r, c, i, j] = sum_h sum_w f[b_r, c, h, w] Wy[r, i, h] Wx[r, j, w] / |bin|,   Wx[r, j, w] = hat_cdf(x1 - w) - hat_cdf(x0 - w),
and the coordinate gradient from the four edge line integrals (f against hat(x0 - w) Wy[h], ...), as in csrc/prroi.cu.  Each returns,
next to the value, a magnitude term N (the same sum over absolute values) and a bound B on the error a float32 kernel can make
(`Bins._sum_bound` and the comments at each step derive it).  The geometry comes from the float32 RoIs the kernels get, converted exactly; the scale
must be a power of two (1/8, 1/16 or 1/2 here) so that `roi * scale` is exact in float32 too.

`*_f32` follow the reference CUDA kernel (ltr/external/PreciseRoIPooling/src/prroi_pooling_gpu_impl.cu, restated in
oracle/prroi_oracle.py) cell by cell with its four corner weights, in float32: the error e_32 of that formulation is the yardstick
the tests hold the kernels to, next to B.

`IoUNet64` is AtomIoUNet.predict_iou (ltr/models/bbreg/atom_iou_net.py:96-136) on pooled features: the LinearBlocks' BatchNorm folded
in float64 (as `fold_linear` in csrc/iou_refine_kernels.cuh, but kept in float64), modulation per pooled channel, ReLU, predictor; its
box gradient written out (ReLU mask -> transposed layers -> coordinate backward at both levels -> (x, y, w, h)); and one ascent step
of DiMP.optimize_boxes_default / _relative (pytracking/tracker/dimp/dimp.py:725-793).  `IoUNet64.yardstick` runs the reference's own
float32 order: modulated features, PrRoIPool, Linear, BatchNorm, ReLU, predictor, and its autograd chain backwards.

Kinks: a ReLU unit whose float64 pre-activation lies within 4 x the yardstick's error of 0 may take either side in the kernel; `evaluate` returns, per box and coordinate, the sum over such units of |grad with that unit's mask flipped - grad|
as an allowance, and how many units qualified."""
import math
import os
import re

import torch

U = 2.0 ** -24
F64, F32 = torch.float64, torch.float32


def gamma(n):
    n = torch.as_tensor(n, dtype=F64)
    return n * U / (1 - n * U)


def hat_cdf(t):
    return torch.where(t <= -1, torch.zeros_like(t), torch.where(t <= 0, 0.5 * (t + 1) ** 2, torch.where(t < 1, 1 - 0.5 * (1 - t) ** 2,
                                                                                                        torch.ones_like(t))))


def hat(t):
    return (1 - t.abs()).clamp(min=0)


class Axis:
    """One axis of the bins of R RoIs: window [lo, hi) per bin [R, P], weights Wt = integral of the hat over the window, edge hats
    T0 = hat(lo - w), T1 = hat(hi - w) [R, P, N] for the N cells of the map, and absolute bounds on the kernel's float32 versions."""

    def __init__(self, a, b, P, scale, N):
        dev = a.device
        r0, r1 = a.to(F64) * scale, b.to(F64) * scale
        self.len = (r1 - r0).clamp(min=0)                                  # roi extent in cells [R]
        self.bin = self.len / P
        p = torch.arange(P, dtype=F64, device=dev)
        self.lo = r0[:, None] + self.bin[:, None] * p
        self.hi = self.lo + self.bin[:, None]
        # float32 geometry: roi * scale exact, extent u, bin 2u relative; lo = r0 + bin * p and hi = lo + bin each add one rounding
        self.delta = U * (3 * self.len[:, None] + 2 * self.bin[:, None] + self.lo.abs() + 2 * self.hi.abs())
        self.dlen = 2 * self.delta + U * self.bin[:, None]                 # |(hi - lo) in float32 - bin|
        w = torch.arange(N, dtype=F64, device=dev)
        t0, t1 = self.lo[:, :, None] - w, self.hi[:, :, None] - w
        self.W = hat_cdf(t1) - hat_cdf(t0)
        self.T0, self.T1 = hat(t0), hat(t1)
        d = self.delta[:, :, None]
        near0, near1 = (t0.abs() < 1 + d + 1e-9).to(F64), (t1.abs() < 1 + d + 1e-9).to(F64)
        # hat_cdf(t) in float32: t = x - w rounds (u), one or two squarings and a subtraction (3u); the geometry moves t by delta
        self.dW = (4 * U + d) * (near0 + near1)
        self.dT0, self.dT1 = (2 * U + d) * near0, (2 * U + d) * near1
        # cells the kernel's loop covers: [floor(lo), ceil(hi)] clipped to the map
        self.ncov = (torch.minimum(torch.ceil(self.hi), torch.full_like(self.hi, N - 1)) - torch.floor(self.lo).clamp(min=0) + 1).clamp(min=0)


def _pool(F, Ay, Ax):
    """sum_h sum_w F[r, c, h, w] Ay[r, i, h] Ax[r, j, w] -> [R, C, PH, PW]"""
    return torch.einsum("rchj,rih->rcij", torch.einsum("rchw,rjw->rchj", F, Ax), Ay)


def _spread(O, Ay, Ax):
    """sum_i sum_j O[r, c, i, j] Ay[r, i, h] Ax[r, j, w] -> [R, C, H, W]"""
    return torch.einsum("rciw,rih->rchw", torch.einsum("rcij,rjw->rciw", O, Ax), Ay)


class Bins:
    def __init__(self, feat, rois, PH, PW, scale):
        self.B, self.C, self.H, self.W = feat.shape
        self.R, self.PH, self.PW, self.scale = rois.shape[0], PH, PW, scale
        assert math.frexp(scale)[0] == 0.5, "scale must be a power of two"
        rois = rois.to(F64)
        self.b = rois[:, 0].long()
        self.F = feat.to(F64)[self.b]
        self.A = self.F.abs()
        self.x = Axis(rois[:, 1], rois[:, 3], PW, scale, self.W)
        self.y = Axis(rois[:, 2], rois[:, 4], PH, scale, self.H)
        self.win = self.x.bin * self.y.bin
        self.inv = torch.where(self.win > 0, 1 / torch.where(self.win > 0, self.win, torch.ones_like(self.win)),
                               torch.zeros_like(self.win)).view(-1, 1, 1, 1)
        self.depth = self.y.ncov[:, None, :, None] + self.x.ncov[:, None, None, :] + 2       # fma chain of the kernel's double loop

    def _sum_bound(self, Ty, dTy, Tx, dTx):
        """Bound on |float32 separable sum - exact| for weights Ty (x) Tx known to dTy, dTx:
        gamma(depth) sum |f| (Ty + dTy)(Tx + dTx) + sum |f| (dTy Tx + Ty dTx + dTy dTx)."""
        A = self.A
        full = _pool(A, Ty + dTy, Tx + dTx)
        return gamma(self.depth) * full + (full - _pool(A, Ty, Tx))


def forward(feat, rois, PH, PW, scale):
    """PrRoIPool forward -> (out, N, B), each [R, C, PH, PW]."""
    g = Bins(feat, rois, PH, PW, scale)
    out = _pool(g.F, g.y.W, g.x.W) * g.inv
    N = _pool(g.A, g.y.W, g.x.W) * g.inv
    # the sum, then 1 / |bin| (|bin| = bw bh: 2u + 2u + u, the reciprocal u) and the product (u)
    B = g._sum_bound(g.y.W, g.y.dW, g.x.W, g.x.dW) * g.inv + 8 * U * N
    return out, N, B


def backward(feat, rois, og, PH, PW, scale):
    """PrRoIPool backward w.r.t. the features -> (fgrad, N, B), each [B, C, H, W]."""
    g = Bins(feat, rois, PH, PW, scale)
    o = og.to(F64) * g.inv
    oa = o.abs()
    Wy1, Wx1 = g.y.W + g.y.dW, g.x.W + g.x.dW
    per, full, N = _spread(o, g.y.W, g.x.W), _spread(oa, Wy1, Wx1), _spread(oa, g.y.W, g.x.W)
    # contributions per cell: the atomics add them in any order, so the chain is as long as their count
    cnt = torch.einsum("rih,rjw->rhw", (Wy1 > 0).to(F64), (Wx1 > 0).to(F64))
    shape = (g.B, g.C, g.H, g.W)
    fg = torch.zeros(shape, dtype=F64, device=o.device).index_add_(0, g.b, per)
    Nb = torch.zeros(shape, dtype=F64, device=o.device).index_add_(0, g.b, N)
    Fb = torch.zeros(shape, dtype=F64, device=o.device).index_add_(0, g.b, full)
    n = torch.zeros((g.B, 1, g.H, g.W), dtype=F64, device=o.device).index_add_(0, g.b, cnt[:, None])
    # og / |bin| (7u), Wy Wx (u), the product (u), the atomics' chain; and the weights' own errors
    B = (gamma(n) + 10 * U) * Fb + (Fb - Nb)
    return fg, Nb, B


def coor_backward(feat, rois, top, og, PH, PW, scale, dtop=None, dog=None):
    """PrRoIPool backward w.r.t. (x0, y0, x1, y1) -> (grad, N, B), each [R, 4].  `top` is the pooled output the kernel is given and
    `og` the output gradient; `dtop`, `dog` optional absolute error bounds of the kernel's copies of them."""
    g = Bins(feat, rois, PH, PW, scale)
    C, X, Y = g.C, g.x, g.y
    top, og = top.to(F64), og.to(F64)
    ta, oa = top.abs(), og.abs()
    dtop = torch.zeros_like(ta) if dtop is None else dtop.to(F64)
    dog = torch.zeros_like(oa) if dog is None else dog.to(F64)
    dx, dy = X.bin.view(-1, 1, 1, 1), Y.bin.view(-1, 1, 1, 1)                  # bin width / height
    dlx, dly = X.dlen[:, None, None, :], Y.dlen[:, None, :, None]
    s = g.inv * g.scale
    edges = {}
    # edge x = x0 / x1 integrate over y with Wy; edge y = y0 / y1 over x with Wx.  p = (+-E -+ len * top) / |bin| * scale
    for name, Ty, dTy, Tx, dTx, ln, dln, sign in (("x0", Y.W, Y.dW, X.T0, X.dT0, dy, dly, -1), ("x1", Y.W, Y.dW, X.T1, X.dT1, dy, dly, 1),
                                                   ("y0", Y.T0, Y.dT0, X.W, X.dW, dx, dlx, -1), ("y1", Y.T1, Y.dT1, X.W, X.dW, dx, dlx, 1)):
        E, A = _pool(g.F, Ty, Tx), _pool(g.A, Ty, Tx)
        p = sign * (E - ln * top) * s
        n = (A + ln * ta) * s
        # the edge sum; len in float32 (dln) times top; top's own error; len * top, the difference, 1/|bin| and the product: 9u
        b = (g._sum_bound(Ty, dTy, Tx, dTx) + dln * ta + ln * dtop) * s + 9 * U * n
        edges[name] = (p, n, b)
    pw = torch.arange(g.PW, dtype=F64, device=og.device).view(1, 1, 1, -1)
    ph = torch.arange(g.PH, dtype=F64, device=og.device).view(1, 1, -1, 1)
    cx = ((1 - pw / g.PW, 1 - (pw + 1) / g.PW), (pw / g.PW, (pw + 1) / g.PW))        # gx1: p_x0 (1 - fw0) + p_x1 (1 - fw1); gx2: ...
    cy = ((1 - ph / g.PH, 1 - (ph + 1) / g.PH), (ph / g.PH, (ph + 1) / g.PH))
    # channels: C / 128 terms per thread, a 128-thread tree (7), the bins in order, then (box_step) the two levels and x0 + x1
    depth = math.ceil(C / 128) + 7 + g.PH * g.PW + 3
    out, N, B = [], [], []
    for (a, b_), (c0, c1) in ((("x0", "x1"), cx[0]), (("y0", "y1"), cy[0]), (("x0", "x1"), cx[1]), (("y0", "y1"), cy[1])):
        (pa, na, ba), (pb, nb, bb) = edges[a], edges[b_]
        out.append(((pa * c0 + pb * c1) * og).sum((1, 2, 3)))
        n = ((na * c0 + nb * c1) * oa).sum((1, 2, 3))
        N.append(n)
        # the coefficients (1 - pw / PW: 2u), the two products and the sum (3u); og's own error
        B.append(((ba * c0 + bb * c1) * oa + (na * c0 + nb * c1) * dog).sum((1, 2, 3)) + (gamma(depth) + 5 * U) * n)
    return torch.stack(out, 1), torch.stack(N, 1), torch.stack(B, 1)


# ---- the geometry grid -------------------------------------------------------------------------------------------------------------
CLASSES = ("interior", "straddles left", "straddles right", "straddles top", "straddles bottom", "wholly outside", "covers the map",
           "a bin spans the map", "thin bins 0.02", "thin bins 0.1", "thin bins 0.25", "integer cell edges", "zero width", "zero height", "negative width")
THIN = {"thin bins 0.02": 0.02, "thin bins 0.1": 0.1, "thin bins 0.25": 0.25}
PR_MAXW = int(re.search(r"constexpr int PR_MAXW = (\d+);", open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                                             "pytracking_b200", "csrc", "prroi_kernels.cuh")).read()).group(1))


def bin_cells(rois, PH, PW, scale, H, W):
    """Cells nw, nh [R, PH, PW] the kernel's loops cover per bin, from bin_geom's float32 arithmetic (at most W, H; the shared
    arrays hold PR_MAXW)."""
    ws, hs, we, he, _ = _geom32(rois, PH, PW, scale)
    nw = (torch.clamp(torch.ceil(we), max=W - 1) - torch.clamp(torch.floor(ws), min=0) + 1).clamp(min=0)
    nh = (torch.clamp(torch.ceil(he), max=H - 1) - torch.clamp(torch.floor(hs), min=0) + 1).clamp(min=0)
    return nw.long(), nh.long()


def geometry_rois(H, W, PH, PW, scale, B, seed, per_class=2):
    """float32 RoIs [n, 5] in image coordinates (cells / scale) with `per_class` RoIs of every class of CLASSES, batch indices < B."""
    g = torch.Generator().manual_seed(seed)
    u = lambda a, b: a + (b - a) * float(torch.rand(1, generator=g))
    out = []
    for cls in CLASSES:
        for k in range(per_class):
            x0, y0 = u(1, W * 0.6), u(1, H * 0.6)
            x1, y1 = x0 + u(1.5, W * 0.4), y0 + u(1.5, H * 0.4)
            if cls == "straddles left":
                x0, x1 = u(-3, -0.05), u(0.5, W * 0.5)
            elif cls == "straddles right":
                x0, x1 = u(W * 0.5, W - 1.5), u(W - 0.9, W + 3)
            elif cls == "straddles top":
                y0, y1 = u(-3, -0.05), u(0.5, H * 0.5)
            elif cls == "straddles bottom":
                y0, y1 = u(H * 0.5, H - 1.5), u(H - 0.9, H + 3)
            elif cls == "wholly outside":           # past the last cell's hat (x >= W), or before the first (x1 <= -1)
                if k % 2:
                    x0 = u(W, W + 4); x1 = x0 + u(1, 6)
                else:
                    y1 = u(-6, -1); y0 = y1 - u(1, 6)
            elif cls == "covers the map":
                x0, y0, x1, y1 = u(-6, -0.5), u(-6, -0.5), u(W + 0.5, W + 6), u(H + 0.5, H + 6)
            elif cls == "a bin spans the map":      # bins W (H) cells wide, the second exactly [0, W]: nw = W, the most the map allows
                if k % 2 == 0:
                    x0, x1 = -float(W), float((PW - 1) * W)
                else:
                    y0, y1 = -float(H), float((PH - 1) * H)
            elif cls in THIN:
                x1 = x0 + THIN[cls] * PW
                if k % 2 == 0:
                    y1 = y0 + THIN[cls] * PH
            elif cls == "integer cell edges":       # on the first / last cell and inside
                x0, y0 = (0.0, float(int(u(1, H - 4)))) if k % 2 == 0 else (float(int(u(1, W - 4))), 0.0)
                x1 = float(W - 1) if k % 2 == 0 else float(W)
                y1 = float(H) if k % 2 == 0 else float(H - 1)
            elif cls == "zero width":
                x1 = x0
            elif cls == "zero height":
                y1 = y0
            elif cls == "negative width":
                x1 = x0 - u(0.5, 3)
            b = int(torch.randint(0, B, (1,), generator=g))
            out.append([b, x0 / scale, y0 / scale, x1 / scale, y1 / scale])
    return torch.tensor(out, dtype=F32)


def classify(rois, H, W, PH, PW, scale):
    """The classes of CLASSES each RoI [5] reaches, read back from its float32 geometry."""
    x0, y0, x1, y1 = [float(v) * scale for v in rois[1:5]]
    c = set()
    w, h = x1 - x0, y1 - y0
    if w < 0:
        c.add("negative width")
    elif w == 0:
        c.add("zero width")
    if h == 0:
        c.add("zero height")
    if w <= 0 or h <= 0:
        return c
    if x0 >= W or x1 <= -1 or y0 >= H or y1 <= -1:
        c.add("wholly outside")
        return c
    if x0 < 0 and x1 > W - 1 and y0 < 0 and y1 > H - 1:
        c.add("covers the map")
    else:
        for name, lo, hi, n in (("left", x0, x1, W), ("top", y0, y1, H)):
            if lo < 0 < hi:
                c.add("straddles " + name)
        for name, lo, hi, n in (("right", x0, x1, W), ("bottom", y0, y1, H)):
            if lo < n - 1 < hi:
                c.add("straddles " + name)
    nw, nh = bin_cells(torch.as_tensor(rois, dtype=F32).reshape(1, 5), PH, PW, scale, H, W)
    if int(nw.max()) == W or int(nh.max()) == H:
        c.add("a bin spans the map")
    for name, t in THIN.items():
        if abs(w / PW - t) < 1e-5 or abs(h / PH - t) < 1e-5:
            c.add(name)
    if all(v == int(v) for v in (x0, y0, x1, y1)):
        c.add("integer cell edges")
    if not c:
        c.add("interior")
    return c


# ---- the reference's float32 formulation (prroi_pooling_gpu_impl.cu), cell by cell -------------------------------------------------
def _geom32(rois, PH, PW, scale):
    r = rois.to(F32)
    sc = torch.tensor(scale, dtype=F32, device=r.device)
    x0, y0, x1, y1 = r[:, 1] * sc, r[:, 2] * sc, r[:, 3] * sc, r[:, 4] * sc
    bw, bh = (x1 - x0).clamp(min=0) / PW, (y1 - y0).clamp(min=0) / PH
    pw = torch.arange(PW, dtype=F32, device=r.device)
    ph = torch.arange(PH, dtype=F32, device=r.device)
    ws = (x0[:, None] + bw[:, None] * pw)[:, None, :].expand(-1, PH, -1)       # [R, PH, PW]
    hs = (y0[:, None] + bh[:, None] * ph)[:, :, None].expand(-1, -1, PW)
    we, he = ws + bw.view(-1, 1, 1), hs + bh.view(-1, 1, 1)
    win = (bw * bh).clamp(min=0).view(-1, 1, 1)
    return ws, hs, we, he, win


def _cells32(ws, hs, we, he, H, W):
    """The reference's cell range [floor(start), ceil(end)) per bin, less the cells none of whose corners lie on the map (they add
    exact zeros in the reference's sum)."""
    sw, sh = torch.floor(ws).long().clamp(min=-1), torch.floor(hs).long().clamp(min=-1)
    ew, eh = torch.ceil(we).long().clamp(max=W), torch.ceil(he).long().clamp(max=H)
    return sw, sh, ew, eh


def _getter(feat, b):
    """data(h, w) for index arrays [R, PH, PW] -> [R, C, PH, PW] in float32, zero outside the map."""
    f = feat.to(F32)
    Bn, C, H, W = f.shape

    def get(h, w):
        ok = (h >= 0) & (h < H) & (w >= 0) & (w < W)
        v = f[b.view(-1, 1, 1), :, h.clamp(0, H - 1), w.clamp(0, W - 1)]            # [R, PH, PW, C]
        return (v * ok[..., None].to(F32)).permute(0, 3, 1, 2)
    return get


def _aw(lo, hi):
    return hi - 0.5 * hi * hi - lo + 0.5 * lo * lo


def forward_f32(feat, rois, PH, PW, scale):
    """PrRoIPoolingForward: per cell the four corner weights (PrRoIPoolingMatCalculation), accumulated cell by cell in float32."""
    ws, hs, we, he, win = _geom32(rois, PH, PW, scale)
    get = _getter(feat, rois[:, 0].long())
    sw, sh, ew, eh = _cells32(ws, hs, we, he, feat.shape[2], feat.shape[3])
    acc = torch.zeros(rois.shape[0], feat.shape[1], PH, PW, dtype=F32, device=feat.device)
    nx, ny = (ew - sw).clamp(min=0), (eh - sh).clamp(min=0)
    n, nyd = nx * ny, ny.clamp(min=1)
    for idx in range(int(n.max()) if n.numel() else 0):      # cell by cell, w outer and h inner, as the reference loops
        w_it, h_it = sw + idx // nyd, sh + idx % nyd
        ok = (idx < n).to(F32)
        x0, x1 = torch.maximum(ws, w_it.to(F32)), torch.minimum(we, (w_it + 1).to(F32))
        y0, y1 = torch.maximum(hs, h_it.to(F32)), torch.minimum(he, (h_it + 1).to(F32))
        ax, axr = _aw(x0 - w_it, x1 - w_it), _aw((w_it + 1) - x1, (w_it + 1) - x0)
        ay, ayr = _aw(y0 - h_it, y1 - h_it), _aw((h_it + 1) - y1, (h_it + 1) - y0)
        s = get(h_it, w_it) * (ax * ay * ok)[:, None]
        s = s + get(h_it, w_it + 1) * (axr * ay * ok)[:, None]
        s = s + get(h_it + 1, w_it) * (ax * ayr * ok)[:, None]
        s = s + get(h_it + 1, w_it + 1) * (axr * ayr * ok)[:, None]
        acc = acc + s
    return torch.where(win[:, None] > 0, acc / torch.where(win > 0, win, torch.ones_like(win))[:, None], torch.zeros_like(acc))


def backward_f32(feat, rois, og, PH, PW, scale):
    """PrRoIPoolingBackward: every cell's four corner weights times og / |bin| added into the feature gradient in float32."""
    ws, hs, we, he, win = _geom32(rois, PH, PW, scale)
    Bn, C, H, W = feat.shape
    b = rois[:, 0].long()
    top = torch.where(win[:, None] > 0, og.to(F32) / torch.where(win > 0, win, torch.ones_like(win))[:, None], torch.zeros_like(og, dtype=F32))
    sw, sh, ew, eh = _cells32(ws, hs, we, he, H, W)
    fg = torch.zeros(Bn, C, H + 2, W + 2, dtype=F32, device=feat.device)     # one cell of padding on each side takes the overflow
    bi = b.view(-1, 1, 1, 1).expand(-1, C, PH, PW)
    ci = torch.arange(C, device=feat.device).view(1, -1, 1, 1).expand(rois.shape[0], -1, PH, PW)
    nx, ny = (ew - sw).clamp(min=0), (eh - sh).clamp(min=0)
    n, nyd = nx * ny, ny.clamp(min=1)
    for idx in range(int(n.max()) if n.numel() else 0):      # cell by cell, w outer and h inner, as the reference loops
        w_it, h_it = sw + idx // nyd, sh + idx % nyd
        ok = (idx < n).to(F32)
        x0, x1 = torch.maximum(ws, w_it.to(F32)), torch.minimum(we, (w_it + 1).to(F32))
        y0, y1 = torch.maximum(hs, h_it.to(F32)), torch.minimum(he, (h_it + 1).to(F32))
        ax, axr = _aw(x0 - w_it, x1 - w_it), _aw((w_it + 1) - x1, (w_it + 1) - x0)
        ay, ayr = _aw(y0 - h_it, y1 - h_it), _aw((h_it + 1) - y1, (h_it + 1) - y0)
        for hh, ww, wt in ((h_it, w_it, ax * ay), (h_it, w_it + 1, axr * ay), (h_it + 1, w_it, ax * ayr), (h_it + 1, w_it + 1, axr * ayr)):
            inside = ((hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)).to(F32) * ok
            v = top * (wt * inside)[:, None]
            hi = (hh.clamp(-1, H) + 1)[:, None].expand(-1, C, -1, -1)
            wi = (ww.clamp(-1, W) + 1)[:, None].expand(-1, C, -1, -1)
            fg.index_put_((bi, ci, hi, wi), v, accumulate=True)
    return fg[:, :, 1:-1, 1:-1]


def coor_backward_f32(feat, rois, top, og, PH, PW, scale):
    """PrRoIPoolingCoorBackward: the edge integrals by PrRoIPoolingSingleCoorIntegral of interpolated values, per cell row / column.
    Its double literals (0.5 * ..., 1.0 - ...) are evaluated in float64 and rounded, as the CUDA code does."""
    ws, hs, we, he, win = _geom32(rois, PH, PW, scale)
    get = _getter(feat, rois[:, 0].long())
    top, og = top.to(F32), og.to(F32)
    R, C = rois.shape[0], feat.shape[1]

    def interp(h, w):                                   # h, w float32 [R, PH, PW]
        h1, w1 = torch.floor(h), torch.floor(w)
        out = 0
        for a in (0, 1):
            for b in (0, 1):
                hh, ww = h1 + a, w1 + b
                co = (1 - (h - hh).abs()) * (1 - (w - ww).abs())
                out = out + get(hh.long(), ww.long()) * co[:, None]
        return out

    def single(s, t, c1, c2):
        s, t = s.to(F64)[:, None], t.to(F64)[:, None]
        d = (t.to(F32) * t.to(F32) - s.to(F32) * s.to(F32)).to(F64)
        return (0.5 * d * c2.to(F64) + (t - 0.5 * t * t - s + 0.5 * s * s) * c1.to(F64)).to(F32)

    z = torch.zeros(R, C, PH, PW, dtype=F32, device=feat.device)
    gx1, gx2, gy1, gy2 = z.clone(), z.clone(), z.clone(), z.clone()
    sw, sh, ew, eh = torch.floor(ws), torch.floor(hs), torch.ceil(we), torch.ceil(he)
    for dh in range(int((eh - sh).max().clamp(min=0))):
        h_it = sh + dh
        ok = (h_it < eh)[:, None].to(F32)
        s_, t_ = torch.maximum(hs, h_it) - h_it, torch.minimum(he, h_it + 1) - h_it
        gx1 = gx1 + single(s_, t_, interp(h_it, ws), interp(h_it + 1, ws)) * ok
        gx2 = gx2 + single(s_, t_, interp(h_it, we), interp(h_it + 1, we)) * ok
    for dw in range(int((ew - sw).max().clamp(min=0))):
        w_it = sw + dw
        ok = (w_it < ew)[:, None].to(F32)
        s_, t_ = torch.maximum(ws, w_it) - w_it, torch.minimum(we, w_it + 1) - w_it
        gy1 = gy1 + single(s_, t_, interp(hs, w_it), interp(hs, w_it + 1)) * ok
        gy2 = gy2 + single(s_, t_, interp(he, w_it), interp(he, w_it + 1)) * ok
    dh_, dw_ = (he - hs)[:, None], (we - ws)[:, None]
    w_ = torch.where(win > 0, win, torch.ones_like(win))[:, None]
    sc = torch.tensor(scale, dtype=F32, device=feat.device)
    px1, py1 = (-gx1 + dh_ * top) / w_ * sc, (-gy1 + dw_ * top) / w_ * sc
    px2, py2 = (gx2 - dh_ * top) / w_ * sc, (gy2 - dw_ * top) / w_ * sc
    live = ((win[:, None] > 0) & (og / w_ != 0)).to(F64)
    pw = torch.arange(PW, dtype=F64, device=feat.device).view(1, 1, 1, -1)
    ph = torch.arange(PH, dtype=F64, device=feat.device).view(1, 1, -1, 1)
    o = og.to(F64) * live
    P = [p.to(F64) for p in (px1, py1, px2, py2)]
    terms = ((P[0] * (1.0 - pw / PW) + P[2] * (1.0 - (pw + 1) / PW)) * o, (P[1] * (1.0 - ph / PH) + P[3] * (1.0 - (ph + 1) / PH)) * o,
             (P[2] * (pw + 1) / PW + P[0] * pw / PW) * o, (P[3] * (ph + 1) / PH + P[1] * ph / PH) * o)
    return torch.stack([t.to(F32).sum((1, 2, 3)) for t in terms], 1)


# ---- predict_iou and the box steps ---------------------------------------------------------------------------------------------------
def boxes_to_rois(boxes):
    """(x, y, w, h) [R, 4] -> (0, x0, y0, x1, y1) [R, 5] in float32, as make_rois_kernel."""
    b = boxes.to(F32)
    return torch.cat([torch.zeros_like(b[:, :1]), b[:, :2], b[:, :2] + b[:, 2:]], 1)


def xywh(g):
    """d/d(x0, y0, x1, y1) [R, 4] -> d/d(x, y, w, h): x1 = x + w, y1 = y + h."""
    return torch.stack([g[:, 0] + g[:, 2], g[:, 1] + g[:, 3], g[:, 2], g[:, 3]], 1)


class IoUNet64:
    LEVELS = ((3, 1.0 / 8), (4, 1.0 / 16))

    def __init__(self, sd, prefix="bb_regressor.", device="cpu"):
        def t(k):
            return sd[prefix + k].detach().to(device)
        self.raw, self.fold = {}, {}
        for lv, _ in self.LEVELS:
            n = "fc%d_rt." % lv
            W, b = t(n + "linear.weight").float(), t(n + "linear.bias").float()
            bn = [t(n + "bn." + k).float() for k in ("weight", "bias", "running_mean", "running_var")]
            self.raw[lv] = (W, b, bn)
            sc = bn[0].double() / torch.sqrt(bn[3].double() + 1e-5)
            self.fold[lv] = (W.double() * sc[:, None], b.double() * sc + bn[1].double() - bn[2].double() * sc)
        self.wp, self.bp = t("iou_predictor.weight").float().reshape(-1), t("iou_predictor.bias").float().reshape(-1)
        self.C = {lv: self.raw[lv][0].shape[1] for lv, _ in self.LEVELS}
        self.C[3] //= 25
        self.C[4] //= 9
        self.P = {3: 5, 4: 3}
        self.D3 = self.raw[3][0].shape[0]

    def evaluate(self, mod, feat, boxes, grad=True, yardstick=True):
        """float64 predict_iou of boxes [R, 4] (x, y, w, h) on one image's modulation [C] x 2 and features [1, C, H, W] x 2, with N, B
        and (yardstick) the reference's float32 values; with `grad` also the box gradient, its N, B, the kink allowance and count."""
        rois = boxes_to_rois(boxes)
        R = rois.shape[0]
        out = {"rois": rois}
        zs, zn, zb, pools = [], [], [], {}
        for lv, scale in self.LEVELS:
            P, m = self.P[lv], mod[lv - 3].reshape(-1).to(F64)
            pool, pN, pB = forward(feat[lv - 3], rois, P, P, scale)
            pools[lv] = (pool, pB)
            W, b = self.fold[lv]
            mk = m.repeat_interleave(P * P)                                   # pooled element k belongs to channel k // (P P)
            x = pool.reshape(R, -1) * mk
            zs.append(x @ W.T + b)
            zn.append(pool.abs().reshape(R, -1) * mk.abs() @ W.abs().T)
            K = x.shape[1]
            # FC: W and b rounded (u), pooled x mod (u), 20 terms per lane, a 5-level warp sum, the K slices in order and the bias
            depth = math.ceil(min(640, K) / 32) + 5 + math.ceil(K / 640) + 1
            zb.append((pB.reshape(R, -1) * mk.abs()) @ W.abs().T + (gamma(depth) + 3 * U) * zn[-1] + 2 * U * b.abs())
        z, zN, zB = torch.cat(zs, 1), torch.cat(zn, 1), torch.cat(zb, 1)
        wp, bp = self.wp.double(), float(self.bp.double())
        a = z.clamp(min=0)
        out["z"], out["zB"] = z, zB
        out["iou"] = a @ wp + bp
        out["iouN"] = a.abs() @ wp.abs() + abs(bp)
        D = z.shape[1]
        out["iouB"] = zB @ wp.abs() + gamma(math.ceil(D / 32) + 6) * out["iouN"]
        if yardstick:
            out.update(self.yardstick(mod, feat, rois, grad))
        if not grad:
            return out
        # B is a worst-case bound, some 10^3 times the typical error of these sums: as a kink threshold it would flag about one unit
        # per box.  The yardstick's own error is the threshold.
        thr = 4 * (out["z32"].double() - z).abs() if yardstick else torch.zeros_like(z)
        mask = (z > 0).to(F64)
        s = mask * wp
        g, gN, gB = self._coor(mod, feat, rois, pools, s, grad_bound=True)
        out["grad"], out["gradN"], out["gradB"] = g, gN, gB
        # kinks: flip each qualifying unit's mask; the gradient is linear in s, so its change is the gradient of +-wp_j alone
        kinks = (z.abs() <= thr).nonzero().tolist()
        allow = torch.zeros_like(g)
        for r, j in kinks:
            ds = torch.zeros_like(s)
            ds[r, j] = -wp[j] if mask[r, j] > 0 else wp[j]
            allow += self._coor(mod, feat, rois, pools, ds)[0].abs()
        out["allow"], out["kinks"] = allow, len(kinks)
        return out

    def _coor(self, mod, feat, rois, pools, s, grad_bound=False):
        R = rois.shape[0]
        gs, ns, bs = 0, 0, 0
        for lv, scale in self.LEVELS:
            P, m = self.P[lv], mod[lv - 3].reshape(-1).to(F64)
            mk = m.repeat_interleave(P * P)
            W, _ = self.fold[lv]
            sl = s[:, :self.D3] if lv == 3 else s[:, self.D3:]
            og = (sl @ W) * mk
            dog = None
            if grad_bound:      # fc_backward: D sequential fma terms over the rounded weights, then x mod
                dog = (gamma(W.shape[0] + 2) + U) * (sl.abs() @ W.abs()) * mk.abs()
                dog = dog.reshape(R, -1, P, P)
            pool, pB = pools[lv]
            g, n, b = coor_backward(feat[lv - 3], rois, pool, og.reshape(R, -1, P, P), P, P, scale, dtop=pB if grad_bound else None, dog=dog)
            gs, ns, bs = gs + g, ns + n, bs + b
        return xywh(gs), xywh(ns), xywh(bs)

    def yardstick(self, mod, feat, rois, grad):
        """The reference's float32 order: features x modulation, PrRoIPool, Linear, BatchNorm (eval), ReLU, predictor; then autograd's
        chain backwards to the boxes."""
        R = rois.shape[0]
        zs, pooled, fm = [], {}, {}
        for lv, scale in self.LEVELS:
            P = self.P[lv]
            f = feat[lv - 3].to(F32) * mod[lv - 3].to(F32).reshape(1, -1, 1, 1)
            fm[lv] = f
            p = forward_f32(f, rois, P, P, scale)
            pooled[lv] = p
            W, b, (g, be, mu, var) = self.raw[lv]
            y = p.reshape(R, -1) @ W.T + b
            zs.append((y - mu) / torch.sqrt(var + 1e-5) * g + be)
        z = torch.cat(zs, 1)
        a = z.clamp(min=0)
        out = {"z32": z, "iou32": a @ self.wp + self.bp}
        if not grad:
            return out
        s = (z > 0).to(F32) * self.wp
        g = 0
        for lv, scale in self.LEVELS:
            P = self.P[lv]
            W, b, (gm, be, mu, var) = self.raw[lv]
            sl = s[:, :self.D3] if lv == 3 else s[:, self.D3:]
            og = ((sl * gm / torch.sqrt(var + 1e-5)) @ W).reshape(R, -1, P, P)
            g = g + coor_backward_f32(fm[lv], rois, pooled[lv], og, P, P, scale)
        out["grad32"] = xywh(g.double())
        return out


def rect_to_rel(b, sz):
    return torch.stack([(b[:, 0] + 0.5 * b[:, 2]) / sz[0], (b[:, 1] + 0.5 * b[:, 3]) / sz[1], torch.log(b[:, 2]), torch.log(b[:, 3])], 1)


def rel_to_rect(r, sz):
    w, h = torch.exp(r[:, 2]), torch.exp(r[:, 3])
    return torch.stack([r[:, 0] * sz[0] - 0.5 * w, r[:, 1] * sz[1] - 0.5 * h, w, h], 1)


def box_step(boxes, g, step, relative, sz_norm=None, gN=None, gB=None):
    """One ascent step from the float32 boxes [R, 4] with the gradient g [R, 4] (x, y, w, h) in float64 -> d = b_next - b, and, given
    the gradient's N and B, the step's N, B and the part Br of B that is the boxes' own rounding: N, B propagated through the step's Jacobian in g, plus the float32 rounding of the
    boxes themselves (one rounding of b_next in default space; in relative space the device keeps its own rel copy, whose exp / log
    round trip and the rel -> rect products move b by a few ulp of the largest of |b|, |b_next| and the centre: 16 ulp)."""
    b = boxes.to(F64)
    if not relative:
        wh = b[:, 2:].repeat(1, 2)
        d = step * g * wh
        if gN is None:
            return d
        N = (step * wh).abs() * gN
        Br = U * (3 * d.abs() + (b + d).abs())
        return d, N, (step * wh).abs() * gB + Br, Br
    sz = sz_norm.to(F64)
    rel = rect_to_rel(b, sz)
    w, h = b[:, 2], b[:, 3]
    grel = torch.stack([g[:, 0] * sz[0], g[:, 1] * sz[1], (g[:, 2] - 0.5 * g[:, 0]) * w, (g[:, 3] - 0.5 * g[:, 1]) * h], 1)
    bn = rel_to_rect(rel + step * grel, sz)
    d = bn - b
    if gN is None:
        return d
    wn, hn = bn[:, 2], bn[:, 3]
    s = abs(step)

    def jac(v):
        ax = s * sz[0] ** 2 * v[:, 0] + 0.25 * s * wn * w * v[:, 0] + 0.5 * s * wn * w * v[:, 2]
        ay = s * sz[1] ** 2 * v[:, 1] + 0.25 * s * hn * h * v[:, 1] + 0.5 * s * hn * h * v[:, 3]
        aw = 0.5 * s * wn * w * v[:, 0] + s * wn * w * v[:, 2]
        ah = 0.5 * s * hn * h * v[:, 1] + s * hn * h * v[:, 3]
        return torch.stack([ax, ay, aw, ah], 1)
    centre = torch.stack([rel[:, 0] * sz[0], rel[:, 1] * sz[1], w, h], 1).abs()
    Br = 16 * U * (b.abs() + bn.abs() + centre) + 4 * U * d.abs()
    return d, jac(gN), jac(gB) + Br, Br


def step_allowance(boxes, g, allow, step, relative, sz_norm=None):
    """|d(g +- allow) - d(g)| per entry: the kink allowance carried through one step (linear in default space)."""
    if not relative:
        return (step * boxes.to(F64)[:, 2:].repeat(1, 2)).abs() * allow
    d0 = box_step(boxes, g, step, True, sz_norm)
    return torch.maximum((box_step(boxes, g + allow, step, True, sz_norm) - d0).abs(), (box_step(boxes, g - allow, step, True, sz_norm) - d0).abs())


# ---- the checks both test tiers run --------------------------------------------------------------------------------------------------
PRROI_MAPS = ((36, 1.0 / 8), (44, 1.0 / 8), (18, 1.0 / 16), (22, 1.0 / 16))
PRROI_CASES = [(n, sc, P, B) for n, sc in PRROI_MAPS for P in (5, 3, 7) for B in (1, 3)] + [(62, 1.0 / 8, 3, 1)]   # 62: nw = PR_MAXW - 2
IOU_MAPS = {"dimp 288": (36, 18), "prdimp 352": (44, 22)}


def ratios(ker, ref, N, B, r32):
    """Per entry: e = |ker - ref| / N and e_32 = |r32 - ref| / N; returns (e / max(4 e_32, B / N) [max], e [max], e_32 [max], number of
    entries with N == 0 that are not exactly 0 in the kernel)."""
    ker, ref, r32 = ker.to(F64), ref.to(F64), r32.to(F64)
    live = N > 0
    Ns = torch.where(live, N, torch.ones_like(N))
    e, e32 = (ker - ref).abs() / Ns, (r32 - ref).abs() / Ns
    bar = torch.maximum(4 * e32, B / Ns)
    q = torch.where(live, e / bar, torch.zeros_like(e))
    dead = int(((~live) & (ker != 0)).sum())
    return (float(q.max()) if q.numel() else 0.0, float(e[live].max()) if live.any() else 0.0, float(e32[live].max()) if live.any() else 0.0,
            dead)


YARD, FLOOR = 20, 64 * U


def yardstick_ratio(ker, ref, N, r32, slack=None):
    """The float32-yardstick check of one case, which the worst-case bound B alone is too loose for where long sums cancel
    (predict_iou, its gradient and the steps): max over entries of e = max(|ker - ref| - slack, 0) / N must stay within
    YARD x the max over entries of e_32 = |r32 - ref| / N, plus FLOOR (64 ulp of the magnitude term, for cases of a few entries whose
    e_32 is small by chance).  Returns e_max / (YARD e32_max + FLOOR)."""
    ker, ref, r32 = ker.to(F64), ref.to(F64), r32.to(F64)
    live = N > 0
    if not bool(live.any()):
        return 0.0
    d = (ker - ref).abs()
    if slack is not None:
        d = (d - slack).clamp(min=0)
    e, e32 = (d / N)[live].max(), ((r32 - ref).abs() / N)[live].max()
    return float(e / (YARD * e32 + FLOOR))


def prroi_inputs(n, scale, P, B, C, seed, device):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, C, n, n, generator=g).to(device)
    rois = geometry_rois(n, n, P, P, scale, B, seed).to(device)
    og = torch.randn(rois.shape[0], C, P, P, generator=g).to(device)
    return feat, rois, og


def check_prroi(fwd, bwd, coor, n, scale, P, B, C, seed, device):
    """Run the three kernels (callables on float32 tensors of `device`) on one case of the grid; returns {(kernel, class): (worst
    e / bar, worst e, worst e_32)}, the classes reached and the most cells a bin covers.  Asserts every entry within its bar, exact zeros
    where N == 0, and a bin covering all n cells of a row or column."""
    feat, rois, og = prroi_inputs(n, scale, P, B, C, seed, device)
    classes = [classify(r.cpu(), n, n, P, P, scale) for r in rois]
    out = fwd(feat, rois, P, scale)
    o64, oN, oB = forward(feat, rois, P, P, scale)
    o32 = forward_f32(feat, rois, P, P, scale)
    fg = bwd(feat, rois, out, og, P, scale)
    f64, fN, fB = backward(feat, rois, og, P, P, scale)
    f32 = backward_f32(feat, rois, og, P, P, scale)
    rg = coor(feat, rois, out, og, P, scale)
    r64, rN, rB = coor_backward(feat, rois, out, og, P, P, scale)
    r32 = coor_backward_f32(feat, rois, out, og, P, P, scale)
    res = {}
    for i, cl in enumerate(classes):
        for kname, k, ref, N, Bd, y in (("forward", out[i], o64[i], oN[i], oB[i], o32[i]), ("coor_backward", rg[i, 1:], r64[i], rN[i], rB[i], r32[i])):
            q = ratios(k, ref, N, Bd, y)
            assert q[0] <= 1 and q[3] == 0, (kname, sorted(cl), rois[i].tolist(), q)
            for c in cl:
                prev = res.get((kname, c), (0.0, 0.0, 0.0))
                res[(kname, c)] = tuple(max(a, b) for a, b in zip(prev, q[:3]))
        if "wholly outside" in cl or "zero width" in cl or "zero height" in cl or "negative width" in cl:
            assert float(out[i].abs().max()) == 0 and float(rg[i].abs().max()) == 0, (sorted(cl), rois[i].tolist())
    assert float(rg[:, 0].abs().max()) == 0
    q = ratios(fg, f64, fN, fB, f32)
    assert q[0] <= 1 and q[3] == 0, ("backward", q)
    res[("backward", "all")] = q[:3]
    # the map-spanning RoIs give bins of n cells, the most bin_geom can clip to (PR_MAXW - 2 on the 62 map)
    nw, nh = bin_cells(rois.cpu(), P, P, scale, n, n)
    cells = max(int(nw.max()), int(nh.max()))
    assert cells == n <= PR_MAXW - 2, (cells, n, PR_MAXW)
    return res, set().union(*classes), cells


def iou_inputs_on(maps, C, seed, device):
    """Modulation [C] x 2 and features [1, C, H, W] x 2 for the maps (H3, H4): ReLU of Gaussians, as the IoU branch's output."""
    g = torch.Generator().manual_seed(seed)
    f3 = torch.relu(torch.randn(1, C, maps[0], maps[0], generator=g))
    f4 = torch.relu(torch.randn(1, C, maps[1], maps[1], generator=g))
    mod = [torch.randn(C, generator=g).abs(), torch.randn(C, generator=g).abs()]
    return [m.to(device) for m in mod], [f3.to(device), f4.to(device)]


def class_boxes(maps, seed, device, positive=False):
    """28 boxes (x, y, w, h) in image coordinates, two of each class of CLASSES on the 1/8 map (`positive`: only those with w, h > 0)."""
    rois = geometry_rois(maps[0], maps[0], 5, 5, 1.0 / 8, 1, seed)
    b = torch.cat([rois[:, 1:3], rois[:, 3:5] - rois[:, 1:3]], 1)
    if positive:
        b = b[(b[:, 2] > 0) & (b[:, 3] > 0)]
    return b.to(device)


def check_predict(run, net, maps, R, mod, feat, boxes):
    """`run(boxes) -> (iou [R], grad [R, 4])` on float32 tensors; checks IoU and gradient per box and coordinate against the bar and,
    case by case, against the yardstick (`yardstick_ratio`; the gradient less its kink allowance).  Returns (worst IoU e / bar, e, e_32,
    worst gradient e / bar, e, e_32, kink units, IoU and gradient yardstick ratios)."""
    iou, grad = run(boxes)
    out = net.evaluate(mod, feat, boxes)
    qi = ratios(iou, out["iou"], out["iouN"], out["iouB"], out["iou32"])
    assert qi[0] <= 1, ("iou", qi)
    qg = ratios(grad, out["grad"], out["gradN"], out["gradB"] + out["allow"], out["grad32"])
    assert qg[0] <= 1 and qg[3] == 0, ("grad", qg)
    yi = yardstick_ratio(iou, out["iou"], out["iouN"], out["iou32"])
    yg = yardstick_ratio(grad, out["grad"], out["gradN"], out["grad32"], out["allow"])
    assert yi <= 1 and yg <= 1, ("yardstick", yi, yg)
    return qi[:3] + qg[:3] + (out["kinks"], yi, yg)


def refine_configs():
    """(name, relative, iterations, step, decay): dimp50 / ATOM, prdimp50, and each once more with the on-device step decay."""
    return [("default", False, 5, 1.0, 1.0), ("relative", True, 10, 2.5e-3, 1.0), ("default decay", False, 5, 1.0, 0.8),
            ("relative decay", True, 10, 2.5e-3, 0.8)]


def check_refine(refine, net, mod, feat, boxes, relative, iters, step, decay):
    """`refine(boxes, k) -> (boxes_k, iou)` with k iterations.  Every step d_k = b_{k+1} - b_k against the float64 step from b_k (bar
    as above, widened by the kink allowance and by the float32 step length's rounding after k decays); the IoUs of the N-iteration call
    must be those of b_{N-1}.  Each step is also held to the yardstick (`yardstick_ratio`), less the allowances and the boxes' own float32
    rounding.  Returns ((worst e / bar, e, e_32, kink units, worst yardstick ratio), the iterates)."""
    bs = [boxes.float()]
    for k in range(1, iters + 1):
        bs.append(refine(boxes, k)[0])
    sz = boxes[0, 2:].to(F64)
    worst, ew, e32w, kinks, yw = 0.0, 0.0, 0.0, 0, 0.0
    for k in range(iters):
        s = step * decay ** k
        out = net.evaluate(mod, feat, bs[k])
        d64, N, B, Br = box_step(bs[k], out["grad"], s, relative, sz, out["gradN"], out["gradB"])
        d32 = box_step(bs[k], out["grad32"], s, relative, sz)
        allow = step_allowance(bs[k], out["grad"], out["allow"], s, relative, sz)
        dker = bs[k + 1].to(F64) - bs[k].to(F64)
        slack = allow + 2 * (k + 1) * U * d64.abs()
        q = ratios(dker, d64, N, B + slack, d32)
        y = yardstick_ratio(dker, d64, N, d32, slack + Br)
        assert q[0] <= 1 and q[3] == 0 and y <= 1, (k, q, y)
        yw = max(yw, y)
        worst, ew, e32w = max(worst, q[0]), max(ew, q[1]), max(e32w, q[2])
        kinks += out["kinks"]
    return (worst, ew, e32w, kinks, yw), bs
