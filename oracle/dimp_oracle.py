"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch-CPU fp32) of the reference's per-frame hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs may import this module; the product path (`pytracking_b200/`) never does and fails loudly
when its CUDA library is missing.

Parity status: PINNED against the reference itself.  `oracle/gen_golden.py` runs the unmodified
reference (visionml/pytracking @ 7eb9e74) in the build container through `oracle/ref_shims.py`
and commits its outputs under `tests/golden/`; `tests/test_oracle_golden.py` checks every
function below against those vectors (the reference repo holds no known-answer tests of its own
for these stages, SURVEY.md section 4 -- the only one, PrRoIPool forward == avg_pool2d, is
replayed in tests/test_prroi_oracle.py).

Each function cites the reference lines it restates (paths relative to the reference root).
The formulas are written out explicitly (SURVEY.md section 9) instead of re-issuing the
reference's grouped-conv tricks, so that the oracle is an independent statement of the maths.
"""
import math
from collections import OrderedDict

import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# Stage 1: backbone + classification head
# ----------------------------------------------------------------------------------------------
def preprocess_image(im, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
    """pytracking/features/net_wrappers.py:55-69 -- /255, -mean, /std (rgb)."""
    m = torch.tensor(mean, dtype=torch.float32).view(1, -1, 1, 1)
    s = torch.tensor(std, dtype=torch.float32).view(1, -1, 1, 1)
    return (im / 255 - m) / s


def _bn_eval(x, sd, p, eps=1e-5):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        training=False, eps=eps)


def _bottleneck(x, sd, p, stride):
    """ltr/models/backbone/resnet.py:56-92 (stride sits on the 3x3)."""
    out = F.relu(_bn_eval(F.conv2d(x, sd[p + "conv1.weight"]), sd, p + "bn1"))
    out = F.relu(_bn_eval(F.conv2d(out, sd[p + "conv2.weight"], stride=stride, padding=1), sd, p + "bn2"))
    out = _bn_eval(F.conv2d(out, sd[p + "conv3.weight"]), sd, p + "bn3")
    if (p + "downsample.0.weight") in sd:
        x = _bn_eval(F.conv2d(x, sd[p + "downsample.0.weight"], stride=stride), sd, p + "downsample.1")
    return F.relu(out + x)


def _basicblock(x, sd, p, stride):
    """ltr/models/backbone/resnet.py:15-53."""
    out = F.relu(_bn_eval(F.conv2d(x, sd[p + "conv1.weight"], stride=stride, padding=1), sd, p + "bn1"))
    out = _bn_eval(F.conv2d(out, sd[p + "conv2.weight"], padding=1), sd, p + "bn2")
    if (p + "downsample.0.weight") in sd:
        x = _bn_eval(F.conv2d(x, sd[p + "downsample.0.weight"], stride=stride), sd, p + "downsample.1")
    return F.relu(out + x)


def resnet_forward(sd, im, arch="resnet50", output_layers=("layer2", "layer3"), prefix="feature_extractor."):
    """ResNet.forward with early exit after the last requested layer (resnet.py:175-221).
    `im` is the already normalised crop [S,3,H,W]."""
    from pytracking_b200.synth import RESNET_ARCH
    block, layers = RESNET_ARCH[arch]
    out = OrderedDict()
    x = F.relu(_bn_eval(F.conv2d(im, sd[prefix + "conv1.weight"], stride=2, padding=3), sd, prefix + "bn1"))
    if "conv1" in output_layers:
        out["conv1"] = x
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    last = max(int(l[-1]) for l in output_layers if l.startswith("layer"))
    for li in range(last):
        for bi in range(layers[li]):
            p = "%slayer%d.%d." % (prefix, li + 1, bi)
            stride = 2 if (li > 0 and bi == 0) else 1
            x = _bottleneck(x, sd, p, stride) if block == "bottleneck" else _basicblock(x, sd, p, stride)
        name = "layer%d" % (li + 1)
        if name in output_layers:
            out[name] = x
    return out


def instance_l2norm(x, scale, eps=1e-5):
    """ltr/models/layers/normalization.py:15-20 (size_average=True)."""
    n = x.shape[0]
    ss = (x * x).reshape(n, -1).sum(dim=1).reshape(n, 1, 1, 1)
    return x * (scale * torch.sqrt((x.shape[1] * x.shape[2] * x.shape[3]) / (ss + eps)))


def clf_head_dimp50(sd, layer3, filter_size=4, prefix="classifier.feature_extractor."):
    """residual_bottleneck(num_blocks=0, final_conv=True): conv3x3 1024->512 + InstanceL2Norm
    (ltr/models/target_classifier/features.py:50-73, norm scale ltr/models/tracking/dimpnet.py:159)."""
    w = sd[prefix + "0.weight"]
    x = F.conv2d(layer3, w, padding=1)
    return instance_l2norm(x, math.sqrt(1.0 / (w.shape[0] * filter_size * filter_size)))


def clf_head_dimp18(sd, layer3, filter_size=4, prefix="classifier.feature_extractor."):
    """residual_basic_block(num_blocks=1, final_conv=True) (features.py:9-28): torchvision BasicBlock + conv3x3."""
    x = _basicblock(layer3, sd, prefix + "0.", 1)
    w = sd[prefix + "1.weight"]
    x = F.conv2d(x, w, padding=1)
    return instance_l2norm(x, math.sqrt(1.0 / (w.shape[0] * filter_size * filter_size)))


# ----------------------------------------------------------------------------------------------
# Stage 2: correlation and its adjoint, arg-max
# ----------------------------------------------------------------------------------------------
def _padded_windows(feat, k):
    """All k x k windows of the zero-padded (pad k//2) feature map: [n, C, Ho, Wo, k, k]."""
    p = k // 2
    xp = F.pad(feat, (p, p, p, p))
    return xp.unfold(2, k, 1).unfold(3, k, 1)


def apply_filter(feat, w):
    """ltr/models/layers/filter.py:5-57 for one sequence: feat [n,C,H,W], w [1,C,k,k] -> [n,1,Ho,Wo] in feat's dtype,
    s[i,y,x] = sum_{c,u,v} xpad[i,c,y+u,x+v] * w[c,u,v], pad k//2 on all sides (19x19 for 18x18, k=4)."""
    k = w.shape[-1]
    win = _padded_windows(feat, k)
    return torch.einsum("ncyxuv,cuv->nyx", win.double(), w[0].double()).to(feat.dtype).unsqueeze(1)


def apply_feat_transpose(feat, r, k):
    """ltr/models/layers/filter.py:91-107,129-182 (v2 and v3 are the same exact adjoint):
    g[c,u,v] = sum_{i,y,x} r[i,y,x] * xpad[i,c,y+u,x+v]. r is [n,1,Ho,Wo]; returns [1,C,k,k]."""
    win = _padded_windows(feat, k)
    return torch.einsum("ncyxuv,nyx->cuv", win.double(), r[:, 0].double()).to(feat.dtype).unsqueeze(0)


def max2d(a):
    """pytracking/libs/dcf.py:156-164 -- row max, then col max, first index on ties."""
    max_val_row, argmax_row = torch.max(a, dim=-2)          # per column: best row (first on ties)
    max_val, argmax_col = torch.max(max_val_row, dim=-1)    # best column (first on ties)
    rows = torch.gather(argmax_row, -1, argmax_col.unsqueeze(-1)).squeeze(-1)
    return max_val, torch.stack((rows, argmax_col), dim=-1)


# ----------------------------------------------------------------------------------------------
# Stage 3a: DiMP steepest-descent Gauss-Newton
# ----------------------------------------------------------------------------------------------
def radial_lut(lut, rho):
    """DistanceMap (ltr/models/layers/distance.py:17-39) followed by a 1x1 conv with `lut` as weights
    == piece-wise linear interpolation of `lut` at rho, last bin clamping (SURVEY.md 9.2)."""
    nb = lut.numel()
    out = torch.zeros_like(rho)
    for b in range(nb - 1):
        out = out + lut[b] * F.relu(1.0 - torch.abs(rho - b))
    out = out + lut[nb - 1] * (1.0 + (rho - (nb - 1))).clamp(0, 1)
    return out


def dimp_label_maps(bb, params, out_sz, filter_size=4, feat_stride=16, bin_displacement=0.1):
    """optimizer.py:111-119: label y, target mask m = sigmoid(.), spatial weight v per sample; [n,Ho,Wo] each."""
    off = (filter_size % 2) / 2.0
    center = ((bb[:, :2] + bb[:, 2:] / 2) / feat_stride).flip((1,)) - off   # (row, col)
    k0 = torch.arange(out_sz[0], dtype=bb.dtype, device=bb.device).view(1, -1, 1)
    k1 = torch.arange(out_sz[1], dtype=bb.dtype, device=bb.device).view(1, 1, -1)
    d0 = k0 - center[:, 0].view(-1, 1, 1)
    d1 = k1 - center[:, 1].view(-1, 1, 1)
    rho = torch.sqrt(d0 * d0 + d1 * d1) / bin_displacement
    y = radial_lut(params["label_map_predictor.weight"].reshape(-1), rho)
    m = torch.sigmoid(radial_lut(params["target_mask_predictor.0.weight"].reshape(-1), rho))
    v = radial_lut(params["spatial_weight_predictor.weight"].reshape(-1), rho)
    return y, m, v


def dimp_sd_gn(w, feat, bb, sample_weight, params, num_iter, min_filter_reg=1e-3, alpha_eps=0.0,
               feat_stride=16, bin_displacement=0.1, compute_losses=True):
    """DiMPSteepestDescentGN.forward (ltr/models/target_classifier/optimizer.py:85-170), one sequence,
    score_act='relu', mask_act='sigmoid'. w [1,C,k,k], feat [n,C,H,W], bb [n,4], sample_weight [n] or None.
    Returns (w_final, [iterates], [losses])."""
    n = feat.shape[0]
    k = w.shape[-1]
    out_sz = (feat.shape[-2] + (k + 1) % 2, feat.shape[-1] + (k + 1) % 2)
    step = torch.exp(params["log_step_length"]).item()
    reg = max(params["filter_reg"].item() ** 2, min_filter_reg ** 2)
    y, m, v = dimp_label_maps(bb, params, out_sz, k, feat_stride, bin_displacement)
    if sample_weight is None:
        vh = math.sqrt(1.0 / n) * v
    else:
        vh = sample_weight.sqrt().reshape(n, 1, 1) * v
    iterates = [w]
    losses = []
    for _ in range(num_iter):
        s = apply_filter(feat, w)[:, 0]
        act = (1.0 - m) / 2.0 * s.abs() + (1.0 + m) / 2.0 * s          # activation.py:36-37
        dact = (1.0 - m) / 2.0 * torch.sign(s) + (1.0 + m) / 2.0       # activation.py:43-44
        r = vh * (act - y)
        if compute_losses:
            losses.append((r ** 2).sum() + reg * (w ** 2).sum())
        g = apply_feat_transpose(feat, (dact * (vh * r)).unsqueeze(1), k) + reg * w
        q = apply_filter(feat, g)[:, 0]
        h = vh * (dact * q)
        a_num = (g * g).sum()
        a_den = ((h * h).sum() + (reg + alpha_eps) * a_num).clamp(min=1e-8)
        w = w - (step * (a_num / a_den)) * g
        iterates.append(w)
    if compute_losses:
        s = apply_filter(feat, w)[:, 0]
        act = (1.0 - m) / 2.0 * s.abs() + (1.0 + m) / 2.0 * s
        losses.append(((vh * (act - y)) ** 2).sum() + reg * (w ** 2).sum())
    return w, iterates, losses


def dimp_l2_sd_gn(w, feat, bb, sample_weight, log_step_length, filter_reg, num_iter, gauss_sigma, hinge_threshold=-999.0,
                  min_filter_reg=1e-3, alpha_eps=0.0, feat_stride=16, compute_losses=True):
    """DiMPL2SteepestDescentGN.forward (ltr/models/target_classifier/optimizer.py:211-291), one sequence."""
    n = feat.shape[0]
    k = w.shape[-1]
    out_sz = (feat.shape[-2] + (k + 1) % 2, feat.shape[-1] + (k + 1) % 2)
    step = math.exp(float(log_step_length))
    reg = max(float(filter_reg) ** 2, min_filter_reg ** 2)
    off = (k % 2) / 2.0
    center = ((bb[:, :2] + bb[:, 2:] / 2) / feat_stride).flip((1,)) - off
    k0 = torch.arange(out_sz[0], dtype=bb.dtype, device=bb.device).view(1, -1, 1)
    k1 = torch.arange(out_sz[1], dtype=bb.dtype, device=bb.device).view(1, 1, -1)
    g0 = torch.exp(-1.0 / (2 * gauss_sigma ** 2) * (k0 - center[:, 0].view(-1, 1, 1)) ** 2)
    g1 = torch.exp(-1.0 / (2 * gauss_sigma ** 2) * (k1 - center[:, 1].view(-1, 1, 1)) ** 2)
    y = g0 * g1
    m = (y > hinge_threshold).to(y.dtype)
    y = y * m
    sw = math.sqrt(1.0 / n) if sample_weight is None else sample_weight.sqrt().reshape(n, 1, 1)
    iterates, losses = [w], []
    for _ in range(num_iter):
        s = apply_filter(feat, w)[:, 0]
        act = m * s + (1.0 - m) * F.relu(s)
        dact = m + (1.0 - m) * (s > 0).float()
        r = sw * (act - y)
        if compute_losses:
            losses.append((r ** 2).sum() + reg * (w ** 2).sum())
        g = apply_feat_transpose(feat, (dact * (sw * r)).unsqueeze(1), k) + reg * w
        h = sw * (dact * apply_filter(feat, g)[:, 0])
        a_num = (g * g).sum()
        a_den = ((h * h).sum() + (reg + alpha_eps) * a_num).clamp(min=1e-8)
        w = w - (step * (a_num / a_den)) * g
        iterates.append(w)
    if compute_losses:
        s = apply_filter(feat, w)[:, 0]
        act = m * s + (1.0 - m) * F.relu(s)
        losses.append(((sw * (act - y)) ** 2).sum() + reg * (w ** 2).sum())
    return w, iterates, losses


def gn_sd_hinge(w, feat, train_label, sample_weight, filter_reg, num_iter, hinge_threshold=-999.0, activation_leak=0.0,
                score_act="relu", act_param=1.0, steplength_reg=0.0, compute_losses=True):
    """GNSteepestDescent.forward (ltr/models/meta/steepestdescent.py:32-105) over LinearFilterHinge
    (ltr/models/target_classifier/residual_modules.py:89-135), one sequence, with g = J^T r and h = J g written out.
    train_label [n,Ho,Wo]."""
    n = feat.shape[0]
    k = w.shape[-1]
    sw = math.sqrt(1.0 / n) if sample_weight is None else sample_weight.sqrt().reshape(n, 1, 1)
    m = ((train_label > hinge_threshold).to(train_label.dtype) + activation_leak).clamp(max=1.0)
    y = m * train_label

    def act_fn(s):
        if score_act == "bentpar":
            rt = torch.sqrt(s * s + 4.0 * act_param * act_param)
            return (1.0 - m) / 2.0 * (rt - 2.0 * act_param) + (1.0 + m) / 2.0 * s, (1.0 - m) / 2.0 * (s / rt) + (1.0 + m) / 2.0
        return (1.0 - m) / 2.0 * s.abs() + (1.0 + m) / 2.0 * s, (1.0 - m) / 2.0 * torch.sign(s) + (1.0 + m) / 2.0

    numel = n * train_label.shape[-2] * train_label.shape[-1] + w.numel()
    iterates, losses = [w], []
    for _ in range(num_iter):
        s = apply_filter(feat, w)[:, 0]
        a, d = act_fn(s)
        r = sw * (a - y)
        if compute_losses:
            losses.append(((r ** 2).sum() + (filter_reg * w).pow(2).sum()) / numel)
        g = apply_feat_transpose(feat, (d * (sw * r)).unsqueeze(1), k) + filter_reg * filter_reg * w
        h = sw * (d * apply_filter(feat, g)[:, 0])
        gg = (g * g).sum()
        hh = (h * h).sum() + (filter_reg * g).pow(2).sum()
        alpha = gg / (hh + steplength_reg * gg).clamp(min=1e-8)
        w = w - alpha * g
        iterates.append(w)
    if compute_losses:
        a, _ = act_fn(apply_filter(feat, w)[:, 0])
        losses.append((((sw * (a - y)) ** 2).sum() + (filter_reg * w).pow(2).sum()) / numel)
    return w, iterates, losses


# ----------------------------------------------------------------------------------------------
# Stage 3b: PrDiMP steepest-descent Newton
# ----------------------------------------------------------------------------------------------
def prdimp_label_density(bb, out_sz, gauss_sigma, filter_size=4, feat_stride=16, label_threshold=0.0,
                         normalize_label=False, label_shrink=0.0, uni_weight=0.0):
    """get_label_density (optimizer.py:331-353), gauss_sigma > 0."""
    off = (filter_size % 2) / 2.0
    center = ((bb[:, :2] + bb[:, 2:] / 2) / feat_stride).flip((1,)) - off
    k0 = torch.arange(out_sz[0], dtype=bb.dtype, device=bb.device).view(1, -1, 1)
    k1 = torch.arange(out_sz[1], dtype=bb.dtype, device=bb.device).view(1, 1, -1)
    g0 = torch.exp(-1.0 / (2 * gauss_sigma ** 2) * (k0 - center[:, 0].view(-1, 1, 1)) ** 2)
    g1 = torch.exp(-1.0 / (2 * gauss_sigma ** 2) * (k1 - center[:, 1].view(-1, 1, 1)) ** 2)
    gauss = (g0 / (2 * math.pi * gauss_sigma ** 2)) * g1
    gauss = gauss * (gauss > label_threshold).to(gauss.dtype)
    if normalize_label:
        gauss = gauss / (gauss.sum(dim=(-2, -1), keepdim=True) + 1e-8)
    return (1.0 - label_shrink) * ((1.0 - uni_weight) * gauss + uni_weight / (out_sz[0] * out_sz[1]))


def softmax_reg(s, reg):
    """ltr/models/layers/activation.py:7-16 over the flattened map with one extra logit `reg`."""
    n = s.shape[0]
    flat = s.reshape(n, -1)
    if reg is None:
        return torch.softmax(flat, dim=1).reshape(s.shape)
    ext = torch.cat((flat, torch.full((n, 1), float(reg), dtype=s.dtype, device=s.device)), dim=1)
    return torch.softmax(ext, dim=1)[:, :-1].reshape(s.shape)


def prdimp_sd_newton(w, feat, bb, sample_weight, log_step_length, filter_reg, num_iter, gauss_sigma,
                     min_filter_reg=1e-3, alpha_eps=0.0, softmax_reg_val=None, label_threshold=0.0,
                     normalize_label=False, label_shrink=0.0, uni_weight=0.0, feat_stride=16,
                     compute_losses=True):
    """PrDiMPSteepestDescentNewton.forward (optimizer.py:355-439), one sequence."""
    n = feat.shape[0]
    k = w.shape[-1]
    out_sz = (feat.shape[-2] + (k + 1) % 2, feat.shape[-1] + (k + 1) % 2)
    step = math.exp(float(log_step_length))
    reg = max(float(filter_reg) ** 2, min_filter_reg ** 2)
    p = prdimp_label_density(bb, out_sz, gauss_sigma, k, feat_stride, label_threshold, normalize_label,
                             label_shrink, uni_weight)
    if sample_weight is None:
        sw = torch.full((n, 1, 1), 1.0 / n, dtype=feat.dtype, device=feat.device)
    else:
        sw = sample_weight.reshape(n, 1, 1)
    exp_reg = 0.0 if softmax_reg_val is None else math.exp(softmax_reg_val)

    def loss_fn(s, w_):
        return (sw.reshape(n) * (torch.log(s.exp().sum(dim=(-2, -1)) + exp_reg) - (p * s).sum(dim=(-2, -1)))).sum() \
            + reg * (w_ ** 2).sum()

    iterates = [w]
    losses = []
    for _ in range(num_iter):
        s = apply_filter(feat, w)[:, 0]
        sm = softmax_reg(s, softmax_reg_val)
        res = sw * (sm - p)
        if compute_losses:
            losses.append(loss_fn(s, w))
        g = apply_feat_transpose(feat, res.unsqueeze(1), k) + reg * w
        q = apply_filter(feat, g)[:, 0]
        smq = sm * q
        hq = smq - sm * smq.sum(dim=(-2, -1), keepdim=True)
        ghg = (q * hq).reshape(n, -1).sum(dim=1).clamp(min=0)
        ghg = (sw.reshape(n) * ghg).sum()
        a_num = (g * g).sum()
        a_den = (ghg + (reg + alpha_eps) * a_num).clamp(min=1e-8)
        w = w - (step * (a_num / a_den)) * g
        iterates.append(w)
    if compute_losses:
        losses.append(loss_fn(apply_filter(feat, w)[:, 0], w))
    return w, iterates, losses


# ----------------------------------------------------------------------------------------------
# Library-call formulation (what the reference actually executes on CPU: grouped F.conv2d), used as the
# timed CPU baseline in bench.py; tests check it against the explicit formulas above.
# ----------------------------------------------------------------------------------------------
def apply_filter_conv(feat, w):
    """filter.py:54-57 -- one sequence: a plain conv with the filter as the single output channel."""
    k = w.shape[-1]
    return F.conv2d(feat, w, padding=k // 2)


def apply_feat_transpose_conv(feat, r, k):
    """filter.py:129-155 (_v2, the eval-mode path): features as kernels, groups = samples, sum, flip."""
    n, c = feat.shape[:2]
    g = F.conv2d(r.reshape(1, n, r.shape[-2], r.shape[-1]), feat.reshape(n * c, 1, feat.shape[-2], feat.shape[-1]),
                 padding=(k - 1) // 2, groups=n)
    return g.reshape(n, c, g.shape[-2], g.shape[-1]).sum(dim=0, keepdim=True).flip((2, 3))


def dimp_sd_gn_conv(w, feat, bb, sample_weight, params, num_iter, min_filter_reg=1e-3, alpha_eps=0.0,
                    feat_stride=16, bin_displacement=0.1):
    """Same iteration as dimp_sd_gn but with the reference's three library sweeps per iteration (no losses)."""
    n = feat.shape[0]
    k = w.shape[-1]
    out_sz = (feat.shape[-2] + (k + 1) % 2, feat.shape[-1] + (k + 1) % 2)
    step = torch.exp(params["log_step_length"]).item()
    reg = max(params["filter_reg"].item() ** 2, min_filter_reg ** 2)
    y, m, v = dimp_label_maps(bb, params, out_sz, k, feat_stride, bin_displacement)
    vh = (math.sqrt(1.0 / n) * v) if sample_weight is None else sample_weight.sqrt().reshape(n, 1, 1) * v
    for _ in range(num_iter):
        s = apply_filter_conv(feat, w)[:, 0]
        act = (1.0 - m) / 2.0 * s.abs() + (1.0 + m) / 2.0 * s
        dact = (1.0 - m) / 2.0 * torch.sign(s) + (1.0 + m) / 2.0
        r = vh * (act - y)
        g = apply_feat_transpose_conv(feat, (dact * (vh * r)).unsqueeze(1), k) + reg * w
        h = vh * (dact * apply_filter_conv(feat, g)[:, 0])
        a_num = (g * g).sum()
        a_den = ((h * h).sum() + (reg + alpha_eps) * a_num).clamp(min=1e-8)
        w = w - (step * (a_num / a_den)) * g
    return w
