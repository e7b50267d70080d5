"""Float64 reference of ONE step of the steepest-descent filter optimisers, and a mirror of the tensor-core kernel's work partition.

`Problem` holds one optimiser problem (sample memory, labels, hyper-parameters) in float64 on the device of its inputs; `step(prob, w)`
evaluates, for a stack of filters w [K, C, 4, 4], the exact step d = alpha * g each of the four modes takes from w, the loss at w and the
per-cell quantities the kink allowance of tests/test_sd_steps_f64_gpu.py needs:

  "gn"      DiMPSteepestDescentGN        (oracle/dimp_oracle.py dimp_sd_gn)
  "newton"  PrDiMPSteepestDescentNewton  (prdimp_sd_newton)
  "l2"      DiMPL2SteepestDescentGN      (dimp_l2_sd_gn)
  "hinge"   GNSteepestDescent over LinearFilterHinge, relu or bentpar activation (gn_sd_hinge)

The label maps come from the oracle's own functions; the apply and adjoint correlations are F.conv2d calls (no window tensor), so the
step of a 50-sample, 512-channel memory costs a few float64 convolutions on the GPU.  tests/test_sd_step_ref_cpu.py pins every mode to
the oracle's num_iter = 1 run.

`tf32=True` rounds the features and w to TF32 (round to nearest, ties away from zero: what `split_tf32_bits` in sd_tc.cu gives as the
high part) before the step is evaluated in float64: the step a single-pass TF32 kernel would be expected to take.

`tc_partition` restates the integer arithmetic of `launch_sd_tc` / `sd_tc_kernel` (part_lo, part_owner, state slots, smax, apply
segments) and lists the partition features a call reaches; `cases()` is the case list of the GPU test, and the CPU test asserts that it
reaches every feature at G = 132."""
import math

import torch
import torch.nn.functional as F

from oracle import dimp_oracle as O

MODES = ("gn", "newton", "l2", "hinge")


def tf32_round(x):
    """Round float32 values to TF32, ties away from zero: bits (u + 0x1000) & 0xffffe000 for finite values, u & 0xffffe000 otherwise."""
    f = x.detach().to(torch.float32).contiguous()
    u = f.view(torch.int32)
    r = torch.where(torch.isfinite(f), (u + 0x1000) & -8192, u & -8192)
    return r.view(torch.float32).to(x.dtype)


class Problem:
    """One optimiser call's fixed data in float64: the sample memory X [n, C, H, W], its zero-padded transpose for the adjoint, the label
    maps and the hyper-parameters.  Inputs are taken as the kernel gets them (float32 values, converted exactly).

    gn:     bb, sample_weight, luts = (label, mask, spatial), step_length, reg, alpha_eps, bin_displacement, feat_stride
    newton: bb, sample_weight, gauss_sigma, step_length, reg, alpha_eps, softmax_reg, label_threshold, normalize_label, label_shrink,
            uni_weight, feat_stride
    l2:     bb, sample_weight, gauss_sigma, hinge_threshold, step_length, reg, alpha_eps, feat_stride
    hinge:  label [n, Ho, Wo], sample_weight, filter_reg, hinge_threshold, activation_leak, score_act, act_param, steplength_reg"""

    def __init__(self, mode, feat, sample_weight=None, **hp):
        assert mode in MODES, mode
        self.mode, self.hp = mode, hp
        d = torch.float64
        self.X = feat.to(d)
        self.n, self.C, self.H, self.W = self.X.shape
        self.OS = (self.H + 1, self.W + 1)
        dev = self.X.device
        n = self.n
        self.sw = None if sample_weight is None else sample_weight.to(d).reshape(n)
        swv = self.sw if self.sw is not None else torch.full((n,), 1.0 / n, dtype=d, device=dev)
        fs = hp.get("feat_stride", 16.0)
        if mode == "gn":
            params = {"label_map_predictor.weight": hp["luts"][0].to(d), "target_mask_predictor.0.weight": hp["luts"][1].to(d),
                      "spatial_weight_predictor.weight": hp["luts"][2].to(d)}
            y, m, v = O.dimp_label_maps(hp["bb"].to(d), params, self.OS, 4, fs, hp.get("bin_displacement", 0.1))
            self.y, self.m, self.vh = y, m, swv.sqrt().view(n, 1, 1) * v
            self.step_length, self.reg, self.eps = hp["step_length"], hp["reg"], hp.get("alpha_eps", 0.0)
        elif mode == "l2":
            bb = hp["bb"].to(d)
            center = ((bb[:, :2] + bb[:, 2:] / 2) / fs).flip((1,))
            k0 = torch.arange(self.OS[0], dtype=d, device=dev).view(1, -1, 1)
            k1 = torch.arange(self.OS[1], dtype=d, device=dev).view(1, 1, -1)
            sg = hp["gauss_sigma"]
            y = torch.exp(-1.0 / (2 * sg ** 2) * (k0 - center[:, 0].view(-1, 1, 1)) ** 2) * \
                torch.exp(-1.0 / (2 * sg ** 2) * (k1 - center[:, 1].view(-1, 1, 1)) ** 2)
            self.label_raw, self.threshold = y, hp["hinge_threshold"]
            self.m = (y > hp["hinge_threshold"]).to(d)
            self.y, self.vh = y * self.m, swv.sqrt().view(n, 1, 1).expand(n, *self.OS)
            self.step_length, self.reg, self.eps = hp["step_length"], hp["reg"], hp.get("alpha_eps", 0.0)
        elif mode == "hinge":
            lab = hp["label"].to(d).reshape(n, *self.OS)
            self.label_raw, self.threshold = lab, hp.get("hinge_threshold", -999.0)
            self.m = ((lab > self.threshold).to(d) + hp.get("activation_leak", 0.0)).clamp(max=1.0)
            self.y, self.vh = self.m * lab, swv.sqrt().view(n, 1, 1).expand(n, *self.OS)
            self.step_length, self.reg, self.eps = 1.0, hp["filter_reg"] ** 2, hp.get("steplength_reg", 0.0)
            self.act, self.act_param = hp.get("score_act", "relu"), hp.get("act_param", 1.0)
            self.numel = n * self.OS[0] * self.OS[1] + self.C * 16
        else:
            self.p = O.prdimp_label_density(hp["bb"].to(d), self.OS, hp["gauss_sigma"], 4, fs, hp.get("label_threshold", 0.0),
                                            hp.get("normalize_label", False), hp.get("label_shrink", 0.0), hp.get("uni_weight", 0.0))
            self.swn = swv
            self.step_length, self.reg, self.eps = hp["step_length"], hp["reg"], hp.get("alpha_eps", 0.0)
            self.softmax_reg = hp.get("softmax_reg")
        self._ops = {}

    def label_margin(self):
        """Smallest |label - threshold| / |threshold| over the maps whose mask jumps at a threshold (l2, hinge; PrDiMP's threshold jumps
        by its own value, so it counts when it is not 0).  inf when no mask depends on a threshold."""
        if self.mode in ("l2", "hinge"):
            lab, thr = self.label_raw, self.threshold
        elif self.mode == "newton" and self.hp.get("label_threshold", 0.0) != 0.0:
            sg = self.hp["gauss_sigma"]
            bb = self.hp["bb"].to(torch.float64)
            lab = O.prdimp_label_density(bb, self.OS, sg, 4, self.hp.get("feat_stride", 16.0), -1.0, False, 0.0, 0.0)
            thr = self.hp["label_threshold"]
        else:
            return math.inf
        return float((lab - thr).abs().min()) / max(abs(thr), 1e-300)

    def operands(self, tf32):
        """(X, X padded and transposed to [C, n, H + 4, W + 4]) in float64, TF32-rounded when asked; cached."""
        if tf32 not in self._ops:
            X = tf32_round(self.X.to(torch.float32)).to(torch.float64) if tf32 else self.X
            self._ops[tf32] = (X, F.pad(X, (2, 2, 2, 2)).transpose(0, 1).contiguous())
        return self._ops[tf32]


def apply(X, w):
    """s[k, i, y, x] = sum_{c,u,v} Xpad[i, c, y+u, x+v] w[k, c, u, v]: [n, C, H, W] x [K, C, 4, 4] -> [K, n, H+1, W+1]."""
    return F.conv2d(X, w, padding=2).transpose(0, 1)


def adjoint(Xt, r):
    """g[k, c, u, v] = sum_{i,y,x} r[k, i, y, x] Xpad[i, c, y+u, x+v]: Xt = Xpad as [C, n, H+4, W+4], r [K, n, H+1, W+1] -> [K, C, 4, 4]."""
    return F.conv2d(Xt, r).transpose(0, 1)


def activation(prob, s):
    """(activation, derivative) of the GN-family modes at scores s."""
    m = prob.m
    if prob.mode == "l2":
        return m * s + (1.0 - m) * F.relu(s), m + (1.0 - m) * (s > 0).to(s.dtype)
    if prob.mode == "hinge" and prob.act == "bentpar":
        b = prob.act_param
        rt = torch.sqrt(s * s + 4.0 * b * b)
        return (1.0 - m) / 2.0 * (rt - 2.0 * b) + (1.0 + m) / 2.0 * s, (1.0 - m) / 2.0 * (s / rt) + (1.0 + m) / 2.0
    return (1.0 - m) / 2.0 * s.abs() + (1.0 + m) / 2.0 * s, (1.0 - m) / 2.0 * torch.sign(s) + (1.0 + m) / 2.0


def flipped_dact(prob, s):
    """The GN-family derivative taken from the other side of its kink at s = 0 (for s = 0: from the positive side)."""
    m = prob.m
    if prob.mode == "l2":
        return m + (1.0 - m) * (s <= 0).to(s.dtype)
    sg = torch.where(s > 0, -torch.ones_like(s), torch.ones_like(s))
    return (1.0 - m) / 2.0 * sg + (1.0 + m) / 2.0


def has_kinks(prob):
    return prob.mode in ("gn", "l2") or (prob.mode == "hinge" and prob.act == "relu")


def step(prob, w, tf32=False, dact=None, ghg_flip=None, detail=False):
    """One optimiser step from each filter of w [K, C, 4, 4] (or [C, 4, 4] / [1, C, 4, 4]), in float64.

    dact [K, n, Ho, Wo]: derivative override of the GN-family modes; ghg_flip [K, n] (bool): Newton's per-sample curvature taken from
    the other side of max(gHg, 0).  Returns a dict with d = alpha g [K, C, 4, 4], loss [K] at w, s [K, n, Ho, Wo], g and alpha.  With
    `detail` also the intermediate maps (r, da, q, h, sm, ghg, gg, curv) that kink_steps / ghg_steps / fp32_bound use, the scale of a
    kernel's score error per cell tau_s = |X| * |w|, the magnitudes g_abs = |X|^T |r'| + reg |w| of the gradient sums and
    qa = |X| * |g| of the A g sums, and loss_abs (the loss's sum of magnitudes)."""
    X, Xt = prob.operands(tf32)
    w = w.to(torch.float64).reshape(-1, prob.C, 4, 4)
    if tf32:
        w = tf32_round(w.to(torch.float32)).to(torch.float64)
    K, n = w.shape[0], prob.n
    s = apply(X, w)
    wsq = (w * w).sum((1, 2, 3))
    out = {"s": s}
    if prob.mode != "newton":
        act, da = activation(prob, s)
        if dact is not None:
            da = dact
        r = prob.vh * (act - prob.y)
        loss = (r * r).sum((1, 2, 3)) + prob.reg * wsq
        if prob.mode == "hinge":
            loss = loss / prob.numel
        rt = da * (prob.vh * r)
        g = adjoint(Xt, rt) + prob.reg * w
        q = apply(X, g)
        h = prob.vh * (da * q)
        curv = (h * h).sum((1, 2, 3))
        out.update(r=r, da=da, h=h, loss_abs=loss)
    else:
        sm = O.softmax_reg(s.reshape(K * n, *prob.OS), prob.softmax_reg).reshape(s.shape)
        sw = prob.swn.view(1, n, 1, 1)
        flat = s.reshape(K, n, -1)
        if prob.softmax_reg is not None:
            flat = torch.cat((flat, torch.full((K, n, 1), float(prob.softmax_reg), dtype=s.dtype, device=s.device)), 2)
        lse = torch.logsumexp(flat, 2)
        ps = (prob.p.unsqueeze(0) * s).sum((2, 3))
        loss = (prob.swn.view(1, n) * (lse - ps)).sum(1) + prob.reg * wsq
        rt = sw * (sm - prob.p)
        g = adjoint(Xt, rt) + prob.reg * w
        q = apply(X, g)
        smq = sm * q
        ghg_raw = (q * (smq - sm * smq.sum((2, 3), keepdim=True))).sum((2, 3))
        ghg = ghg_raw.clamp(min=0)
        if ghg_flip is not None:
            ghg = torch.where(ghg_flip, torch.where(ghg_raw > 0, torch.zeros_like(ghg_raw), ghg_raw), ghg)
        curv = (prob.swn.view(1, n) * ghg).sum(1)
        out.update(sm=sm, ghg=ghg_raw, ghg_used=ghg,
                   loss_abs=(prob.swn.view(1, n) * (lse.abs() + (prob.p.unsqueeze(0) * s.abs()).sum((2, 3)))).sum(1) + prob.reg * wsq)
    gg = (g * g).sum((1, 2, 3))
    alpha = prob.step_length * gg / (curv + (prob.reg + prob.eps) * gg).clamp(min=1e-8)
    out.update(d=alpha.view(K, 1, 1, 1) * g, loss=loss, g=g, alpha=alpha, q=q, gg=gg, curv=curv)
    if detail:
        Xa, Xta = X.abs(), Xt.abs()
        out["tau_s"] = apply(Xa, w.abs())
        out["g_abs"] = adjoint(Xta, rt.abs()) + prob.reg * w.abs()
        out["qa"] = apply(Xa, g.abs())
        if prob.mode == "newton":
            out["tau_ghg"] = (out["sm"] * out["qa"] ** 2).sum((2, 3))
    return out


def kink_steps(prob, ref, k, cells):
    """GN family: the step from filter k of `ref` (a detail step) with the derivative of each cell (i, y, x) of cells [F, 3] taken from
    the other side of its kink, one cell at a time -> [F, C, 4, 4].  Exact by linearity: flipping cell (i, y, x) adds
    c * Xpad[i, :, y:y+4, x:x+4] to g (c = the change of the cell's weighted residual) and c * A(that window) to q."""
    X, Xt = prob.operands(False)
    i, y, x = cells[:, 0], cells[:, 1], cells[:, 2]
    s, da, r = ref["s"][k], ref["da"][k], ref["r"][k]
    da_f = flipped_dact(prob, s)[i, y, x]
    vh = prob.vh[i, y, x]
    c = (da_f - da[i, y, x]) * vh * r[i, y, x]                                   # [F]
    oy = torch.arange(4, device=cells.device)
    win = Xt[:, i.view(-1, 1, 1), (y.view(-1, 1) + oy).view(-1, 4, 1), (x.view(-1, 1) + oy).view(-1, 1, 4)]   # [C, F, 4, 4]
    win = win.transpose(0, 1)
    g = ref["g"][k].unsqueeze(0) + c.view(-1, 1, 1, 1) * win
    q = ref["q"][k].unsqueeze(0) + c.view(-1, 1, 1, 1) * apply(X, win)         # [F, n, Ho, Wo]
    daf = da.unsqueeze(0).repeat(len(c), 1, 1, 1)
    f = torch.arange(len(c), device=cells.device)
    daf[f, i, y, x] = da_f
    h = prob.vh * (daf * q)
    gg = (g * g).sum((1, 2, 3))
    alpha = prob.step_length * gg / ((h * h).sum((1, 2, 3)) + (prob.reg + prob.eps) * gg).clamp(min=1e-8)
    return alpha.view(-1, 1, 1, 1) * g


def ghg_steps(prob, ref, k, samples):
    """Newton: the step from filter k of `ref` with sample i's curvature taken from the other side of max(gHg, 0), for each i of
    samples [F] -> [F, C, 4, 4]."""
    raw, used = ref["ghg"][k, samples], ref["ghg_used"][k, samples]
    other = torch.where(raw > 0, torch.zeros_like(raw), raw)
    curv = ref["curv"][k] + prob.swn[samples] * (other - used)
    gg = ref["gg"][k]
    alpha = prob.step_length * gg / (curv + (prob.reg + prob.eps) * gg).clamp(min=1e-8)
    return alpha.view(-1, 1, 1, 1) * ref["g"][k].unsqueeze(0)


def fp32_bound(prob, ref, depth_g, depth_q, depth_s):
    """Relative bound [K] on max|d error| / max|d| that float32 rounding of a kernel's fixed-order reductions alone can cause: every
    gradient entry summed from partials in a chain of depth_g additions (error <= depth_g u g_abs), every A g cell from depth_q
    partials, and the scalars |g|^2, curvature and loss from chains of depth_s.  Worst-case (linear in depth) bounds."""
    u = 2.0 ** -24
    g, q, qa = ref["g"], ref["q"], ref["qa"]
    dg = depth_g * u * ref["g_abs"]
    dgg = 2 * (g.abs() * dg).sum((1, 2, 3)) + depth_s * u * ref["gg"]
    if prob.mode != "newton":
        dcurv = 2 * depth_q * u * (ref["h"].abs() * prob.vh * ref["da"].abs() * qa).sum((1, 2, 3))
    else:
        sm = ref["sm"]
        dcurv = 4 * depth_q * u * (prob.swn.view(1, -1) * (sm * qa * (qa + (sm * qa).sum((2, 3), keepdim=True))).sum((2, 3))).sum(1)
    dcurv = dcurv + depth_s * u * ref["curv"].abs()
    den = (ref["curv"] + (prob.reg + prob.eps) * ref["gg"]).clamp(min=1e-8)
    dalpha = dgg / ref["gg"] + (dcurv + (prob.reg + prob.eps) * dgg) / den + (depth_s + 4) * u
    bound = ref["alpha"].view(-1, 1, 1, 1) * dg + ref["d"].abs() * dalpha.view(-1, 1, 1, 1)
    return bound.flatten(1).max(1).values / ref["d"].flatten(1).abs().max(1).values


# ---- the tensor-core kernel's work partition (sd_tc.cu) ----------------------------------------------------------------------------
FEATURES = ("empty adjoint range", "run spans 2 CTAs", "run spans >= 3 CTAs", "range crosses a chunk boundary",
            "range starts at a sample boundary", "range starts mid-sample", "apply segment cut by a range boundary",
            "fs18 last box past the image", "fs22 last box partial")


def tc_partition(n, C, fs, G):
    """Partition facts of one sd_tc launch: smax (state slots, as launch_sd_tc computes it), the longest run of apply segments summed per
    sample (qn), the most CTAs contributing to one gradient chunk, and the set of FEATURES reached.  A "run" is the KBT adjoint units of
    one (chunk, sample); the CTAs that hold parts of it each keep a replica of the sample's state, and only the owner adds its loss and
    curvature terms."""
    npx = fs * fs
    kbt, npt, kba, nchk = (npx + 31) // 32, (npx + 127) // 128, C // 32, C // 128
    UT, UA = nchk * n * kbt, n * npt * kba

    def lo(U, b):
        return (U * b) // G

    def owner(U, u):
        return ((u + 1) * G - 1) // U

    feats = set()
    per_chunk = n * kbt
    smax = 1
    for b in range(G):
        a, e = lo(UT, b), lo(UT, b + 1)
        if e <= a:
            feats.add("empty adjoint range")
            continue
        if a // per_chunk != (e - 1) // per_chunk:
            feats.add("range crosses a chunk boundary")
        if b > 0:
            feats.add("range starts at a sample boundary" if a % kbt == 0 else "range starts mid-sample")
        smax = max(smax, len({(u // kbt) % n for u in range(a, e)}))
    for r in range(nchk * n):
        span = owner(UT, (r + 1) * kbt - 1) - owner(UT, r * kbt) + 1
        if span == 2:
            feats.add("run spans 2 CTAs")
        elif span >= 3:
            feats.add("run spans >= 3 CTAs")
    for b in range(1, G):
        a = lo(UA, b)
        if a < UA and a % kba != 0 and lo(UA, b + 1) > a:
            feats.add("apply segment cut by a range boundary")
    qn = max(sum(1 for r in range(npt * kba) if r % kba == 0 or lo(UA, owner(UA, s * npt * kba + r)) == s * npt * kba + r)
             for s in range(n))
    contrib = max(sum(1 for b in range(owner(UT, c * per_chunk), owner(UT, (c + 1) * per_chunk - 1) + 1) if lo(UT, b + 1) > lo(UT, b))
                  for c in range(nchk))
    feats.add("fs18 last box past the image" if fs == 18 else "fs22 last box partial")
    return {"smax": smax, "qn": qn, "contrib": contrib, "features": feats}


# ---- the GPU test's cases ------------------------------------------------------------------------------------------------------------
# (kernel, mode, fs, C, n, sample weights given): kernel "default" = the dispatch the trackers get (tensor cores from 32 samples), "cuda" /
# "tc" force B200TRK_SD_TC=0 / 1.  Modes of section C: "l2", "hinge_relu", "hinge_bent".
def cases():
    out = []
    out += [("default", "gn", 18, 512, n, True) for n in range(1, 51)]                      # A: tracker shapes, every memory fill
    out += [("default", "newton", 22, 512, n, True) for n in range(1, 51)]
    for mode, fs in (("gn", 18), ("newton", 22)):                                            # B: the other kernel
        out += [("cuda", mode, fs, 512, n, True) for n in range(32, 51)]
        out += [("tc", mode, fs, 512, n, True) for n in (1, 2, 5, 9, 16, 31)]
    for mi, mode in enumerate(("l2", "hinge_relu", "hinge_bent")):                           # C: other channel counts and modes
        for fs in (18, 22):
            for ci, (C, n) in enumerate(((128, 7 + 5 * mi), (256, 24 + mi), (384, 45 - 3 * mi))):
                for kernel in ("cuda", "tc"):
                    out.append((kernel, mode, fs, C, n, not (fs == 18 and ci == 0)))
    return out


def kernel_for(kernel, n):
    """"tc" or "cuda": the kernel a case runs on (the default dispatch takes the tensor cores from 32 samples; every case has C % 128 == 0)."""
    if kernel == "default":
        return "tc" if n >= 32 else "cuda"
    return kernel
