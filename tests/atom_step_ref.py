"""Float64 reference of ATOM's filter optimisers step by step, float32 bounds for one step, and a mirror of the CG kernel's launch plan.

Both optimisers reset their state every call (ConjugateGradient with direction_forget_factor = 0; GaussNewtonCG relinearises every GN
iteration), so the float64 result of k CG iterations from a start point is the dtype-preserving oracle run for k iterations on float64
operands: `ConvProblem.step(w, k)` is `atom_cg_filter(..., num_iter=k)`'s delta and `FactorizedProblem.step(w, P, k)` is one
`atom_gn_joint(..., num_cg_iter=k, num_gn_iter=1)` step (dw, dP).  What this module adds:

  * `single_bound`: max|error| / max|d| that float32 rounding can cause in the first CG step d = alpha_0 z_0 (z_0 = M^-1 r_0, alpha_0 =
    <r_0, z_0> / <z_0, A z_0>), first-order, from the summation depth of every reduction the kernel performs (a sum of N terms rounded in
    any order is within (N - 1) u sum|terms| of the exact sum; where the kernel's order is known the depth is its chain length).  The
    score error feeds into the residual and the curvature through phi' and phi''; the GN preconditioner's division by projection_reg
    (1e-4 by default) multiplies the P block's errors by 10^4 and is part of the propagation.
  * `kink_cells` / `kink_allowance`: relu and mlu change their derivative (mlu its second derivative) at s = 0; a cell whose float64
    score lies within 2^-16 (|X| * |w|) of 0 may fall on either side in a kernel.  The allowance is the sum over those cells of |d_flip -
    d|, d_flip the k-iteration step with that one cell's derivative taken from the other side.
  * `step32` / `e32`: the same k iterations in float32 with the channels permuted (another summation order), e_f32(k) = max|d_32 - d| /
    max|d| over two orders: the float32 accuracy the problem's conditioning allows after k iterations.  The worst-case bound above is
    10^3-10^4 times the error float32 actually makes (it sums |terms| over thousands of terms of both signs), so the tests also hold a
    kernel to F32_FACTOR * e_f32(k): that is the bar that catches an error of 10^-4 in a step.
  * `cg_plan(n, C, FS, sms)`: the integer arithmetic of launch_cg (csrc/atom_cg.cu): channel passes, channel chunks NCH, sample groups
    NG, samples per CTA spc and pipeline depth NST; `plan_features` names what a plan reaches."""
import math

import torch

from oracle import atom_oracle as A

U = 2.0 ** -24
TAU = 2.0 ** -16
CG_SPC_MAX = 8
F32_FACTOR = 16


# ---- launch_cg's plan ------------------------------------------------------------------------------------------------------------------
def corr2(fs):
    """Corr2<FS>'s constants (csrc/corr2.cuh)."""
    os_ = fs + 1
    nty, ntx = (os_ + 4) // 5, (os_ + 3) // 4
    rows0 = nty * 5 + 3
    rows = rows0 if rows0 & 1 else rows0 + 1
    return dict(OS=os_, NPOS=os_ * os_, NT=nty * ntx, SLOTS=16, ITEM_FLOATS=16 * rows * 28, PMAP=nty * 5 * ntx * 4, NCONS=nty * ntx * 16,
                VEC_STRIDE=20, RED_STRIDE=17)


def cg_plan(n, C, fs, sms):
    """launch_cg's choice for n samples of C channels at FS x FS on `sms` SMs: dict(passes, NCH, NG, spc, NST), or None when the launcher
    refuses the problem (no channel split keeps a CTA's samples within CG_SPC_MAX, or the samples do not fit shared memory)."""
    K = corr2(fs)
    for p in (1, 2, 4):
        if C % (K["SLOTS"] * p):
            continue
        nch = C // (K["SLOTS"] * p)
        if nch > sms:
            continue
        ng = max(1, min(sms // nch, n))
        spc = (n + ng - 1) // ng
        if spc <= CG_SPC_MAX:
            break
    else:
        return None
    cchunk = p * K["SLOTS"]
    fixed = 4 * (K["NT"] * K["SLOTS"] * K["RED_STRIDE"] + 6 * cchunk * K["VEC_STRIDE"] + spc * (2 * K["NPOS"] + K["PMAP"]) + K["NCONS"] * 4)
    limit, item = 227 * 1024 - 512, 4 * K["ITEM_FLOATS"]
    nst = next((s for s in (4, 3, 2) if fixed + s * item <= limit), None)
    if nst is None:
        return None
    return dict(passes=p, NCH=nch, NG=ng, spc=spc, NST=nst)


PLAN_FEATURES = ("NCH = 1", "NCH > 1", "passes 1", "passes 2", "passes 4", "NG = n", "NG < n, uneven groups", "spc = CG_SPC_MAX",
                 "n = NG * CG_SPC_MAX", "NST 4", "NST 3", "NST 2", "FS 18", "FS 22")


def plan_features(n, C, fs, sms):
    pl = cg_plan(n, C, fs, sms)
    f = {"NCH = 1" if pl["NCH"] == 1 else "NCH > 1", "passes %d" % pl["passes"], "NST %d" % pl["NST"], "FS %d" % fs}
    if pl["NG"] == n:
        f.add("NG = n")
    elif n % pl["NG"]:
        f.add("NG < n, uneven groups")
    if pl["spc"] == CG_SPC_MAX:
        f.add("spc = CG_SPC_MAX")
        if n == pl["NG"] * CG_SPC_MAX:
            f.add("n = NG * CG_SPC_MAX")
    return f


def cg_depths(n, C, fs, sms):
    """Chain depths of the CG kernel's float32 sums under its plan: score cells (the chunk's 16-tap x cchunk-channel sweep, then the
    NCH-way ordered_sum), gradient entries (a CTA's spc x NPOS transpose sweep, the NG-way reduce_groups, + reg p) and the inner products
    (ceil(E / NTH) per thread, the block tree, the NCH-way exchange).  corr2.cuh: a thread of the apply sweep chains the 16 taps of its
    channel slot over the passes, then a 16-slot butterfly; a thread of the transpose sweep chains its tile's 20 cells over the CTA's
    samples, then the NT tiles are summed."""
    pl, K = cg_plan(n, C, fs, sms), corr2(fs)
    cchunk = pl["passes"] * 16
    ds = 16 * pl["passes"] + 4 + pl["NCH"]
    dg = pl["spc"] * 20 + K["NT"] + pl["NG"] + 2
    dip = -(-16 * cchunk // K["NCONS"]) + math.ceil(math.log2(K["NCONS"])) + pl["NCH"] + 1
    return ds, dg, dip


# ---- activations ----------------------------------------------------------------------------------------------------------------------
def dact2_abs(s, act, param):
    """|phi''(s)| away from the kink (what a score error does to phi')."""
    if act == "elu":
        return torch.where(s > 0, torch.zeros_like(s), torch.exp(s))
    if act == "mlu":
        return torch.where(s >= 0, torch.zeros_like(s), torch.exp(s / param) / param)
    return torch.zeros_like(s)


def flipped_dact(s, act, param):
    """phi'(s) taken from the other side of s = 0 (relu, mlu)."""
    if act == "relu":
        return (s <= 0).to(s.dtype)
    if act == "mlu":
        return torch.where(s >= 0, torch.exp(s / param), torch.ones_like(s))
    raise ValueError(act)


def _apply(X, w):
    """conv 'same' of the oracle, full (FS + 1)^2 map cropped: [n, C, H, W] x [1, C, 4, 4] -> [n, 1, H, W]."""
    return A.conv_same(X, w)


def _adj(X, u):
    return A.conv_same_adjoint_filter(X, u, 4)


def _ip(a, b):
    return float((a * b).sum())


def _step_bound(r, er, m, q_of, eq_of, dip):
    """Shared tail of the single-step bound, first order.  r: exact residual blocks, er: bounds of their float32 errors, m: the
    preconditioner's factor per block (z = M^-1 r), q_of: z -> exact q = A z, eq_of: z -> bound of the rounding of q's sums (q computed
    from an exact z), dip: inner-product depth.  An error dz of z moves rho = <r, z> by 2 <z, dr> and sigma = <z, A z> by 2 <A z, dz> (A
    symmetric): those are bounded through |z| er and |q| ez, not through |A|."""
    z = [m_ * r_ for m_, r_ in zip(m, r)]
    ez = [m_ * e_ + U * z_.abs() for m_, e_, z_ in zip(m, er, z)]
    q, eq = q_of(z), eq_of(z)
    rho = sum(_ip(r_, z_) for r_, z_ in zip(r, z))
    sig = sum(_ip(z_, q_) for z_, q_ in zip(z, q))
    erho = sum(2 * _ip(z_.abs(), e_) + dip * U * _ip(r_.abs(), z_.abs()) for r_, z_, e_ in zip(r, z, er))
    esig = sum(2 * _ip(q_.abs(), e_) + _ip(z_.abs(), f_) + dip * U * _ip(z_.abs(), q_.abs()) for z_, q_, e_, f_ in zip(z, q, ez, eq))
    alpha = rho / sig
    ea = abs(alpha) * (erho / abs(rho) + esig / abs(sig) + 2 * U)
    d = [alpha * z_ for z_ in z]
    ed = [abs(alpha) * e_ + ea * z_.abs() + U * d_.abs() for e_, z_, d_ in zip(ez, z, d)]
    return d, ed


# ---- ConvProblem (per-frame CG) -------------------------------------------------------------------------------------------------------
class ConvProblem:
    """One atom_cg_filter call's data in float64.  Samples with zero weight contribute nothing to any sum (their terms are exactly 0) and
    are dropped from the float64 evaluation; the kernel's summation depths still count them (they come from `plan`)."""

    def __init__(self, X, y, sw, reg, act="mlu", act_param=0.05, fletcher_reeves=False):
        sw = sw.reshape(-1)
        keep = torch.nonzero(sw > 0).reshape(-1).cpu()
        d = torch.float64
        self.n_all, self.C, self.FS = X.shape[0], X.shape[1], X.shape[-1]
        self.X32, self.y32, self.sw32 = (t.detach().cpu().float()[keep].contiguous() for t in (X, y.reshape(X.shape[0], 1, self.FS, self.FS), sw))
        self.X, self.y, self.sw = self.X32.to(d), self.y32.to(d), self.sw32.to(d)
        self.reg, self.act, self.param, self.fr = float(reg), act, float(act_param), bool(fletcher_reeves)

    def step(self, w, k, dact=None):
        """Float64 delta of k CG iterations from w."""
        w = w.detach().cpu().reshape(1, self.C, 4, 4).double()
        return A.atom_cg_filter(w, self.X, self.y, self.sw, self.reg, k, self.act, self.param, self.fr, dact=dact)[1]

    def step32(self, w, k, seed=0):
        """The same k iterations in float32 with the channels permuted (another summation order of every channel sum)."""
        perm = torch.randperm(self.C, generator=torch.Generator().manual_seed(seed))
        w = w.detach().cpu().reshape(1, self.C, 4, 4).float()
        d = A.atom_cg_filter(w[:, perm].contiguous(), self.X32[:, perm].contiguous(), self.y32, self.sw32, self.reg, k, self.act,
                             self.param, self.fr)[1]
        out = torch.empty_like(d)
        out[:, perm] = d
        return out.double()

    def e32(self, w, k, ref):
        """e_f32(k): the larger error of two float32 runs with different channel orders against the float64 step ref."""
        return max(float((self.step32(w, k, seed) - ref).abs().max() / ref.abs().max()) for seed in (0, 1))

    def kink_cells(self, w):
        if self.act not in ("relu", "mlu"):
            return torch.zeros(0, 4, dtype=torch.long)
        w = w.detach().cpu().reshape(1, self.C, 4, 4).double()
        s = _apply(self.X, w)
        return torch.nonzero(s.abs() <= TAU * _apply(self.X.abs(), w.abs()))

    def kink_allowance(self, w, k, cells, ref=None):
        """Per entry: sum over cells of |d_k with that cell's phi' from the other side - d_k|."""
        w64 = w.detach().cpu().reshape(1, self.C, 4, 4).double()
        ref = self.step(w, k) if ref is None else ref
        out = torch.zeros_like(ref)
        if len(cells) == 0:
            return out
        s = _apply(self.X, w64)
        d0 = A.activation_deriv(s, self.act, self.param)
        fl = flipped_dact(s, self.act, self.param)
        for c in cells:
            i, _, yy, xx = c.tolist()
            dd = d0.clone()
            dd[i, 0, yy, xx] = fl[i, 0, yy, xx]
            out += (self.step(w, k, dact=dd) - ref).abs()
        return out

    def single_bound(self, w, depths):
        """Relative float32 bound on the first CG step from w for the depths (ds, dg, dip) of `cg_depths`."""
        ds, dg, dip = depths
        X, Xa, y, swv = self.X, self.X.abs(), self.y, self.sw.view(-1, 1, 1, 1)
        w = w.detach().cpu().reshape(1, self.C, 4, 4).double()
        s = _apply(X, w)
        es = ds * U * _apply(Xa, w.abs())
        a, d = A.activation(s, self.act, self.param), A.activation_deriv(s, self.act, self.param)
        d2 = dact2_abs(s, self.act, self.param)
        u0 = swv * d * (a - y)
        eu0 = swv * (d * d + d2 * (a - y).abs()) * es + 4 * U * u0.abs()
        b = -(_adj(X, u0) + self.reg * w)
        eb = _adj(Xa, eu0) + dg * U * (_adj(Xa, u0.abs()) + self.reg * w.abs())
        D = swv * d * d
        eD = swv * 2 * d.abs() * d2 * es + 2 * U * D

        def q_of(z):
            return [_adj(X, D * _apply(X, z[0])) + self.reg * z[0]]

        def eq_of(z):
            Ap = _apply(X, z[0])
            t = D * Ap
            et = eD * Ap.abs() + D * ds * U * _apply(Xa, z[0].abs()) + U * t.abs()
            return [_adj(Xa, et) + dg * U * (_adj(Xa, t.abs()) + self.reg * z[0].abs())]

        d, ed = _step_bound([b], [eb], [1.0], q_of, eq_of, dip)
        return float(ed[0].max() / d[0].abs().max())


# ---- FactorizedConvProblem (first-frame Gauss-Newton) ---------------------------------------------------------------------------------
class FactorizedProblem:
    """One atom_gn_joint_ call's data in float64 (projection_activation = identity, as ATOM uses it)."""

    def __init__(self, X, y, sw, reg_w, reg_P, act="mlu", act_param=0.05, fletcher_reeves=True):
        d = torch.float64
        self.X32, self.y32, self.sw32 = (t.detach().cpu().float().contiguous() for t in (X, y, sw.reshape(-1)))
        self.X, self.y, self.sw = self.X32.to(d), self.y32.to(d).reshape(X.shape[0], 1, X.shape[-2], X.shape[-1]), self.sw32.to(d)
        self.n, self.Cin, self.FS = X.shape[0], X.shape[1], X.shape[-1]
        self.reg_w, self.reg_P, self.act, self.param, self.fr = float(reg_w), float(reg_P), act, float(act_param), bool(fletcher_reeves)

    def step(self, w, P, k):
        """Float64 (dw, dP) of one GN iteration with k CG iterations from (w, P)."""
        w, P = w.detach().cpu().double(), P.detach().cpu().double()
        w1, P1 = A.atom_gn_joint(w, P, self.X, self.y, self.sw, self.reg_w, self.reg_P, k, 1, self.act, self.param, self.fr)
        return w1 - w, P1 - P

    def step32(self, w, P, k, seed=0):
        """The same GN step in float32 with the compressed and the input channels permuted."""
        g = torch.Generator().manual_seed(seed)
        pc, pi = torch.randperm(w.shape[1], generator=g), torch.randperm(self.Cin, generator=g)
        w, P = w.detach().cpu().float(), P.detach().cpu().float().reshape(w.shape[1], self.Cin, 1, 1)
        wp, Pp = w[:, pc].contiguous(), P[pc][:, pi].contiguous()
        w1, P1 = A.atom_gn_joint(wp, Pp, self.X32[:, pi].contiguous(), self.y32.reshape(self.y.shape), self.sw32, self.reg_w, self.reg_P, k, 1,
                                 self.act, self.param, self.fr)
        dw, dP = torch.empty_like(w), torch.empty_like(P)
        dw[:, pc] = w1 - wp
        dP[pc.view(-1, 1), pi.view(1, -1)] = P1 - Pp
        return dw.double(), dP.double()

    def single_bound(self, w, P):
        """Relative float32 bounds (w block, P block) on the first CG step of a GN iteration from (w, P): sums bounded by their term
        counts -- conv1x1 Cin, conv2d_same 16 Cc, apply_feat_transpose n (FS + 1)^2, the expand 16 and gn_txt / the per-sample reduction
        n FS^2 -- and the inner products by the N = 16 Cc + Cc Cin terms of gn_init / gn_step's block reduction."""
        X, Xa, y, swv = self.X, self.X.abs(), self.y, self.sw.view(-1, 1, 1, 1)
        w, P = w.detach().cpu().double(), P.detach().cpu().double()
        Cc, FS, n = w.shape[1], self.FS, self.n
        HW = FS * FS
        comp = A.conv1x1(X, P)
        ecomp = self.Cin * U * A.conv1x1(Xa, P.abs())
        compa = comp.abs()
        s = A.conv_same(comp, w)
        es = 16 * Cc * U * A.conv_same(compa, w.abs()) + A.conv_same(ecomp, w.abs())
        a, d = A.activation(s, self.act, self.param), A.activation_deriv(s, self.act, self.param)
        d2 = dact2_abs(s, self.act, self.param)
        D = swv * d * d
        eD = swv * 2 * d.abs() * d2 * es + 2 * U * D
        u0 = swv * d * (a - y)
        eu0 = swv * (d * d + d2 * (a - y).abs()) * es + 4 * U * u0.abs()
        dgw, dgP = n * (FS + 1) ** 2 + 1, 16 + HW + n + 1

        def JT(u):
            return A.conv_same_adjoint_filter(comp, u, 4), torch.einsum("ncp,nkp->ck", A.conv_same_adjoint_input(u, w, FS, FS).flatten(2),
                                                                            X.flatten(2)).reshape(P.shape)

        def eJT(u, eu):
            gw = _adj(compa, eu) + _adj(ecomp, u.abs()) + dgw * U * _adj(compa, u.abs())
            Ta = A.conv_same_adjoint_input(u.abs(), w.abs(), FS, FS)
            eT = A.conv_same_adjoint_input(eu, w.abs(), FS, FS) + 16 * U * Ta
            gP = torch.einsum("ncp,nkp->ck", eT.flatten(2), Xa.flatten(2)) + dgP * U * torch.einsum("ncp,nkp->ck", Ta.flatten(2), Xa.flatten(2))
            return gw, gP.reshape(P.shape)

        gw, gP = JT(u0)
        egw, egP = eJT(u0, eu0)
        r = [-(gw + self.reg_w * w), -(gP + self.reg_P * P)]
        er = [egw + U * (gw.abs() + self.reg_w * w.abs()), egP + U * (gP.abs() + self.reg_P * P.abs())]

        def Jv(z):
            return A.conv_same(comp, z[0]) + A.conv_same(A.conv1x1(X, z[1]), w)

        def q_of(z):
            qw, qP = JT(D * Jv(z))
            return [qw + self.reg_w * z[0], qP + self.reg_P * z[1]]

        def eq_of(z):
            t1a = A.conv_same(compa, z[0].abs())
            t2a = A.conv_same(A.conv1x1(Xa, z[1].abs()), w.abs())
            e_jv = A.conv_same(ecomp, z[0].abs()) + 16 * Cc * U * t1a + (self.Cin + 16 * Cc) * U * t2a + U * (t1a + t2a)
            jv = Jv(z)
            t = D * jv
            et = eD * jv.abs() + D * e_jv + U * t.abs()
            qw, qP = JT(t)
            eqw, eqP = eJT(t, et)
            return [eqw + U * (qw.abs() + self.reg_w * z[0].abs()), eqP + U * (qP.abs() + self.reg_P * z[1].abs())]

        N = Cc * 16 + Cc * self.Cin
        dd, ed = _step_bound(r, er, [1.0 / self.reg_w, 1.0 / self.reg_P], q_of, eq_of, -(-N // 1024) + 12)
        return float(ed[0].max() / dd[0].abs().max()), float(ed[1].max() / dd[1].abs().max())
