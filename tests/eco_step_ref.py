"""Float64 reference of ECO's two Fourier-domain optimisers step by step, float32 bounds for one step, and their launch plans.

A kernel call's step is its output minus its input, exact in float64; the reference step is the float64 oracle (oracle/eco_oracle.py
filter_optim_run / joint_gn_run) run from the same float32 start, on float64 copies of the same operands, with the scalar parameters
rounded to float32 as the kernel receives them.  What this module adds:

  * `FilterProblem` (eco_filter_cg_): `step` -- the filter step, the exported CG state (p, r_prev, rho) and the sample energy of k CG
    iterations from a start and a carried state; `single_bound` -- the first-order float32 bound on one iteration, built from the
    summation depth of every reduction as eco_cg_kernel.cuh sums it under its plan: the forward product over C (CPL serial terms, then
    log2 G shuffle levels), the adjoint over N (N / GPP rows per lane group, the regularisation taps in the same chain, GPP shared-memory
    partials), inner_prod_fs (a thread's serial sum over the CTA's elements, block_sum, the warp sum over the nb CTA partials) and the
    division by diag_M (whose channel mean is a sum of C terms); `step32` / `e32` -- the same iterations in float32 with the channel and
    the sample order permuted (both exact symmetries of the problem), e_f32 = the larger error of two such runs against float64.
  * `JointProblem` (eco_joint_gn_): one GN iteration with k CG iterations from (hf, P) with a given preconditioner, its float32 runs
    with permuted channels / input channels / samples, and the single-step bound of its first CG step (the compressed samples c0 = X P
    and their rounding, the data residual, the two adjoints, the projection gradient's coefficient sum split SPL ways, the P block
    divided by diag_M_proj).
  * `plan_features` / `joint_plan_features`: what a plan of pytracking_b200/eco_plan.py (the kernels' own plan arithmetic restated)
    reaches.

Errors are bounded per complex entry on its modulus (a component sum of K complex products is within K u sum |a||b| of the exact one,
sqrt 2 for the modulus).  The worst-case bound is orders of magnitude above what float32 really does, so the tests also hold every
step to F32_FACTOR * e_f32."""
import math

import torch

from oracle import eco_oracle as E
from pytracking_b200.eco_plan import BLOCK, eco_joint_plan, eco_plan

U = 2.0 ** -24
F32_FACTOR = 16
S2 = math.sqrt(2.0)


def f32(v):
    return float(torch.tensor(float(v), dtype=torch.float32))


# ---- plans ---------------------------------------------------------------------------------------------------------------------------
PLAN_FEATURES = ("G 16", "G 32", "CPL 1", "CPL 2", "CPL 4", "GPP 1", "GPP 2", "GPP 4", "GPP 8", "GPP 16", "residency full",
                 "residency partial", "residency none", "grid < SMs", "uneven coefficient ranges", "N % (4 GPP) != 0")


def plan_features(H, Wh, N, C, sms):
    pl = eco_plan(H, Wh, N, C, 1, sms)
    f = {"G %d" % pl["G"], "CPL %d" % pl["CPL"], "GPP %d" % pl["GPP"]}
    f.add("residency full" if pl["res_slabs"] >= pl["npx_max"] else "residency partial" if pl["res_slabs"] else "residency none")
    if pl["grid"] < sms:
        f.add("grid < SMs")
    if (H * Wh) % pl["grid"]:
        f.add("uneven coefficient ranges")
    if N % (4 * pl["GPP"]):
        f.add("N % (4 GPP) != 0")
    return f


def plan_label(pl):
    return "grid %d G %d CPL %d GPP %d res %d/%d" % (pl["grid"], pl["G"], pl["CPL"], pl["GPP"], pl["res_slabs"], pl["npx_max"])


JOINT_PLAN_FEATURES = ("wide 0", "wide 1", "stage_pm 0", "stage_pm 1", "residency full", "residency partial", "residency none", "SPL 1",
                       "SPL > 1", "several tiles per CTA", "grid < SMs")


def joint_plan_features(H, Wh, N, Cin, C, sms):
    pl = eco_joint_plan(H, Wh, N, Cin, C, 1, 1, sms)
    f = {"wide %d" % pl["wide"], "stage_pm %d" % pl["stage_pm"], "SPL 1" if pl["SPL"] == 1 else "SPL > 1"}
    f.add("residency full" if pl["res_slabs"] >= pl["npx_max"] else "residency partial" if pl["res_slabs"] else "residency none")
    if -(-Cin * C // pl["EPB"]) > pl["grid"]:
        f.add("several tiles per CTA")
    if pl["grid"] < sms:
        f.add("grid < SMs")
    return f


def joint_plan_label(pl):
    return "grid %d wide %d stage_pm %d res %d/%d EPB %d SPL %d" % (pl["grid"], pl["wide"], pl["stage_pm"], pl["res_slabs"], pl["npx_max"],
                                                                  pl["EPB"], pl["SPL"])


# ---- complex helpers ------------------------------------------------------------------------------------------------------------------
def mag(t):
    return (t[..., 0] ** 2 + t[..., 1] ** 2).sqrt()


def cplx(m):
    return torch.stack((m, torch.zeros_like(m)), -1)


def kw_of(Wh, like):
    w = torch.full((Wh,), 2.0, dtype=like.dtype, device=like.device)
    w[0] = 1.0
    return w


def nz_taps(reg):
    """Non-zero taps of the composite filter W (*) W the kernels compact."""
    r = reg.reshape(1, 1, *reg.shape[-2:]).double().cpu()
    return int((torch.nn.functional.conv2d(r, r.flip((2, 3)), padding=(r.shape[-2] - 1, r.shape[-1] - 1)) != 0).sum())


def _cpu32(t):
    return None if t is None else t.detach().float().contiguous()


# ---- eco_filter_cg_ -------------------------------------------------------------------------------------------------------------------
class FilterProblem:
    """One eco_filter_cg_ call's fixed operands.  Zero-weight samples contribute exactly nothing to any sum and are dropped from the
    float64 evaluation (the kernel's summation depths still count all N rows).  `dev`: where the oracle runs (float64 on the GPU is as
    good as on the CPU, and much faster at ECO's block sizes)."""

    def __init__(self, samples, yf, sw, reg, fletcher_reeves=False, standard_alpha=True, dff=0.0, lr=0.0075, pdp=0.3, prp=0.15, dev="cpu"):
        self.dev = dev
        sw = sw.reshape(-1)
        keep = torch.nonzero(sw.cpu() > 0).reshape(-1)
        self.H, self.Wh, self.N, self.C = samples.shape[0], samples.shape[1], samples.shape[2], samples.shape[3]
        self.X32 = _cpu32(samples).to(dev)[:, :, keep.to(dev)].contiguous()
        self.sw32 = _cpu32(sw).to(dev)[keep.to(dev)].contiguous()
        self.yf32 = _cpu32(yf).to(dev).reshape(1, 1, self.H, self.Wh)
        self.reg32 = _cpu32(reg).to(dev).reshape(1, 1, *reg.shape[-2:])
        self.X, self.sw, self.yf, self.reg = (t.double() for t in (self.X32, self.sw32, self.yf32, self.reg32))
        self.fr, self.sa = bool(fletcher_reeves), bool(standard_alpha)
        self.kw = dict(precond_learning_rate=f32(lr), precond_data_param=f32(pdp), precond_reg_param=f32(prp), fletcher_reeves=self.fr,
                       standard_alpha=self.sa, direction_forget_factor=f32(dff))
        self.dff = f32(dff)
        self.nz = nz_taps(reg)

    def _state(self, state, dt, perm=None):
        """The oracle's state from a kernel state dict (None / no p: no direction)."""
        if not state or state.get("p") is None or self.dff == 0 or float(state["rho"].reshape(-1)[0]) == 0.0:
            return {}
        pc = (lambda t: t) if perm is None else (lambda t: t[:, perm].contiguous())
        p = pc(_cpu32(state["p"]).to(self.dev).to(dt))
        rp = None if self.fr or state.get("r_prev") is None else pc(_cpu32(state["r_prev"]).to(self.dev).to(dt))
        return {"p": p, "r_prev": rp, "rho": float(state["rho"].reshape(-1)[0])}

    def run(self, hf, energy, state, k, new_xf, dt=torch.float64, perm=None):
        """k iterations of the oracle in dtype dt from float32 operands; perm = (channel permutation, sample permutation) or None.
        Returns dict(hf, energy, p, r_prev, rho) in the caller's channel order."""
        d = lambda t: None if t is None else _cpu32(t).to(self.dev).to(dt)
        X, sw, yf, reg = d(self.X32), d(self.sw32), d(self.yf32), d(self.reg32)
        hf, en, nx = d(hf).reshape(1, self.C, self.H, self.Wh, 2), d(energy), d(new_xf)
        en = None if en is None else en.reshape(1, self.C, self.H, self.Wh)
        nx = None if nx is None else nx.reshape(1, self.C, self.H, self.Wh, 2)
        pc = None
        if perm is not None:
            pc, pn = (q.to(self.dev) for q in perm)
            X, sw = X[:, :, pn][:, :, :, pc].contiguous(), sw[pn].contiguous()
            hf = hf[:, pc].contiguous()
            en = None if en is None else en[:, pc].contiguous()
            nx = None if nx is None else nx[:, pc].contiguous()
        st = self._state(state, dt, pc)
        x, en1, st1 = E.filter_optim_run(hf, X, yf, sw, reg, en, st, k, nx, **self.kw)
        out = {"hf": x, "energy": en1, "p": st1.get("p"), "r_prev": st1.get("r_prev"), "rho": st1.get("rho")}
        if pc is not None:
            inv = torch.argsort(pc)
            out = {key: (v[:, inv] if torch.is_tensor(v) and v.dim() >= 4 else v) for key, v in out.items()}
        return out

    def step(self, hf, energy, state, k, new_xf):
        r = self.run(hf, energy, state, k, new_xf)
        r["d"] = r["hf"] - _cpu32(hf).to(self.dev).double().reshape(r["hf"].shape)
        return r

    def e32(self, hf, energy, state, k, new_xf, ref):
        """e_f32 of the filter step and of p, r_prev, rho: the larger error of two float32 runs in other channel and sample orders."""
        out = {}
        g = torch.Generator().manual_seed(17)
        for _ in range(2):
            perm = (torch.randperm(self.C, generator=g), torch.randperm(self.X32.shape[2], generator=g))
            r = self.run(hf, energy, state, k, new_xf, torch.float32, perm)
            r["d"] = r["hf"].double() - _cpu32(hf).to(self.dev).double().reshape(r["hf"].shape)
            for key in ("d", "p", "r_prev", "rho"):
                if ref.get(key) is None:
                    continue
                out[key] = max(out.get(key, 0.0), rel_err(r[key], ref[key]))
        return out

    # -- the single-iteration bound ----------------------------------------------------------------------------------------------------
    def depths(self, sms):
        pl = eco_plan(self.H, self.Wh, self.N, self.C, 1, sms)
        G, CPL, GPP = pl["G"], pl["CPL"], pl["GPP"]
        ds = CPL + int(math.log2(G)) + 2
        da = -(-self.N // GPP) + -(-self.nz // GPP) + GPP + 2
        db = -(-self.N // GPP) + GPP + 2
        dip = -(-pl["npx_max"] * self.C // BLOCK) + 13 + -(-pl["grid"] // 32) + 5 + 2
        return pl, ds, da, db, dip

    def _data_abs(self, m):
        """sum_n sw_n |X_n,c| sum_c' |X_n,c'| m_c'   (m [1,C,H,Wh] >= 0)."""
        M = mag(self.X)                                                              # [H,Wh,n,C]
        s = torch.einsum("hwnc,chw->hwn", M, m[0])
        return torch.einsum("hwnc,hwn->chw", M, s * self.sw.view(1, 1, -1)).unsqueeze(0)

    def _reg_abs(self, m):
        return E.reg_term(cplx(m), self.reg.abs())[..., 0].clamp(min=0)

    def single_bound(self, hf, energy, state, new_xf, sms):
        """Relative float32 bounds of one CG iteration from (hf, energy, state): dict(d, p, r_prev, rho)."""
        pl, ds, da, db, dip = self.depths(sms)
        rr = self.reg.shape[-2] * self.reg.shape[-1]
        X, sw, yf, reg = self.X, self.sw, self.yf, self.reg
        C, H, Wh = self.C, self.H, self.Wh
        x = _cpu32(hf).to(self.dev).double().reshape(1, C, H, Wh, 2)
        kw = kw_of(Wh, x).view(1, 1, 1, -1)

        def ip(a, b):                                                                # weighted sums of magnitudes
            return float((kw * a * b).sum())

        def eA(m):                                                                   # rounding of A v's sums for an exact v, |v| = m
            return S2 * U * ((ds + da + 1) * self._data_abs(m) + (da + rr + 1) * self._reg_abs(m))

        def absA(m):                                                                 # |A| applied to an error bound
            return self._data_abs(m) + self._reg_abs(m)

        en = None if energy is None else _cpu32(energy).to(self.dev).double().reshape(1, C, H, Wh)
        nx = None if new_xf is None else _cpu32(new_xf).to(self.dev).double().reshape(1, C, H, Wh, 2)
        lr, pdp, prp = self.kw["precond_learning_rate"], self.kw["precond_data_param"], self.kw["precond_reg_param"]
        if nx is not None:
            e = (nx * nx).sum(-1)
            en = e if en is None else (1 - lr) * en + lr * e
        dM = E.diag_M(en, pdp, prp, reg.reshape(-1) @ reg.reshape(-1))
        edM = (C + rr + 16) * U                                                      # relative: energy update, channel mean, reg_energy
        b = E.rhs(X, sw, yf)
        Ax = E.apply_A(x, X, sw, reg)
        r = b - Ax
        sxa = torch.einsum("hwnc,n->chw", mag(X), sw).unsqueeze(0)
        e_r = S2 * U * db * yf.abs() * sxa + U * mag(b) + eA(mag(x)) + U * mag(r)
        mr = mag(r)
        z = r / dM.unsqueeze(-1)
        mz = mag(z)
        e_z = e_r / dM + mz * (edM + U)
        rho = ip(mr, mz)
        e_rho = ip(mz, e_r) + ip(mr, e_z) + dip * U * rho
        st = self._state(state, torch.float64)
        if st:
            p0 = st["p"]
            mp0 = mag(p0)
            rho1 = st["rho"] / self.dff
            e_rho1 = U * abs(rho1)
            num, e_num = rho, e_rho
            if not self.fr:
                rp = st["r_prev"]
                rho2 = float((kw.unsqueeze(-1) * rp * z).sum())
                num = rho - rho2
                e_num = e_rho + ip(mag(rp), e_z) + dip * U * ip(mag(rp), mz) + U * abs(num)
            beta = num / rho1
            e_beta = e_num / abs(rho1) + abs(beta) * (e_rho1 / abs(rho1) + U)
            if beta < 0:
                beta, e_beta = 0.0, max(0.0, beta + e_beta)
            p = z + beta * p0
            e_p = e_z + e_beta * mp0 + U * (beta * mp0 + mag(p))
        else:
            p, e_p = z, e_z
        mp = mag(p)
        Ap = E.apply_A(p, X, sw, reg)
        mAp = mag(Ap)
        pq = float((kw.unsqueeze(-1) * p * Ap).sum())
        e_pq = ip(mAp, e_p) + ip(mp, absA(e_p)) + ip(mp, eA(mp)) + dip * U * ip(mp, mAp)
        if self.sa:
            alpha = rho / pq
            e_alpha = abs(alpha) * (e_rho / abs(rho) + e_pq / abs(pq) + U)
        else:
            pr = float((kw.unsqueeze(-1) * p * r).sum())
            e_pr = ip(mr, e_p) + ip(mp, e_r) + dip * U * ip(mp, mr)
            alpha = pr / pq
            e_alpha = abs(alpha) * (e_pr / abs(pr) + e_pq / abs(pq) + U)
        d = alpha * p
        e_d = abs(alpha) * e_p + e_alpha * mp + U * mag(d)
        out = {"d": float(e_d.max() / mag(d).max()), "p": float(e_p.max() / mp.max()), "rho": e_rho / abs(rho)}
        if not self.fr:
            out["r_prev"] = float(e_r.max() / mr.max())
        return out


def rel_err(k, ref, allow=None):
    """max(|k - ref| - allow, 0) / max|ref| (tensors or scalars)."""
    if not torch.is_tensor(ref):
        return abs(float(k) - float(ref)) / abs(float(ref))
    k = k.detach().to(ref.device).double().reshape(ref.shape)
    e = (k - ref).abs()
    if allow is not None:
        e = (e - allow).clamp(min=0)
    return float(e.max() / ref.abs().max())


# ---- eco_joint_gn_ --------------------------------------------------------------------------------------------------------------------
class JointProblem:
    """One eco_joint_gn_ call's fixed operands: samples [H,Wh,N,Cin,2], yf, sqrt sample weights, the regularisation filter, the
    preconditioner (filter part [1,C,H,Wh], projection part) and projection_reg, all as the kernel receives them (float32)."""

    def __init__(self, samples, yf, sw_sqrt, reg, dMh, dMP, lam, dev="cpu"):
        self.dev = dev
        self.H, self.Wh, self.N, self.Cin = samples.shape[:4]
        self.X32 = _cpu32(samples).to(dev)
        self.sws32 = _cpu32(sw_sqrt).to(dev).reshape(-1)
        self.yf32 = _cpu32(yf).to(dev).reshape(1, 1, self.H, self.Wh)
        self.reg32 = _cpu32(reg).to(dev).reshape(1, 1, *reg.shape[-2:])
        self.dMh32 = _cpu32(dMh).to(dev)
        self.C = self.dMh32.numel() // (self.H * self.Wh)
        self.dMh32 = self.dMh32.reshape(1, self.C, self.H, self.Wh)
        self.dMP, self.lam = f32(dMP), f32(lam)
        self.X, self.sws, self.yf, self.reg, self.dMh = (t.double() for t in (self.X32, self.sws32, self.yf32, self.reg32, self.dMh32))
        self.nz = nz_taps(reg)

    def run(self, hf, P, k, ngn=1, dt=torch.float64, perm=None):
        d = lambda t: _cpu32(t).to(self.dev).to(dt)
        X, sws, yf, reg, dMh = d(self.X32), d(self.sws32), d(self.yf32), d(self.reg32), d(self.dMh32)
        hf, P = d(hf).reshape(1, self.C, self.H, self.Wh, 2), d(P).reshape(self.Cin, self.C)
        if perm is not None:
            pc, pi, pn = (q.to(self.dev) for q in perm)
            X = X[:, :, pn][:, :, :, pi].contiguous()
            sws = sws[pn].contiguous()
            hf, dMh, P = hf[:, pc].contiguous(), dMh[:, pc].contiguous(), P[pi][:, pc].contiguous()
        h1, P1, _ = E.joint_gn_run(hf, P, X, yf, sws * sws, reg, k, ngn, projection_reg=self.lam, precond=(dMh, self.dMP))
        if perm is not None:
            ic, ii = torch.argsort(pc), torch.argsort(pi)
            h1, P1 = h1[:, ic], P1[ii][:, ic]
        return h1, P1

    def step(self, hf, P, k):
        h1, P1 = self.run(hf, P, k)
        return h1 - _cpu32(hf).to(self.dev).double().reshape(h1.shape), P1 - _cpu32(P).to(self.dev).double().reshape(P1.shape)

    def e32(self, hf, P, k, ref):
        g = torch.Generator().manual_seed(23)
        out = [0.0, 0.0]
        for _ in range(2):
            perm = (torch.randperm(self.C, generator=g), torch.randperm(self.Cin, generator=g), torch.randperm(self.N, generator=g))
            h1, P1 = self.run(hf, P, k, 1, torch.float32, perm)
            dh = h1.double() - _cpu32(hf).to(self.dev).double().reshape(h1.shape)
            dP = P1.double() - _cpu32(P).to(self.dev).double().reshape(P1.shape)
            out = [max(out[0], rel_err(dh, ref[0])), max(out[1], rel_err(dP, ref[1]))]
        return out

    def single_bound(self, hf, P, sms):
        """Relative float32 bounds (filter block, projection block) on the first CG step of one GN iteration from (hf, P)."""
        pl = eco_joint_plan(self.H, self.Wh, self.N, self.Cin, self.C, 1, 1, sms)
        X, sws, yf, reg = self.X, self.sws, self.yf, self.reg
        C, Cin, N, H, Wh = self.C, self.Cin, self.N, self.H, self.Wh
        NPIX = H * Wh
        rr = reg.shape[-2] * reg.shape[-1]
        h0 = _cpu32(hf).to(self.dev).double().reshape(1, C, H, Wh, 2)
        P0 = _cpu32(P).to(self.dev).double().reshape(Cin, C)
        w2 = (sws * sws).view(1, 1, -1)
        kw = kw_of(Wh, h0).view(1, 1, 1, -1)
        MX = mag(X)                                                                  # [H,Wh,N,Cin]
        c0 = E.joint_compress(X, P0)                                                 # [H,Wh,N,C,2]
        Mc0 = mag(c0)
        e_c0 = S2 * U * (Cin + 2) * torch.einsum("hwni,ic->hwnc", MX, P0.abs())
        mh0 = mag(h0)[0].permute(1, 2, 0)                                            # [H,Wh,C]
        ntiles = -(-Cin * C // pl["EPB"])
        dip = -(-pl["npx_max"] * C // BLOCK) + -(-ntiles // pl["grid"]) + 13 + -(-pl["grid"] // 32) + 5 + 3
        dgp = 2 * -(-NPIX // pl["SPL"]) + pl["SPL"] + 3

        def regabs(m, ext):                                                          # |J_reg^T J_reg(ext)| on magnitudes m [1,C,H,Wh]
            v = E.joint_reg_residual(cplx(m), reg.abs(), extension=ext)
            return E.joint_reg_adjoint(v, reg.abs(), C, H, Wh)[..., 0].clamp(min=0)

        def adjoints(u, e_u, mreg, e_reg_terms):
            """gh = sum_n conj(c0) u + reg, w = sum_n conj(X) u, gP = sum_pix Re(conj(h0) w): exact values and error bounds."""
            mu = mag(u)
            gh = E.cmul(E.conj(c0), u.unsqueeze(3)).sum(2)                           # [H,Wh,C,2]
            e_gh = torch.einsum("hwnc,hwn->hwc", e_c0, mu) + torch.einsum("hwnc,hwn->hwc", Mc0, e_u) + \
                S2 * U * (N + 2) * torch.einsum("hwnc,hwn->hwc", Mc0, mu)
            e_gh = e_gh.permute(2, 0, 1).unsqueeze(0) + S2 * U * (self.nz + rr + 2) * mreg + e_reg_terms
            w = E.cmul(E.conj(X), u.unsqueeze(3)).sum(2)                             # [H,Wh,Cin,2]
            e_w = torch.einsum("hwni,hwn->hwi", MX, e_u) + S2 * U * (N + 2) * torch.einsum("hwni,hwn->hwi", MX, mu)
            aw = torch.einsum("hwi,hwc->ic", mag(w), mh0)
            e_gP = torch.einsum("hwi,hwc->ic", e_w, mh0) + dgp * U * aw
            return gh, e_gh, e_gP, aw

        # linearisation: u = sw (c0 . h0 - yf), r = -(J^T f)
        h = h0[0].permute(1, 2, 0, 3).unsqueeze(2)                                   # [H,Wh,1,C,2]
        f = E.cmul(c0, h).sum(3)
        f[..., 0] -= yf[0, 0].unsqueeze(-1)
        e_f = torch.einsum("hwnc,hwc->hwn", e_c0, mh0) + S2 * U * (C + 2) * (torch.einsum("hwnc,hwc->hwn", Mc0, mh0) + yf[0, 0].abs().unsqueeze(-1))
        u0 = f * w2.unsqueeze(-1)
        e_u0 = w2 * e_f + 2 * U * mag(u0)
        fr = E.joint_reg_residual(h0, reg)
        greg = E.joint_reg_adjoint(fr, reg, C, H, Wh)
        gh, e_gh, e_gP, aw = adjoints(u0, e_u0, regabs(mag(h0), True), 0)
        rh = -(gh.permute(2, 0, 1, 3).unsqueeze(0) + greg)
        gPv = torch.einsum("hwis,hwcs->ic", E.cmul(E.conj(X), u0.unsqueeze(3)).sum(2), h0[0].permute(1, 2, 0, 3))
        rP = -(gPv + self.lam * P0)
        er = [e_gh + U * mag(rh), e_gP + U * (rP.abs() + self.lam * P0.abs())]
        r = [rh, rP]

        def Jv_terms(zh, zP):
            v = torch.einsum("ic,hwcs->hwis", zP, h0[0].permute(1, 2, 0, 3))        # [H,Wh,Cin,2]
            av = torch.einsum("ic,hwc->hwi", zP.abs(), mh0)
            Jv = E.cmul(c0, zh[0].permute(1, 2, 0, 3).unsqueeze(2)).sum(3) + E.cmul(X, v.unsqueeze(2)).sum(3)
            mzh = mag(zh)[0].permute(1, 2, 0)
            T = torch.einsum("hwnc,hwc->hwn", Mc0, mzh) + torch.einsum("hwni,hwi->hwn", MX, av)
            e_Jv = torch.einsum("hwnc,hwc->hwn", e_c0, mzh) + S2 * U * (C + 2) * torch.einsum("hwni,hwi->hwn", MX, av) + \
                S2 * U * (C + Cin + 3) * T
            return Jv, e_Jv

        def q_of(z):
            zh, zP = z
            Jv, _ = Jv_terms(zh, zP)
            u = Jv * w2.unsqueeze(-1)
            gh = E.cmul(E.conj(c0), u.unsqueeze(3)).sum(2).permute(2, 0, 1, 3).unsqueeze(0)
            gh = gh + E.joint_reg_adjoint(E.joint_reg_residual(zh, reg, extension=False), reg, C, H, Wh)
            w = E.cmul(E.conj(X), u.unsqueeze(3)).sum(2)
            gP = torch.einsum("hwis,hwcs->ic", w, h0[0].permute(1, 2, 0, 3)) + self.lam * zP
            return [gh, gP]

        def eq_of(z):
            zh, zP = z
            Jv, e_Jv = Jv_terms(zh, zP)
            u = Jv * w2.unsqueeze(-1)
            e_u = w2 * e_Jv + 2 * U * mag(u)
            gh, e_gh, e_gP, aw = adjoints(u, e_u, regabs(mag(zh), False), 0)
            return [e_gh + U * mag(gh.permute(2, 0, 1, 3).unsqueeze(0)), e_gP + dgp * U * self.lam * zP.abs()]

        # the first CG step d = alpha z, z = M^-1 r, alpha = <r, z> / <z, A z>
        z = [r[0] / self.dMh.unsqueeze(-1), r[1] / self.dMP]
        mz = [mag(z[0]), z[1].abs()]
        ez = [er[0] / self.dMh + U * mz[0], er[1] / self.dMP + U * mz[1]]
        wts = [kw, torch.ones_like(z[1])]

        def ipm(a, b):
            return sum(float((w_ * a_ * b_).sum()) for w_, a_, b_ in zip(wts, a, b))

        q, eq = q_of(z), eq_of(z)
        mq = [mag(q[0]), q[1].abs()]
        rho = float((kw.unsqueeze(-1) * r[0] * z[0]).sum()) + float((r[1] * z[1]).sum())
        sig = float((kw.unsqueeze(-1) * z[0] * q[0]).sum()) + float((z[1] * q[1]).sum())
        mr = [mag(r[0]), r[1].abs()]
        erho = 2 * ipm(mz, er) + ipm(mr, [U * mz[0], U * mz[1]]) + dip * U * ipm(mr, mz)
        # <z, A dz>_w = <A (w z), dz>: A = J^T J is self-adjoint in the plain real inner product
        Awz = q_of([z[0] * kw.unsqueeze(-1), z[1]])
        esig = ipm(mq, ez) + float((mag(Awz[0]) * ez[0]).sum()) + float((Awz[1].abs() * ez[1]).sum()) + ipm(mz, eq) + dip * U * ipm(mz, mq)
        alpha = rho / sig
        ea = abs(alpha) * (erho / abs(rho) + esig / abs(sig) + 2 * U)
        return [float((abs(alpha) * ez[b] + ea * mz[b] + U * abs(alpha) * mz[b]).max() / (abs(alpha) * mz[b]).max()) for b in (0, 1)]
