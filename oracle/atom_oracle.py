"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch-CPU) of the ATOM rows of the hot path.  Every function computes in the dtype
of its inputs: float32 inputs give the float32 restatement the goldens pin, float64 inputs a float64 computation throughout (the
sums that are accumulated in float64 are rounded back to the input dtype, never to float32).

Same rules as oracle/dimp_oracle.py: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import it.
Parity status: PINNED -- `oracle/gen_golden.py` (gen_atom_cg, gen_fourier) runs the unmodified reference classes
(`ConvProblem` + `ConjugateGradient`, `pytracking/libs/fourier.py`) and commits their outputs; tests/test_oracle_golden.py
checks the functions below against them.

The reference obtains J p and J^T u by double backward through `operation.conv2d` (optimization.py:251,279-280);
here they are written out explicitly (SURVEY.md 9.5).
"""
import math

import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# S2.2 operation.conv2d(mode='same') / conv1x1
# ----------------------------------------------------------------------------------------------
def conv_same(x, w):
    """pytracking/libs/operation.py:5-32 with mode='same': pad k//2, drop the last row/col for even kernels."""
    kh, kw = w.shape[-2:]
    out = F.conv2d(x, w, padding=(kh // 2, kw // 2))
    if kh % 2 == 0:
        out = out[:, :, :-1, :]
    if kw % 2 == 0:
        out = out[:, :, :, :-1]
    return out


def conv_same_adjoint_filter(x, u, k):
    """Adjoint of w -> conv_same(x, w) for a single-output-channel filter: g[c,a,b] = sum_{i,y,x'} u[i,y,x'] xpad[i,c,y+a,x'+b]."""
    p = k // 2
    xp = F.pad(x, (p, p, p, p))
    win = xp.unfold(2, k, 1).unfold(3, k, 1)                 # [n,c,H+1,W+1,k,k] for even k
    win = win[:, :, :u.shape[-2], :u.shape[-1]]
    return torch.einsum("ncyxab,nyx->cab", win.double(), u[:, 0].double()).to(x.dtype).unsqueeze(0)


def conv1x1(x, P):
    """operation.py:35-42."""
    return torch.conv2d(x, P)


def activation(x, kind="none", param=0.05):
    """ATOM response / projection activations (pytracking/tracker/atom/atom.py:440-468)."""
    if kind == "none":
        return x
    if kind == "relu":
        return F.relu(x)
    if kind == "elu":
        return F.elu(x)
    if kind == "mlu":
        return F.elu(F.leaky_relu(x, 1.0 / param), param)
    raise ValueError(kind)


def activation_deriv(x, kind="none", param=0.05):
    if kind == "none":
        return torch.ones_like(x)
    if kind == "relu":
        return (x > 0).to(x.dtype)
    if kind == "elu":
        return torch.where(x > 0, torch.ones_like(x), torch.exp(x))
    if kind == "mlu":
        return torch.where(x >= 0, torch.ones_like(x), torch.exp(x / param))
    raise ValueError(kind)


# ----------------------------------------------------------------------------------------------
# S3.5 ConjugateGradient.run on ConvProblem (the per-frame ATOM filter update)
# ----------------------------------------------------------------------------------------------
def atom_cg_filter(w, feat, y, sw, filter_reg, num_iter, act="mlu", act_param=0.05, fletcher_reeves=False, dact=None):
    """ConjugateGradient.run(num_iter) (pytracking/libs/optimization.py:227-275, run_CG :72-163) on
    ConvProblem (pytracking/tracker/atom/optim.py:71-99), direction_forget_factor = 0 (state reset every run).
    w [1,C,k,k], feat [n,C,H,W], y [n,1,H,W], sw [n]; dact [n,1,H,W] replaces phi'(s) when given (the tests take the
    derivative of a cell at a kink from its other side with it). Returns (w_new, delta, rho_trace)."""
    k = w.shape[-1]
    s = conv_same(feat, w)
    a, d = activation(s, act, act_param), activation_deriv(s, act, act_param)
    if dact is not None:
        d = dact
    swv = sw.view(-1, 1, 1, 1)
    # b = -J^T f0,  f0 = [sqrt(sw) (phi(s) - y), sqrt(reg) w],  J^T u = A^T(sqrt(sw) phi' u_data) + sqrt(reg) u_reg
    b = -(conv_same_adjoint_filter(feat, swv * d * (a - y), k) + filter_reg * w)
    D = swv * d * d

    def A(p):
        return conv_same_adjoint_filter(feat, D * conv_same(feat, p), k) + filter_reg * p

    def ip(u, v):
        return (u.double() * v.double()).sum().to(u.dtype)

    r = b.clone()
    x = None
    p = None
    rho = torch.ones(())
    r_prev = None
    trace = []
    for ii in range(num_iter):
        z = r
        rho1 = rho
        rho = ip(r, z)
        trace.append(float(rho))
        if float(rho) == 0.0:
            break
        if p is None:
            p = z.clone()
        else:
            if fletcher_reeves:
                beta = rho / rho1
            else:
                beta = (rho - ip(r_prev, z)) / rho1
            beta = beta.clamp(0)
            p = z + p * beta
        q = A(p)
        alpha = rho / ip(p, q)
        if not fletcher_reeves:
            r_prev = r.clone()
        x = p * alpha if x is None else x + p * alpha
        if ii < num_iter - 1:
            r = r - q * alpha
    if x is None:
        x = torch.zeros_like(w)
    return w + x, x, trace


# ----------------------------------------------------------------------------------------------
# S2.3 Fourier-series upsampling of the score map (ATOM.localize_target)
# ----------------------------------------------------------------------------------------------
def fourier_interp(scores, kernel_size, output_sz):
    """pytracking/tracker/atom/atom.py:304-316 for one feature type: cfft2 (fourier.py:20-24: rfft2 + rfftshift2, the
    Nyquist row of an even-sized map appears at both ends) / (H*W) -> shift_fs by pi*(1 - (ksz%2)/sz) (:78-92) -> sample_fs
    to output_sz (:35-61: zero padding of the centred half spectrum, irfft2, * prod(output_sz)). scores [S,1,H,W]."""
    S, _, H, W = scores.shape
    oh, ow = int(output_sz[0]), int(output_sz[1])
    f = torch.fft.rfftn(scores.double(), dim=(-2, -1))                       # [S,1,H,W/2+1]
    hh = H + 2
    f = torch.cat((f[:, :, (hh - 1) // 2:, :], f[:, :, :hh // 2, :]), 2)      # rfftshift2: rows -(H//2)..(H//2) (odd count)
    f = f / (H * W)
    nr, nc = f.shape[2], f.shape[3]
    ky = torch.arange(-int((nr - 1) / 2), int(nr / 2 + 1), dtype=torch.float64).view(1, 1, -1, 1)
    kx = torch.arange(0, int((2 * nc - 1) / 2 + 1), dtype=torch.float64).view(1, 1, 1, -1)
    sh_y = math.pi * (1 - (kernel_size[0] % 2) / H)
    sh_x = math.pi * (1 - (kernel_size[1] % 2) / W)
    f = f * torch.exp(1j * sh_y * ky) * torch.exp(1j * sh_x * kx)
    szr, szc = nr, 2 * nc - 1
    tot0, tot1 = oh - szr, ow - szc
    pad_top = int((tot0 + 1) / 2) if szr % 2 == 0 else int(tot0 / 2)
    pad_bottom = tot0 - pad_top
    pad_right = int((tot1 + 1) / 2)
    f = F.pad(torch.view_as_real(f), (0, 0, 0, pad_right, pad_top, pad_bottom))
    f = torch.view_as_complex(f.contiguous())
    mid = int((f.shape[2] - 1) / 2)
    f = torch.cat((f[:, :, mid:, :], f[:, :, :mid, :]), 2)                    # irfftshift2
    out = torch.fft.irfftn(f, s=(oh, ow), dim=(-2, -1)) * (oh * ow)
    return out.to(scores.dtype)


def feature_normalize(x, p=2.0):
    """pytracking/features/featurebase.py:105-108."""
    n = x.shape[0]
    d = (torch.sum(x.abs().reshape(n, 1, 1, -1) ** p, dim=3, keepdim=True) / (x.shape[1] * x.shape[2] * x.shape[3]) + 1e-10) ** (1 / p)
    return x / d


# ----------------------------------------------------------------------------------------------
# S3.5 (init) GaussNewtonCG.run on FactorizedConvProblem: joint filter + projection matrix optimisation
# ----------------------------------------------------------------------------------------------
def conv_same_adjoint_input(u, w, H, W):
    """Adjoint of x -> conv_same(x, w) (single-output-channel filter w [1,C,k,k]) w.r.t. x: [n,1,H,W] -> [n,C,H,W]."""
    k = w.shape[-1]
    p = k // 2
    up = F.pad(u, (0, 1, 0, 1)) if k % 2 == 0 else u                    # undo the crop: zeros on the dropped row / column
    return F.conv_transpose2d(up, w, padding=p)[:, :, :H, :W]


def atom_gn_joint(w, P, X, y, sw, filter_reg, proj_reg, num_cg_iter, num_gn_iter, act="mlu", act_param=0.05, fletcher_reeves=True):
    """GaussNewtonCG.run(num_cg_iter, num_gn_iter) (pytracking/libs/optimization.py:328-421) on FactorizedConvProblem
    (pytracking/tracker/atom/optim.py:6-68), projection_activation = identity. Returns (w, P)."""
    k = w.shape[-1]
    H, Wd = X.shape[-2:]
    swv = sw.view(-1, 1, 1, 1)
    w, P = w.clone(), P.clone()

    def ip(a, b):
        return (a[0].double() * b[0].double()).sum().to(a[0].dtype) + (a[1].double() * b[1].double()).sum().to(a[1].dtype)

    for _ in range(num_gn_iter):
        comp = conv1x1(X, P)
        s = conv_same(comp, w)
        a, d = activation(s, act, act_param), activation_deriv(s, act, act_param)
        r0 = swv * d * (a - y)
        D = swv * d * d

        def JT(u):      # u already carries sw * phi' factors
            gw = conv_same_adjoint_filter(comp, u, k)
            T = conv_same_adjoint_input(u, w, H, Wd)                  # [n,Cc,H,W]
            gP = torch.einsum("ncp,nkp->ck", T.flatten(2).double(), X.flatten(2).double()).to(X.dtype).reshape(P.shape)
            return gw, gP

        gw, gP = JT(r0)
        r = [-(gw + filter_reg * w), -(gP + proj_reg * P)]
        x = None
        p = None
        rho = torch.ones(())
        r_prev = None
        for ii in range(num_cg_iter):
            z = [r[0] / filter_reg, r[1] / proj_reg]
            rho1 = rho
            rho = ip(r, z)
            if float(rho) == 0.0:
                break
            if p is None:
                p = [z[0].clone(), z[1].clone()]
            else:
                beta = rho / rho1 if fletcher_reeves else (rho - ip(r_prev, z)) / rho1
                beta = beta.clamp(0)
                p = [z[0] + p[0] * beta, z[1] + p[1] * beta]
            Jp = D * (conv_same(comp, p[0]) + conv_same(conv1x1(X, p[1]), w))
            qw, qP = JT(Jp)
            q = [qw + filter_reg * p[0], qP + proj_reg * p[1]]
            alpha = rho / ip(p, q)
            if not fletcher_reeves:
                r_prev = [r[0].clone(), r[1].clone()]
            x = [p[0] * alpha, p[1] * alpha] if x is None else [x[0] + p[0] * alpha, x[1] + p[1] * alpha]
            if ii < num_cg_iter - 1:
                r = [r[0] - q[0] * alpha, r[1] - q[1] * alpha]
        if x is not None:
            w, P = w + x[0], P + x[1]
    return w, P
