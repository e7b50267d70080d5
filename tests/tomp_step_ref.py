"""Float64 reference of every launch of the ToMP head, error bounds for its float32 kernels, and torch's own float32 error.

One function per launch kind of csrc/transformer.cu, csrc/tower.cu and csrc/tomp_tokens.cu, and for the 1x1 correlation
(`ops.conv1x1`, the ToMP classifier's `apply_filter`).  Each takes the float32 operands the kernel consumed and returns a `Step`:
  ref    the operation in float64 on those operands
  mag    a magnitude term per entry (the same sum over absolute values; for attention sum_l p_l |v_l| / sum_l p_l)
  bound  a bound on |kernel - ref| per entry for a float32 kernel with the summation order of the CUDA source, with the CUDA Programming
         Guide's error figures for the approximate intrinsics: __expf(x) 2 + floor(|1.173 x|) ulp (both attention kernels), rsqrtf
         2 ulp (LayerNorm, GroupNorm), expf 2 ulp (the exp export)
  r32    torch float32 on the same operands, TF32 off: the yardstick e_32 = |r32 - ref|
  tf32   (GEMMs and convolutions only) a plain TF32 GEMM on the same operands (cvt.rna emulated bitwise), for e_TF32
The kernels may fuse a multiply and an add into an FMA (nvcc contracts device code by default): every bound covers both forms.
Bounds are first order in u = 2^-24; a factor 1 + 2^-10 covers the second-order terms of the operand sizes used here.

GEMMs and convolutions are held to the criterion of tests/test_tc_conv_layers_gpu.py instead of `bound`:
e = max |y - ref| / mag <= e_TF32 / 16, and e <= (K + 2) 2^-23 + 2^-20 (`gemm_bound_rel`)."""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
ULP = 2.0 ** -23              # one ulp of a float32 value, relative, at most
F64, F32 = torch.float64, torch.float32
SECOND = 1 + 2.0 ** -10       # second-order slack on first-order bounds
EXPF_A, EXPF_C = 2.0, 1.173   # __expf: 2 + floor(|1.173 x|) ulp
RSQRT_ULP = 2.0               # rsqrtf: 2 ulp
TINY = 2.0 ** -126            # ex2.approx flushes results below the smallest normal to zero


class Step:
    def __init__(self, ref, mag, bound, r32, tf32=None):
        self.ref, self.mag, self.bound, self.r32, self.tf32 = ref, mag, bound, r32, tf32


def _g(n):
    return n * U / (1 - n * U)


def tf32(x):
    """float32 -> nearest TF32 value (10 explicit mantissa bits), ties away from zero, as cvt.rna.tf32.f32."""
    b = x.to(F32).contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(F32)


def _no_tf32():
    class _Ctx:
        def __enter__(self):
            self.a, self.b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False

        def __exit__(self, *exc):
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = self.a, self.b
    return _Ctx()


# ---- elementwise ------------------------------------------------------------------------------------------------------------------
def add_pos(x, pos):
    """add_pos_kernel: x [L,B,D] + pos [L,Bp,D] (Bp = 1 broadcasts); one float32 add, so the kernel equals torch bit for bit."""
    ref = x.to(F64) + pos.to(F64)
    r32 = x + pos
    return Step(ref, x.to(F64).abs() + pos.to(F64).abs(), U * r32.to(F64).abs(), r32)


# ---- tensor-core GEMMs ------------------------------------------------------------------------------------------------------------
def gemm_bound_rel(K):
    return (K + 2) * 2.0 ** -23 + 2.0 ** -20


def gemm(x, w, b, res=None, relu=False):
    """The encoder's token GEMM (a 1x1 convolution on the wgmma kernel): y = relu?(x w^T + b + res), x [M,K], w [N,K]."""
    xd, wd, bd = x.to(F64), w.to(F64), b.to(F64)
    ref, mag, t = xd @ wd.t() + bd, xd.abs() @ wd.abs().t() + bd.abs(), tf32(x).to(F64) @ tf32(w).to(F64).t() + bd
    with _no_tf32():
        r32 = x @ w.t() + b
    if res is not None:
        rd = res.to(F64)
        ref, mag, t, r32 = ref + rd, mag + rd.abs(), t + rd, r32 + res
    if relu:
        ref, t, r32 = ref.clamp(min=0), t.clamp(min=0), r32.clamp(min=0)
    return Step(ref, mag, gemm_bound_rel(x.shape[1]) * mag, r32, t)


def conv3x3(x, w, b):
    """A tower convolution, NHWC x [S,H,W,Cin], w [Cout,Cin,3,3] (the module's layout), pad 1: the same criterion as `gemm`."""
    xc = x.permute(0, 3, 1, 2)

    def conv(a, f, bias):
        return F.conv2d(a, f, bias, padding=1).permute(0, 2, 3, 1)
    bd = b.to(F64)
    ref = conv(xc.to(F64), w.to(F64), bd)
    mag = conv(xc.to(F64).abs(), w.to(F64).abs(), bd.abs())
    t = conv(tf32(xc.contiguous()).to(F64), tf32(w.contiguous()).to(F64), bd)
    with _no_tf32():
        r32 = conv(xc, w, b)
    return Step(ref, mag, gemm_bound_rel(9 * x.shape[-1]) * mag, r32, t)


# ---- attention ----------------------------------------------------------------------------------------------------------------------
def _heads(t, H):
    L, B, D = t.shape
    return t.reshape(L, B, H, D // H).permute(1, 2, 0, 3)            # [B,H,L,hd]


def _attention(q, k, v, mask, H, scale, rows, exp_ulps, n_acc, n_sum):
    """Shared by both kernels. q [Lq,B,D] (unscaled, as the kernels get it), k, v [L,B,D], mask [B,L] bool (True = padded key), the
    query rows `rows` only.  exp_ulps(x_gap) -> ulps of the exponentials that end up in one weight for a key x_gap below the max; n_acc
    / n_sum: rounding steps on the accumulation of sum p v and of sum p."""
    Lq, B, D = q.shape
    L = k.shape[0]
    hd = D // H
    sc = scale if q.dtype == F64 else float(torch.tensor(scale, dtype=F32))          # the float32 constant the kernels get
    qs32 = (q[rows] * sc)                                             # the kernels scale q in float32 first
    qh, kh, vh = _heads(q[rows].to(F64) * sc, H), _heads(k.to(F64), H), _heads(v.to(F64), H)
    s = qh @ kh.transpose(-1, -2)                                     # [B,H,R,L]
    # score error: the scaled q (u) and a chain of hd FMAs
    ds = _g(hd + 2) * (_heads(qs32.to(F64), H).abs() @ kh.abs().transpose(-1, -2)) + U * s.abs()
    dead = mask.view(B, 1, 1, L) if mask is not None else torch.zeros(B, 1, 1, L, dtype=torch.bool, device=q.device)
    s = s.masked_fill(dead, float("-inf"))
    ds = ds.masked_fill(dead, 0.0)
    M = s.amax(-1, keepdim=True)
    p = torch.exp(s - M)
    Z = p.sum(-1, keepdim=True)
    out = (p @ vh) / Z
    A = (p @ vh.abs()) / Z
    dsmax = ds.amax(-1, keepdim=True)
    gap = (M - s).masked_fill(dead, 0.0) + 2 * dsmax
    rho = ds + dsmax + exp_ulps(gap) * ULP                            # relative error of one weight p_l
    rho = rho.masked_fill(dead, 0.0)
    dN = (p * (rho + _g(n_acc))) @ vh.abs()
    dZ = (p * (rho + _g(n_sum))).sum(-1, keepdim=True)
    bound = SECOND * (dN + out.abs() * dZ) / Z + 2 * U * out.abs() + L * TINY * vh.abs().amax(-2, keepdim=True) / Z

    R = qh.shape[2]

    def back(t):
        return t.permute(2, 0, 1, 3).reshape(R, B, D)
    with _no_tf32():
        q32, k32, v32 = _heads(qs32, H), _heads(k, H), _heads(v, H)
        s32 = (q32 @ k32.transpose(-1, -2)).masked_fill(dead, float("-inf"))
        r32 = torch.softmax(s32, -1) @ v32
    return Step(back(out), back(A.expand_as(out)), back(bound), back(r32))


def attention(qk, v, mask, H, scale, rows=slice(None)):
    """attention_kernel on the encoder's fused projection: qk [L,B,2D] ([q | k], row pitch 2D), v [L,B,D].  Each query's keys are
    split over 8 lanes; a lane walks g = 2 ceil(L / 64) groups of 4 keys, rescales its running sums up to g times, and the 8 states
    merge in 3 levels.  The exponentials that end up in one weight telescope: their arguments sum to the gap to the final max."""
    D = v.shape[-1]
    L = v.shape[0]
    g = 2 * math.ceil(L / 64)
    return _attention(qk[..., :D], qk[..., D:], v, mask, H, scale, rows,
                      lambda gap: EXPF_A * (1 + g + 3) + EXPF_C * gap, n_acc=5 * g + 6, n_sum=5 * g + 6)


def attention_q1(q, k, v, mask, H, scale):
    """attention_q1_kernel: q [B,D] (one query per batch element), k, v [L,B,D].  One exponential per key against the exact max of
    the scores; 256 threads sum ceil(L / 256) weights each, then a block tree (10 levels); 8 warps accumulate ceil(L / 8) keys each and
    their partials add in order."""
    L = k.shape[0]
    st = _attention(q[None], k, v, mask, H, scale, slice(None), lambda gap: EXPF_A + EXPF_C * gap,
                    n_acc=math.ceil(L / 8) + 8, n_sum=math.ceil(L / 256) + 10)
    return Step(st.ref[0], st.mag[0], st.bound[0], st.r32[0])


# ---- normalisations -----------------------------------------------------------------------------------------------------------------
def _norm(x, gamma_c, beta_c, n_chain, eps, count):
    """Shared LayerNorm / GroupNorm(1) bound.  x [..., n] (the normalised set last), gamma_c / beta_c broadcastable to x.
    mean = (chain of n_chain adds) / n; c = x - mean; var = (chain of n_chain FMAs of c c) / n; rstd = rsqrtf(var + eps);
    y = c rstd gamma + beta."""
    xd = x.to(F64)
    n = count
    mu = xd.mean(-1, keepdim=True)
    c = xd - mu
    var = (c * c).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    g, b = gamma_c.to(F64), beta_c.to(F64)
    y = c * rstd * g + b
    dmu = _g(n_chain + 1) * xd.abs().mean(-1, keepdim=True)
    V = var * n
    dV = (_g(n_chain + 1) + 3 * U) * (V + n * dmu ** 2) + n * dmu ** 2
    rv = (dV / n + U * var + U * (var + eps)) / (var + eps)
    rr = rv / 2 + RSQRT_ULP * ULP
    gc = (g * c * rstd).abs()
    bound = SECOND * ((g.abs() * rstd * dmu) + gc * (rr + 3 * U) + U * (y.abs() + b.abs()))
    return y, gc + b.abs(), bound


def layernorm(x, w, b):
    """layernorm_kernel: one warp per token, x [T,D]; each lane sums D / 32 entries, then a 5-level shuffle tree."""
    D = x.shape[-1]
    ref, mag, bound = _norm(x, w, b, D // 32 + 5, 1e-5, D)
    with _no_tf32():
        r32 = F.layer_norm(x, (D,), w, b, 1e-5)
    return Step(ref, mag, bound, r32)


def groupnorm_relu(x, w, b):
    """groupnorm1_relu_kernel in place on NHWC x [S,H,W,C]: one CTA of 1024 threads per sample, each summing ceil(n / 1024) entries,
    then the block tree (10 levels); ReLU after the affine step (1-Lipschitz, so the bound carries over)."""
    S, H, W, C = x.shape
    n = H * W * C
    y, mag, bound = _norm(x.reshape(S, n), w.repeat(H * W), b.repeat(H * W), math.ceil(n / 1024) + 10, 1e-5, n)
    with _no_tf32():
        r32 = torch.relu(F.group_norm(x.permute(0, 3, 1, 2), 1, w, b, 1e-5)).permute(0, 2, 3, 1)
    return Step(y.clamp(min=0).reshape(x.shape), mag.reshape(x.shape), bound.reshape(x.shape), r32)


# ---- the decoder's small linear layers ---------------------------------------------------------------------------------------------
def small_linear(x, w, b, res=None, relu=False):
    """small_linear_kernel: one warp per output; each lane sums K / 128 four-term products, then a 5-level shuffle tree, the bias,
    ReLU, the residual."""
    K = x.shape[-1]
    xd, wd, bd = x.to(F64), w.to(F64), b.to(F64)
    ref, mag = xd @ wd.t() + bd, xd.abs() @ wd.abs().t() + bd.abs()
    with _no_tf32():
        r32 = x @ w.t() + b
    if relu:
        ref, r32 = ref.clamp(min=0), r32.clamp(min=0)
    if res is not None:
        ref, mag, r32 = ref + res.to(F64), mag + res.to(F64).abs(), r32 + res
    return Step(ref, mag, SECOND * _g(K // 32 + 9) * mag, r32)


# ---- the tower's import and export -------------------------------------------------------------------------------------------------
def import_scaled(feat, att):
    """import_scaled_kernel: feat [S,C,H,W] * att [S,H,W] -> NHWC; one float32 product, so the kernel equals torch bit for bit."""
    r32 = (feat * att[:, None]).permute(0, 2, 3, 1)
    ref = (feat.to(F64) * att.to(F64)[:, None]).permute(0, 2, 3, 1)
    return Step(ref, ref.abs(), U * ref.abs(), r32)


def export_exp(x):
    """export_exp_kernel: NHWC x [S,H,W,4] -> NCHW exp(x) with expf (2 ulp)."""
    ref = torch.exp(x.to(F64)).permute(0, 3, 1, 2)
    r32 = torch.exp(x).permute(0, 3, 1, 2)
    return Step(ref, ref, 2 * ULP * ref, r32)


# ---- token assembly ----------------------------------------------------------------------------------------------------------------
def tokens(train_feat, test_feat, label, ltrb, fg, test_token, w1, b1, w2t, b2, w3t, b3, B):
    """tomp_tokens_kernel -> [(n + m) H W, B, D].  Train cells: h1 = relu(b1 + 4 FMAs), h2 = relu(b2 + D1 FMAs over h1), e = b3 + D
    FMAs over h2, v = (feat + fg label) + e; each layer's bound carries the previous one's through |W|.  Test cells: feat (+ token), one
    add."""
    n, D, H, W = train_feat.shape
    m = test_feat.shape[0]
    HW = H * W
    d = lambda t: t.to(F64)
    lt = d(ltrb).reshape(n, 4, HW)
    z1 = torch.einsum("jk,fkp->fjp", d(w1), lt) + d(b1)[None, :, None]
    h1 = z1.clamp(min=0)
    dh1 = _g(5) * (torch.einsum("jk,fkp->fjp", d(w1).abs(), lt.abs()) + d(b1).abs()[None, :, None])
    W2, W3 = d(w2t).t(), d(w3t).t()                                  # [D, D1], [D, D]
    z2 = torch.einsum("cj,fjp->fcp", W2, h1) + d(b2)[None, :, None]
    h2 = z2.clamp(min=0)
    M2 = torch.einsum("cj,fjp->fcp", W2.abs(), h1 + dh1) + d(b2).abs()[None, :, None]
    dh2 = _g(W2.shape[1] + 1) * M2 + torch.einsum("cj,fjp->fcp", W2.abs(), dh1)
    e = torch.einsum("ck,fkp->fcp", W3, h2) + d(b3)[None, :, None]
    M3 = torch.einsum("ck,fkp->fcp", W3.abs(), h2 + dh2) + d(b3).abs()[None, :, None]
    de = _g(D + 1) * M3 + torch.einsum("ck,fkp->fcp", W3.abs(), dh2)
    tf = d(train_feat).reshape(n, D, HW)
    fl = d(fg)[None, :, None] * d(label).reshape(n, 1, HW)
    v = (tf + fl) + e
    mag_tr = tf.abs() + fl.abs() + M3
    b_tr = SECOND * (de + 2 * U * (tf.abs() + fl.abs()) + U * v.abs())
    te = d(test_feat).reshape(m, D, HW) + (d(test_token)[None, :, None] if test_token is not None else 0.0)
    mag_te = d(test_feat).reshape(m, D, HW).abs() + (d(test_token).abs()[None, :, None] if test_token is not None else 0.0)
    with _no_tf32():
        x32 = ltrb.reshape(n, 4, HW)
        a1 = torch.relu(torch.einsum("jk,fkp->fjp", w1, x32) + b1[None, :, None])
        a2 = torch.relu(torch.einsum("jc,fjp->fcp", w2t, a1) + b2[None, :, None])
        e32 = torch.einsum("kc,fkp->fcp", w3t, a2) + b3[None, :, None]
        v32 = (train_feat.reshape(n, D, HW) + fg[None, :, None] * label.reshape(n, 1, HW)) + e32
        t32 = test_feat.reshape(m, D, HW) + (test_token[None, :, None] if test_token is not None else 0.0)

    def tok(a, b_):
        return torch.cat([a.permute(0, 2, 1).reshape(-1, D), b_.permute(0, 2, 1).reshape(-1, D)], 0)[:, None].expand(-1, B, -1)
    return Step(tok(v, te), tok(mag_tr, mag_te), tok(b_tr, U * te.abs()), tok(v32, t32))


# ---- the 1x1 correlation -----------------------------------------------------------------------------------------------------------
def conv1x1(x, P):
    """conv1x1_kernel: x [S,Cin,H,W], P [Cout,Cin] -> [S,Cout,H,W]; one FMA chain of Cin terms from 0 per output."""
    xd, Pd = x.to(F64), P.reshape(P.shape[0], -1).to(F64)
    ref = torch.einsum("oc,schw->sohw", Pd, xd)
    mag = torch.einsum("oc,schw->sohw", Pd.abs(), xd.abs())
    with _no_tf32():
        r32 = torch.einsum("oc,schw->sohw", P.reshape(P.shape[0], -1), x)
    return Step(ref, mag, SECOND * _g(x.shape[1] + 1) * mag, r32)


# ---- checks ------------------------------------------------------------------------------------------------------------------------
YARD, FLOOR = 20, 64 * U


def check(ker, st, what):
    """Every entry within max(4 e_32, bound); returns (worst e / bar, worst e / e_32 yardstick ratio, worst e) for the report."""
    ker, ref, r32 = ker.to(F64), st.ref, st.r32.to(F64)
    d, d32 = (ker - ref).abs(), (r32 - ref).abs()
    assert bool(torch.isfinite(ker).all()), "%s: NaN / Inf" % what
    bar = torch.maximum(4 * d32, st.bound)
    over = d > bar
    if bool(over.any()):
        i = int(torch.nonzero(over.reshape(-1))[0])
        raise AssertionError("%s: %d entries outside max(4 e_32, bound); first flat %d: kernel %.9g ref %.9g |d| %.3g bound %.3g e_32 %.3g" % (
            what, int(over.sum()), i, float(ker.reshape(-1)[i]), float(ref.reshape(-1)[i]), float(d.reshape(-1)[i]),
            float(st.bound.reshape(-1)[i]), float(d32.reshape(-1)[i])))
    live = st.mag > 0
    e = (d / torch.where(live, st.mag, torch.ones_like(st.mag)))[live]
    e32 = (d32 / torch.where(live, st.mag, torch.ones_like(st.mag)))[live]
    ratio_bar = float((d / torch.where(bar > 0, bar, torch.ones_like(bar))).max())
    yard = float(e.max() / (YARD * e32.max() + FLOOR)) if e.numel() else 0.0
    return ratio_bar, yard, float(e.max()) if e.numel() else 0.0


def check_gemm(ker, st, K, what):
    """The GEMM criterion: e <= e_TF32 / 16 and e <= (K + 2) 2^-23 + 2^-20, e = max |y - ref| / mag; returns (e, e_tf32)."""
    m = st.mag + 1e-30
    y = ker.to(F64)
    assert bool(torch.isfinite(y).all()), "%s: NaN / Inf" % what
    e = float(((y - st.ref).abs() / m).max())
    e_tf32 = float(((st.tf32 - st.ref).abs() / m).max())
    assert e <= e_tf32 / 16, "%s: e %.3e is not 16x below plain TF32 (%.3e)" % (what, e, e_tf32)
    assert e <= gemm_bound_rel(K), "%s: e %.3e above the fp32 summation bound %.3e" % (what, e, gemm_bound_rel(K))
    return e, e_tf32


# ---- the transformer's launch sequence ---------------------------------------------------------------------------------------------
# buffer ids of b200trk_transformer_debug_buffer
SRC, QKIN, QK, V, ATT, TMP, FF, MEM_POS, K, TGT, T1, T2, Q, DATT, DFF, QPOS = range(16)
BUFFER_NAMES = ("src", "qkin", "qk", "v", "att", "tmp", "ff", "mem_pos", "k", "tgt", "t1", "t2", "q", "dec_att", "dec_ff", "qpos")
HS = -1


def launch_plan(n_enc, n_dec):
    """The fixed launch sequence of b200trk_transformer_forward: one dict per launch with its kind, the state-dict prefix of its
    parameters, the buffers it reads and the one it writes."""
    P = []
    for i in range(n_enc):
        p = "encoder.layers.%d." % i
        P += [dict(kind="add_pos", ins=(SRC,), out=QKIN),
              dict(kind="gemm", p=p + "self_attn.in_proj", rows=(0, 2), ins=(QKIN,), out=QK),
              dict(kind="gemm", p=p + "self_attn.in_proj", rows=(2, 3), ins=(SRC,), out=V),
              dict(kind="attention", ins=(QK, V), out=ATT),
              dict(kind="gemm", p=p + "self_attn.out_proj", ins=(ATT,), res=SRC, out=TMP),
              dict(kind="layernorm", p=p + "norm1", ins=(TMP,), out=SRC),
              dict(kind="gemm", p=p + "linear1", ins=(SRC,), relu=True, out=FF),
              dict(kind="gemm", p=p + "linear2", ins=(FF,), res=SRC, out=TMP),
              dict(kind="layernorm", p=p + "norm2", ins=(TMP,), out=SRC)]
    P.append(dict(kind="add_pos", ins=(SRC,), out=MEM_POS))
    for i in range(n_dec):
        p = "decoder.layers.%d." % i
        P += [dict(kind="small_linear", p=p + "self_attn.in_proj", rows=(2, 3), ins=(TGT,), out=T1),
              dict(kind="small_linear", p=p + "self_attn.out_proj", ins=(T1,), res=TGT, out=T2),
              dict(kind="layernorm", p=p + "norm1", ins=(T2,), out=TGT),
              dict(kind="add_query_pos", ins=(TGT, QPOS), out=T1),
              dict(kind="small_linear", p=p + "multihead_attn.in_proj", rows=(0, 1), ins=(T1,), out=Q),
              dict(kind="gemm", p=p + "multihead_attn.in_proj", rows=(1, 2), ins=(MEM_POS,), out=K),
              dict(kind="gemm", p=p + "multihead_attn.in_proj", rows=(2, 3), ins=(SRC,), out=V),
              dict(kind="attention_q1", ins=(Q, K, V), out=DATT),
              dict(kind="small_linear", p=p + "multihead_attn.out_proj", ins=(DATT,), res=TGT, out=T2),
              dict(kind="layernorm", p=p + "norm2", ins=(T2,), out=TGT),
              dict(kind="small_linear", p=p + "linear1", ins=(TGT,), relu=True, out=DFF),
              dict(kind="small_linear", p=p + "linear2", ins=(DFF,), res=TGT, out=T2),
              dict(kind="layernorm", p=p + "norm3", ins=(T2,), out=TGT)]
    P.append(dict(kind="layernorm", p="decoder.norm", ins=(TGT,), out=HS))
    return P


def _lin(sd, e):
    """Weight and bias of a plan entry (rows = (a, b): rows [a D, b D) of a packed in_proj)."""
    if e["p"].endswith("in_proj"):
        w, b = sd[e["p"] + "_weight"], sd[e["p"] + "_bias"]
        D = w.shape[1]
        a, z = e["rows"]
        return w[a * D:z * D], b[a * D:z * D]
    return sd[e["p"] + ".weight"], sd[e["p"] + ".bias"]


def run_step(e, bufs, sd, pos, mask, H, scale=1.0 / math.sqrt(32.0)):
    """The float64 reference of launch `e` on the buffers it read (bufs: id -> tensor, encoder [L,B,X], decoder [B,X]); pos [L,Bp,D].
    Returns the Step, shaped like the buffer it writes."""
    k = e["kind"]
    x = bufs[e["ins"][0]]
    if k == "add_pos":
        return add_pos(x, pos)
    if k == "add_query_pos":
        return add_pos(x, bufs[e["ins"][1]])
    if k == "gemm":
        w, b = _lin(sd, e)
        L, B, _ = x.shape
        res = bufs[e["res"]].reshape(L * B, -1) if e.get("res") is not None else None
        st = gemm(x.reshape(L * B, -1), w, b, res, e.get("relu", False))
        for a in ("ref", "mag", "bound", "r32", "tf32"):
            setattr(st, a, getattr(st, a).reshape(L, B, -1))
        return st
    if k == "attention":
        return attention(x, bufs[e["ins"][1]], mask, H, scale)
    if k == "attention_q1":
        return attention_q1(x, bufs[e["ins"][1]], bufs[e["ins"][2]], mask, H, scale)
    if k == "layernorm":
        return layernorm(x, sd[e["p"] + ".weight"], sd[e["p"] + ".bias"])
    if k == "small_linear":
        w, b = _lin(sd, e)
        return small_linear(x, w, b, bufs[e["res"]] if e.get("res") is not None else None, e.get("relu", False))
    raise ValueError(k)


def compose(sd, src, pos, mask, query_embed, H, n_enc, n_dec, dtype=F64):
    """Transformer.forward composed launch by launch from `run_step` (each step fed the previous steps' float64 values, cast to
    `dtype`) -> (hs [B,D], memory [L,B,D])."""
    L, B, D = src.shape
    sd = {k: v.to(dtype) for k, v in sd.items()}
    bufs = {SRC: src.to(dtype), TGT: torch.zeros(B, D, dtype=dtype, device=src.device),
            QPOS: query_embed.reshape(1, D).expand(B, D).to(dtype)}
    memory = None
    for e in launch_plan(n_enc, n_dec):
        if e["kind"] == "add_pos" and e["out"] == MEM_POS:
            memory = bufs[SRC]
        bufs[e["out"]] = run_step(e, bufs, sd, pos.to(dtype), mask, H).ref.to(dtype)
    return bufs[HS], memory
