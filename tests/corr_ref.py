"""Float64 reference of the stage-2 correlation kernels (csrc/corr_kernels.cuh) and a mirror of their launch plan.

    apply    s[i,y,x] = sum_{c,u,v} xpad[i,c,y+u,x+v] w[c,u,v]      F.conv2d(x, w, padding=2); conv2d_same crops it to [:FS, :FS]
    adjoint  g[c,u,v] = sum_{i,y,x} r[i,y,x] xpad[i,c,y+u,x+v]      one F.conv2d with the samples as input channels

Both run on the device of their inputs.  `magnitude` is the same operation on |x|, |w| and |r|: the sum of the absolute terms of every
entry.  `corr_plan(op, n, C, FS, sms)` restates corr_plan of corr_kernels.cuh (tests/test_corr_f64_cpu.py pins it to the kernels' own
function) and adds the summation depth D of each output entry under that plan:

    apply    D = 16 passes + SLOTS + NCH      a slot's FMA chain over its passes, the sum over the slots, the last CTA's sum over the chunks
    adjoint  D = 20 spc_max + NT + NG         a tile's FMA chain over its samples, the sum over the 20 / 30 tiles, the sum over the groups

so that every entry k of the kernel obeys |k - f64| <= gamma_D sum|terms| + u |k|, gamma_D = D u / (1 - D u), u = 2^-24 (`bar`).
`features` names the plan features a call reaches; `cases(sms)` is the case list of tests/test_corr_f64_gpu.py; `max2d_maps` the
maps its max2d check orders."""
import torch
import torch.nn.functional as F

U = 2.0 ** -24
SLOTS = {18: 16, 22: 8}
NT = {18: 20, 22: 30}                      # 5x4 output tiles of a 19x19 / 23x23 map
SPC_CAP = 8
MAX_N = 1024                               # apply: arrival counters per call
MAX_NCH = 1024                             # adjoint: arrival counters per call


def apply(x, w, crop=False):
    """[n,C,FS,FS] x [1,C,4,4] -> [n,1,FS+1,FS+1] in float64 ([n,1,FS,FS] with the 'same' crop)."""
    s = F.conv2d(x.double(), w.double(), padding=2)
    return s[..., :x.shape[-2], :x.shape[-1]] if crop else s


def adjoint(x, r):
    """[n,C,FS,FS], r [n,1,FS+1,FS+1] -> [1,C,4,4] in float64."""
    n, C, H, W = x.shape
    xp = F.pad(x.double(), (2, 2, 2, 2)).transpose(0, 1)          # [C, n, FS+4, FS+4]
    g = F.conv2d(xp, r.double().reshape(1, n, H + 1, W + 1))       # [C, 1, 4, 4]
    return g.reshape(1, C, 4, 4)


def magnitude(op, x, y, crop=False):
    """sum |terms| of every entry: op 'apply' (y = w) or 'adjoint' (y = r)."""
    return apply(x.abs(), y.abs(), crop) if op == "apply" else adjoint(x.abs(), y.abs())


def gamma(D):
    return D * U / (1 - D * U)


def bar(k, mag, D):
    """Entry-wise bound on |k - f64|: gamma_D sum|terms| + u |k|."""
    return gamma(D) * mag + U * k.double().abs()


def corr_plan(op, n, C, FS, sms):
    """corr_plan of corr_kernels.cuh for op 'apply' (also conv2d_same) or 'adjoint', plus the grid and the depth D of every entry."""
    slots = SLOTS[FS]
    passes = 0
    for q in (4, 2, 1) if (op == "adjoint" or n >= 16) else (1,):
        if C % (slots * q) == 0:
            passes = q
            break
    p = dict(op=op, n=n, C=C, FS=FS, sms=sms, slots=slots, passes=passes, nch=0, ng=n, spc_max=1)
    if not passes:
        return p
    nch = C // (slots * passes)
    p["nch"] = nch
    if op == "apply":
        p["grid"] = (nch, n)
        p["depth"] = 16 * passes + slots + nch
        return p
    ng = min(max(sms // nch, 1), n)
    if -(-n // ng) > SPC_CAP:
        ng = -(-n // SPC_CAP)
    p["ng"], p["spc_max"] = ng, -(-n // ng)
    p["grid"] = (nch, ng)
    p["depth"] = 20 * p["spc_max"] + NT[FS] + ng
    return p


def features(p):
    """The plan features one call reaches (names of the form '<op><FS> <feature>')."""
    t = "%s%d " % (p["op"], p["FS"])
    n, nch, slots = p["n"], p["nch"], p["slots"]
    f = {t + "passes%d %s" % (p["passes"], "n<16" if n < 16 else "n>=16")}
    f.add(t + ("nch1" if nch == 1 else "nch>1") + (" n<16" if p["op"] == "apply" and n < 16 else ""))
    if p["op"] == "apply":
        f.add(t + "passes%d nch%s" % (p["passes"], "1" if nch == 1 else ">1"))
        if nch == 512 // slots:
            f.add(t + "nch=512/SLOTS")
        if n in (16, MAX_N):
            f.add(t + "n=%d" % n)
        return f
    f.add(t + "passes%d nch%s" % (p["passes"], "1" if nch == 1 else ">1"))
    ng, sms = p["ng"], p["sms"]
    if ng == n:
        f.add(t + "NG=n")
    elif ng == sms // nch and n % ng:
        f.add(t + "NG=sms/NCH<n uneven")
    elif ng > max(sms // nch, 1):
        f.add(t + "NG raised by the cap")
    if nch > sms:
        f.add(t + "NG=1 NCH>sms")
    if p["spc_max"] == SPC_CAP:
        f.add(t + "spc=8")
    return f


def required_features():
    """Every feature the GPU file must reach at the device's SM count."""
    req = set()
    for FS in (18, 22):
        a = "apply%d " % FS
        req |= {a + "passes1 n<16", a + "passes4 n>=16", a + "passes2 n>=16", a + "passes1 n>=16", a + "nch1 n<16", a + "nch1",
                a + "nch=512/SLOTS", a + "n=16", a + "n=%d" % MAX_N}
        t = "adjoint%d " % FS
        req |= {t + "passes%d nch%s" % (q, m) for q in (4, 2, 1) for m in ("1", ">1")}
        req |= {t + "NG=n", t + "NG=sms/NCH<n uneven", t + "NG raised by the cap", t + "spc=8"}
    req.add("adjoint22 NG=1 NCH>sms")
    return req


def cases(sms, small=False):
    """(op, FS, n, C) of the float and integer checks.  The tracker shapes: DiMP-50 classify (n = 1, C = 512) and its S scales, PrDiMP at
    22x22, ATOM's C = 64 at n = 30 and 250, the memories n = 15 and 50; then the shapes that complete the plan features.  `small` keeps
    the cases the CPU tier can afford."""
    out = []
    for FS in (18, 22):
        s = SLOTS[FS]
        apply_nc = [(1, 512), (3, 512), (15, 512), (1, s), (16, 512), (50, 512), (30, 64 if FS == 18 else 32),
                    (50, 6 * s), (50, 3 * s), (250, 64), (MAX_N, 4 * s)]
        adj_nc = [(3, s), (3, 2 * s), (3, 4 * s), (3, 8 * s), (3, 6 * s), (3, 3 * s), (15, 512), (30, 64), (50, 512), (250, 64),
                  (250, 512), (MAX_N, 512 if FS == 22 else 64)]
        out += [("apply", FS, n, C) for n, C in apply_nc] + [("adjoint", FS, n, C) for n, C in adj_nc]
    out.append(("adjoint", 22, 8, 1080))
    if small:
        out = [c for c in out if c[2] * c[3] <= 4096]
    return out


def all_features(sms, case_list=None):
    got = set()
    for op, FS, n, C in (case_list or cases(sms)):
        got |= features(corr_plan(op, n, C, FS, sms))
    return got


def max2d_maps(N, H, W, seed):
    """N maps of H x W cycling through the value classes dcf.max2d must order: finite, exact ties, +-0, +-inf, denormals, one NaN, several
    NaN, all NaN, all -inf, NaN beside +inf."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(N, H, W, generator=g)
    ri = lambda k: torch.randint(0, H * W, (k,), generator=g)
    for i in range(N):
        m = a[i].view(-1)
        cls = i % 10
        if cls == 1:
            m[ri(3)] = m.max() + 1
        elif cls == 2:
            m.copy_(torch.where(torch.rand(H * W, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0)))
        elif cls == 3:
            m[ri(2)] = float("inf"); m[ri(2)] = float("-inf")
        elif cls == 4:
            m.copy_(torch.randint(-3, 4, (H * W,), generator=g).float() * 1e-45)
        elif cls == 5:
            m[ri(1)] = float("nan")
        elif cls == 6:
            m[ri(4)] = float("nan")
        elif cls == 7:
            m.fill_(float("nan"))
        elif cls == 8:
            m.fill_(float("-inf"))
        elif cls == 9:
            m[ri(1)] = float("inf"); m[ri(2)] = float("nan")
    return a
