"""Launch plans of ECO's two optimiser kernels, the integer arithmetic of `eco_plan` (csrc/eco_cg_kernel.cuh) and `eco_joint_plan`
(csrc/eco_joint_kernel.cuh) restated: which decomposition a problem gets on a device with `sms` SMs.  The plug-in asks whether the joint
kernel takes a feature block before it claims the call; the float64 step tests choose their cases by the plans they reach."""

ECO_MAX_TAPS = 15 * 15
ECO_SMEM_LIMIT = 227 * 1024 - 1024           # what a plan may carve; the launcher refuses more than 227 KB
BLOCK = 256


def _r4(n):
    return (n + 3) & ~3


def eco_fixed_smem_floats(N, C, npx_max, ngrp):
    return 3 * (ECO_MAX_TAPS + 3) + 8 + 32 + _r4(N) + _r4(npx_max) + ngrp * C * 2


def eco_plan(H, Wh, N, C, num_iter, sms, block=BLOCK):
    """eco_cg_kernel's plan: dict(grid, G, CPL, GPP, res_slabs, npx_max, smem_bytes, ws_bytes)."""
    P = H * Wh
    grid = min(P, sms)
    G = 32 if C >= 32 else 16
    npx_max = (P + grid - 1) // grid
    ngrp = block // G
    gpp = 1
    while gpp * 2 * npx_max <= ngrp:
        gpp *= 2
    fixed = eco_fixed_smem_floats(N, C, npx_max, ngrp) * 4
    slab = N * C * 2 * 4
    res = min((ECO_SMEM_LIMIT - fixed) // slab if fixed < ECO_SMEM_LIMIT else 0, npx_max)
    field = P * C * 2 * 4
    off = 256 + 5 * field + field // 2
    off = (off + 255) & ~255
    ws = off + (3 * num_iter + 4) * grid * 2 * 4
    return dict(grid=grid, G=G, CPL=C // G, GPP=gpp, res_slabs=res, npx_max=npx_max, smem_bytes=fixed + res * slab, ws_bytes=ws)


def ecoj_fixed_smem_floats(N, Cin, C, block=BLOCK):
    return 3 * (ECO_MAX_TAPS + 3) + 8 + 32 + _r4(N) + (block // 32) * (4 * C + 2 * Cin + 2 * _r4(N)) + block


def ecoj_stage_floats(Cin, C):
    return (Cin * (C + 1) + 1) & ~1


def eco_joint_fits(N, Cin, C, block=BLOCK):
    """Whether the joint kernel's fixed shared memory fits (the sample slabs may all stream)."""
    return ecoj_fixed_smem_floats(N, Cin, C, block) * 4 <= ECO_SMEM_LIMIT


def eco_joint_plan(H, Wh, N, Cin, C, num_cg, num_gn, sms, block=BLOCK):
    """eco_joint_kernel's plan: dict(grid, res_slabs, npx_max, EPB, SPL, stage_pm, wide, smem_bytes, ws_bytes)."""
    P = H * Wh
    grid = min(P, sms)
    npx_max = (P + grid - 1) // grid
    wide = 1 if npx_max * 2 <= block // 32 else 0
    fixed = ecoj_fixed_smem_floats(N, Cin, C, block) * 4
    slab = N * (Cin + 1) * 2 * 4
    stage_pm = 1 if fixed + ecoj_stage_floats(Cin, C) * 4 <= ECO_SMEM_LIMIT else 0
    if stage_pm:
        fixed += ecoj_stage_floats(Cin, C) * 4
    res = min((ECO_SMEM_LIMIT - fixed) // slab if fixed < ECO_SMEM_LIMIT else 0, npx_max)
    nelem = Cin * C
    epb = min(((nelem + grid - 1) // grid + 15) & ~15, block)
    field = P * C * 2 * 4
    off = 256 + 5 * field + field // 2 + P * N * C * 2 * 4 + P * Cin * 2 * 4 + 4 * nelem * 4
    off = (off + 255) & ~255
    ws = off + ((2 * num_cg + 2) * num_gn + 4) * grid * 2 * 4
    return dict(grid=grid, res_slabs=res, npx_max=npx_max, EPB=epb, SPL=block // epb, stage_pm=stage_pm, wide=wide,
                smem_bytes=fixed + res * slab, ws_bytes=ws)
