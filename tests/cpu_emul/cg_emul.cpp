// TEST INFRASTRUCTURE ONLY.  Runs csrc/atom_cg_kernel.cuh (ATOM's per-frame ConjugateGradient.run on ConvProblem as one persistent
// cooperative kernel on the cp.async sweeps of csrc/corr2.cuh -- the same sources the CUDA build compiles) on the CPU under cuda_shim.h.
// Two builds: plain (OS thread per CUDA thread, what ThreadSanitizer needs) runs ONE CTA -- the kernel keeps small arrays in static __shared__
// storage, which that mode can give to a single live block only; with -DB200_EMUL_COOP_FIBERS (a block = one OS thread, its threads = fibers,
// static __shared__ = thread_local) the grid is the one launch_cg (csrc/atom_cg.cu) picks for `sms` SMs, cross-CTA exchange included.  The pipeline depth NST
// is the one launch_cg picks (4, 3 or 2 stages).  Built and called by tests/test_sd_kernels_cpu.py and tests/test_atom_step_ref_cpu.py.
#include "cuda_shim.h"

#include "../../pytracking_b200/csrc/atom_cg_kernel.cuh"

using namespace b200trk;

template <int FS, int NST>
static int launch_nst(const CgParams& P, int ctas, size_t smem) {
#ifdef B200_EMUL_COOP_FIBERS
    cpu_emul::launch_coop(atom_cg_kernel<FS, NST>, (unsigned)ctas, (unsigned)Corr2<FS>::NCONS, smem, P);
#else
    (void)ctas;
    cpu_emul::launch(atom_cg_kernel<FS, NST>, 1u, (unsigned)Corr2<FS>::NCONS, smem, P);
#endif
    return 0;
}

template <int FS>
static int run_cg(CgParams P, int sms) {
    using K = Corr2<FS>;
    // launch_cg (csrc/atom_cg.cu): fewest channel passes per CTA that still keeps the samples of a CTA within shared memory
    int passes = 0, NCH = 0, NG = 0, spc = 0;
#ifndef B200_EMUL_COOP_FIBERS
    sms = 1;                                                 // one live block only (static __shared__ arrays): everything in one CTA
#endif
    for (int p = 1; p <= 4; p <<= 1) {
        if (P.C % (K::SLOTS * p) != 0) continue;
        const int nch = P.C / (K::SLOTS * p);
        if (nch > sms) continue;
        int ng = sms / nch; if (ng > P.n) ng = P.n; if (ng < 1) ng = 1;
        const int sp = (P.n + ng - 1) / ng;
        if (sp <= CG_SPC_MAX) { passes = p; NCH = nch; NG = ng; spc = sp; break; }
    }
    if (!passes) return 2;
    P.passes = passes; P.NCH = NCH; P.NG = NG; P.spc_max = spc;
    const size_t n_gpart = (size_t)NG * P.C * 16, n_qpart = (size_t)P.n * NCH * K::NPOS, n_dots = (size_t)(2 * P.num_iter + 4) * NCH * 2;
    std::vector<float> ws(n_gpart + n_qpart + n_dots + 128, -1e30f);
    std::vector<unsigned> bar(64, 0u);
    P.barrier = bar.data();
    P.gpart = ws.data(); P.qpart = P.gpart + n_gpart; P.dots = P.qpart + n_qpart;
    const int cchunk = passes * K::SLOTS;
    const size_t fixed = (size_t)(K::NT * K::SLOTS * K::RED_STRIDE + 6 * cchunk * K::VEC_STRIDE + spc * (2 * K::NPOS + K::PMAP) + K::NCONS * 4) * sizeof(float);
    const size_t item = (size_t)K::ITEM_FLOATS * sizeof(float);
    // pipeline depth as launch_cg picks it from the shared-memory budget (227 KB less the static arrays)
    const size_t limit = 227 * 1024 - 512;
    if (fixed + 4 * item <= limit) return launch_nst<FS, 4>(P, NCH * NG, fixed + 4 * item);
    if (fixed + 3 * item <= limit) return launch_nst<FS, 3>(P, NCH * NG, fixed + 3 * item);
    if (fixed + 2 * item > limit) return 2;
    return launch_nst<FS, 2>(P, NCH * NG, fixed + 2 * item);
}

extern "C" int cg_emul_atom_cg_filter(const float* filter, float* filter_out, const float* feat, const float* y, const float* sample_weight, int n, int C,
                                      int H, int W, int num_iter, float filter_reg, int fletcher_reeves, int activation, float act_param, int sms) {
    CgParams P{};
    P.w_in = filter; P.w_out = filter_out; P.feat = feat; P.y = y; P.sample_weight = sample_weight;
    P.n = n; P.C = C; P.num_iter = num_iter; P.fletcher_reeves = fletcher_reeves ? 1 : 0; P.act = activation; P.act_param = act_param; P.reg = filter_reg;
    if (H == 18 && W == 18) return run_cg<18>(P, sms);
    if (H == 22 && W == 22) return run_cg<22>(P, sms);
    return 2;
}
