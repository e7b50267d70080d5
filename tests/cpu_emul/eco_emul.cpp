// TEST INFRASTRUCTURE ONLY.  Runs csrc/eco_cg_kernel.cuh -- the same source the CUDA build compiles -- on the CPU under cuda_shim.h,
// with the launch plan of eco_plan() for `max_ctas` co-resident CTAs of `block` threads.  Built and called by tests/test_eco_cpu.py.
#include "cuda_shim.h"

#include "../../pytracking_b200/csrc/eco_cg_kernel.cuh"
#include "../../pytracking_b200/csrc/eco_joint_kernel.cuh"

#include <cstdlib>

using namespace b200trk;

// plain build: one OS thread per CUDA thread (ThreadSanitizer sees every hand-over; small grids).  -DB200_EMUL_COOP_FIBERS: a block = one OS
// thread, its threads = fibers -- the launch plan of a real H100 (132 CTAs x 256 threads) at ECO's real block sizes becomes affordable.
#ifdef B200_EMUL_COOP_FIBERS
#define ECO_LAUNCH cpu_emul::launch_coop
#else
#define ECO_LAUNCH cpu_emul::launch
#endif

template <int G, int CPL>
static void run(const EcoPlan& pl, const EcoParams& P) {
    ECO_LAUNCH(eco_cg_kernel<G, CPL>, (unsigned)pl.grid, (unsigned)pl.block, pl.smem_bytes, P);
}

extern "C" int eco_emul_filter_cg(float* hf, const float* samples, const float* yf, const float* sw, const float* reg_filter, int rh, int rw,
                                  float* sample_energy, int has_energy, const float* new_xf, float* p_state, float* r_prev_state,
                                  float* rho_state, int has_state, int H, int Wh, int N, int C, int num_iter, int fletcher_reeves,
                                  int standard_alpha, float dff, float lr, float pdp, float prp, int max_ctas, int block,
                                  int force_res_slabs, int* plan_out) {
    if (!(C == 16 || C == 32 || C == 64 || C == 128) || rh > H || rw > Wh || rh > 8 || rw > 8) return 2;   // as b200trk_eco_filter_cg rejects
    EcoPlan pl = eco_plan(H, Wh, N, C, num_iter, max_ctas, block);
    if (force_res_slabs >= 0 && force_res_slabs < pl.res_slabs) pl.res_slabs = force_res_slabs;   // exercise the streaming path
    std::vector<unsigned char> ws(pl.ws_bytes + 64, 0xCD);
    unsigned char* w = ws.data();
    EcoParams P{};
    P.hf = hf; P.samples = samples; P.yf = yf; P.sw = sw; P.reg_filter = reg_filter; P.sample_energy = sample_energy;
    P.new_xf = new_xf; P.p_state = p_state; P.r_prev_state = r_prev_state; P.rho_state = rho_state;
    P.has_state = (has_state && dff != 0.f) ? 1 : 0;
    P.has_energy = has_energy;
    P.H = H; P.Wh = Wh; P.N = N; P.C = C; P.rh = rh; P.rw = rw; P.num_iter = num_iter;
    P.fletcher_reeves = fletcher_reeves; P.standard_alpha = standard_alpha;
    P.dff = dff; P.lr = lr; P.pdp = pdp; P.prp = prp;
    P.xw = (float2*)(w + pl.off_xw); P.pw = (float2*)(w + pl.off_pw); P.resw = (float2*)(w + pl.off_resw);
    P.rpw = (float2*)(w + pl.off_rpw); P.qw = (float2*)(w + pl.off_qw); P.dM = (float*)(w + pl.off_dM);
    P.dots = (float*)(w + pl.off_dots); P.barrier = (unsigned*)w;
    P.GPP = pl.GPP; P.res_slabs = pl.res_slabs; P.npx_max = pl.npx_max;
    if (plan_out) { plan_out[0] = pl.grid; plan_out[1] = pl.G; plan_out[2] = pl.CPL; plan_out[3] = pl.GPP; plan_out[4] = pl.res_slabs; plan_out[5] = pl.npx_max; }
    if (pl.G == 16 && pl.CPL == 1) run<16, 1>(pl, P);
    else if (pl.G == 32 && pl.CPL == 1) run<32, 1>(pl, P);
    else if (pl.G == 32 && pl.CPL == 2) run<32, 2>(pl, P);
    else if (pl.G == 32 && pl.CPL == 4) run<32, 4>(pl, P);
    else return 2;
    return 0;
}

// the launch plan alone (what the CUDA launcher would choose for `max_ctas` SMs): grid, G, CPL, GPP, res_slabs, npx_max, smem bytes
extern "C" void eco_emul_plan(int H, int Wh, int N, int C, int num_iter, int max_ctas, int block, long long* out) {
    const EcoPlan pl = eco_plan(H, Wh, N, C, num_iter, max_ctas, block);
    out[0] = pl.grid; out[1] = pl.G; out[2] = pl.CPL; out[3] = pl.GPP; out[4] = pl.res_slabs; out[5] = pl.npx_max;
    out[6] = (long long)pl.smem_bytes; out[7] = (long long)pl.ws_bytes;
}

// ---- first-frame joint optimisation (csrc/eco_joint_kernel.cuh) ----------------------------------------------------------------
extern "C" int eco_emul_joint_gn(float* hf, float* proj, const float* samples, const float* yf, const float* sw_sqrt, const float* reg_filter,
                                 int rh, int rw, const float* dMh, float dMP, float projection_reg, int H, int Wh, int N, int Cin, int C,
                                 int num_cg, int num_gn, int max_ctas, int block, int force_res_slabs, int* plan_out) {
    if (rh > H || rw > Wh || rh > 8 || rw > 8) return 2;                                      // as b200trk_eco_joint_gn rejects
    EcoJointPlan pl = eco_joint_plan(H, Wh, N, Cin, C, num_cg, num_gn, max_ctas, block);
    if (force_res_slabs >= 0 && force_res_slabs < pl.res_slabs) pl.res_slabs = force_res_slabs;
    if (force_res_slabs == 0) pl.stage_pm = 0;                                                // ... and the projection matrix from global memory
    std::vector<unsigned char> ws(pl.ws_bytes + 64, 0xCD);
    unsigned char* w = ws.data();
    const size_t field = (size_t)H * Wh * C * 2 * sizeof(float), nelem = (size_t)Cin * C;
    EcoJointParams P{};
    P.hf = hf; P.proj = proj; P.samples = samples; P.yf = yf; P.sw_sqrt = sw_sqrt; P.reg_filter = reg_filter; P.dMh_in = dMh;
    P.dMP = dMP; P.lambda = projection_reg;
    P.H = H; P.Wh = Wh; P.N = N; P.Cin = Cin; P.C = C; P.rh = rh; P.rw = rw; P.num_cg = num_cg; P.num_gn = num_gn;
    P.h0w = (float2*)(w + pl.off_fields); P.phw = (float2*)(w + pl.off_fields + field); P.xhw = (float2*)(w + pl.off_fields + 2 * field);
    P.rhw = (float2*)(w + pl.off_fields + 3 * field); P.qhw = (float2*)(w + pl.off_fields + 4 * field);
    P.dMh = (float*)(w + pl.off_dMh); P.c0w = (float2*)(w + pl.off_c0); P.wv = (float2*)(w + pl.off_wv);
    P.pP = (float*)(w + pl.off_P); P.xP = P.pP + nelem; P.rP = P.xP + nelem; P.qP = P.rP + nelem;
    P.dots = (float*)(w + pl.off_dots); P.barrier = (unsigned*)w;
    P.res_slabs = pl.res_slabs; P.npx_max = pl.npx_max; P.EPB = pl.EPB; P.SPL = pl.SPL; P.stage_pm = pl.stage_pm; P.wide = pl.wide;
    if (plan_out) { plan_out[0] = pl.grid; plan_out[1] = pl.res_slabs; plan_out[2] = pl.npx_max; plan_out[3] = pl.EPB; plan_out[4] = pl.SPL; plan_out[5] = (int)pl.smem_bytes; }
    ECO_LAUNCH(eco_joint_kernel, (unsigned)pl.grid, (unsigned)pl.block, pl.smem_bytes, P);
    return 0;
}
