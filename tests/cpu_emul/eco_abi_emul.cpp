// TEST INFRASTRUCTURE ONLY -- the ECO entry points of the C ABI (include/b200trk.h) as a HOST library: the launchers' source files
// themselves (csrc/eco_cg.cu, csrc/eco_loc.cu: validation, launch plans, workspace, parameter binding) compiled as C++ over cuda_shim.h /
// cuda_host_shim.h, the kernels executed by the shim's launchers (a block = one OS thread, its threads = fibers; cooperative grids with the
// pthread grid barrier) with the launch an H100 makes (device_sm_count() = 132).  tests/test_eco_gpu_file_on_cpu.py loads it in place of
// libb200trk.so to run tests/test_zz_eco_gpu.py -- the `-m gpu` tests of these entry points -- on the CPU.
#include "cuda_shim.h"
#include "cuda_host_shim.h"

#include "../../pytracking_b200/csrc/eco_cg.cu"
#include "../../pytracking_b200/csrc/eco_loc.cu"

extern "C" const char* b200trk_last_error(void) { return b200trk::g_emul_error; }
