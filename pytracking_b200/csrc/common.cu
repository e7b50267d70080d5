// Error reporting, launch accounting and the per-device scratch workspace of libb200trk.
#include "common.cuh"
#include <cstring>
#include <mutex>

namespace b200trk {

static thread_local char g_err[1024] = "";
std::atomic<uint64_t> g_launch_count{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

constexpr int kMaxDevices = 16;
constexpr int kSlots = 8;
struct Ws { void* ptr = nullptr; size_t bytes = 0; };
static Ws g_ws[kMaxDevices][kSlots];
static int g_sm_count[kMaxDevices] = {0};
static std::mutex g_mu;

void* workspace(size_t bytes, int slot) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices || slot < 0 || slot >= kSlots) {
        set_error("workspace: bad device/slot (%d/%d)", dev, slot);
        return nullptr;
    }
    std::lock_guard<std::mutex> lk(g_mu);
    Ws& w = g_ws[dev][slot];
    if (w.bytes >= bytes) return w.ptr;
    // grow: previous users of the old buffer are stream ordered before us on the caller's single stream, but the
    // free itself is not, so drain the device first (rare: only while sizes are still growing).
    if (w.ptr) {
        cudaDeviceSynchronize();
        cudaFree(w.ptr);
        w.ptr = nullptr; w.bytes = 0;
    }
    size_t want = bytes + bytes / 4 + 4096;
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        set_error("workspace: cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        return nullptr;
    }
    cudaMemset(p, 0, want);
    w.ptr = p; w.bytes = want;
    return p;
}

int device_sm_count() {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices) return 1;
    if (g_sm_count[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        g_sm_count[dev] = n > 0 ? n : 1;
    }
    return g_sm_count[dev];
}

}  // namespace b200trk

// debug: copy the SD optimiser phase trace (128 x u64) to the host
extern "C" int b200trk_debug_sd_trace(unsigned long long* out_host) {
    void* p = b200trk::workspace(1024, 3);
    if (!p || !out_host) return 1;
    return cudaMemcpy(out_host, p, 1024, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : 1;
}

// debug: per-unit pipeline stamps of the tensor-core SD kernel ([16 units][16] x u64 SM clocks, CTA 0, first adjoint sweep; cleared after the read)
extern "C" int b200trk_debug_sd_units(unsigned long long* out_host) {
    char* p = (char*)b200trk::workspace(4096, 3);
    if (!p || !out_host) return 1;
    if (cudaMemcpy(out_host, p + 1024, 2048, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    return cudaMemset(p + 1024, 0, 2048) == cudaSuccess ? 0 : 1;      // (stamps of the next run start from a clean table)
}

extern "C" int b200trk_version(void) { return B200TRK_VERSION; }
extern "C" const char* b200trk_last_error(void) { return b200trk::g_err; }
extern "C" uint64_t b200trk_launch_count(void) { return b200trk::g_launch_count.load(); }
