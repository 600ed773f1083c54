// Error plumbing and device queries shared by all translation units.
#include "common.cuh"

#include <mutex>

namespace b2 {

static thread_local std::string g_err;

void set_error(const std::string& msg) { g_err = msg; }

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    char buf[512];
    snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    g_err = buf;
    cudaGetLastError();   // clear sticky-less errors
    return B2_ERR_CUDA;
}

int sm_count() {
    static int cached = 0;
    if (cached) return cached;
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cached = n;
    return n;
}

}  // namespace b2

extern "C" {

const char* b2_last_error(void) { return b2::g_err.c_str(); }

int b2_version(void) { return 100; }   // 0.1.0

int b2_device_count(int* count) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (count) *count = (e == cudaSuccess) ? n : 0;
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        b2::set_error("no CUDA device visible");
        return B2_ERR_NO_DEVICE;
    }
    return B2_OK;
}

}  // extern "C"
