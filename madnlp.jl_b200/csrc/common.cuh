// Shared helpers for the b200kkt CUDA translation units.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>

#include "../../include/b200kkt.h"

namespace b2 {

void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define B2_CUDA(call)                                                         \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) return ::b2::cuda_fail(e__, #call, __FILE__, __LINE__); \
    } while (0)

#define B2_CUDA_THROW(call)                                                   \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) { ::b2::cuda_fail(e__, #call, __FILE__, __LINE__); throw std::runtime_error("cuda"); } \
    } while (0)

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    cudaError_t alloc(size_t count) {
        release();
        n = count;
        if (count == 0) return cudaSuccess;
        return cudaMalloc((void**)&p, count * sizeof(T));
    }
    cudaError_t upload(const T* h, size_t count) {
        cudaError_t e = alloc(count);
        if (e != cudaSuccess || count == 0) return e;
        return cudaMemcpy(p, h, count * sizeof(T), cudaMemcpyHostToDevice);
    }
    size_t bytes() const { return n * sizeof(T); }
};

inline cudaStream_t as_stream(void* s) { return (cudaStream_t)s; }

// number of SMs of the current device (cached)
int sm_count();

// ---- programmatic dependent launch (PDL).  A kernel launched through launch_pdl() may be scheduled while its predecessor
// in the stream is still running; it must not touch anything the predecessor produces before pdl_wait() returns (and must
// pass pdl_wait() before it exits, so that ITS completion implies the predecessor's).  Kernels with nothing to prefetch
// simply start with pdl_sync(): what overlaps is the launch latency.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_trigger(); pdl_wait(); }
template <typename... P, typename... A>
inline cudaError_t launch_pdl(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<A>(args)...);
}
#endif

}  // namespace b2
