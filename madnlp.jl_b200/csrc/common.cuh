// Shared helpers for the b200kkt CUDA translation units.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>

#include "../../include/b200kkt.h"
#ifdef __CUDACC__
#include "ptx.cuh"
#endif

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

// grid of a grid-stride elementwise kernel of 256-thread CTAs over n entries
inline int grid_elem(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, 8 * sm_count())); }

// argument check of a C entry point: on failure, records "<who>: invalid argument" and returns B2_ERR_INVALID
#define B2_NEED(cond, who) do { if (!(cond)) { ::b2::set_error(who ": invalid argument"); return B2_ERR_INVALID; } } while (0)

#ifdef __CUDACC__
#define GRID_STRIDE(i, n) for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

__device__ __forceinline__ double dinf() { return __longlong_as_double(0x7ff0000000000000LL); }
// sign flip as Julia's unary minus does it, NaN payload and sign included (neg.f64 returns the canonical NaN)
__device__ __forceinline__ double neg(double v) { return __longlong_as_double(__double_as_longlong(v) ^ (long long)0x8000000000000000ULL); }

// Julia's min / max on Float64 (base/math.jl): diff = x - y; a NaN operand returns diff, otherwise the sign of diff decides
// (so -0.0 is below +0.0)
__device__ __forceinline__ double jl_min(double x, double y) {
    const double d = __dsub_rn(x, y);
    if (x != x || y != y) return d;
    return signbit(d) ? x : y;
}
__device__ __forceinline__ double jl_max(double x, double y) {
    const double d = __dsub_rn(x, y);
    if (x != x || y != y) return d;
    return signbit(d) ? y : x;
}
// Julia's clamp(x, lo, hi) = x > hi ? hi : (x < lo ? lo : x)
__device__ __forceinline__ double jl_clamp(double x, double lo, double hi) { return x > hi ? hi : (x < lo ? lo : x); }

// is key in the ascending index array a[0:n)?  (ind_llb / ind_uub membership of dual_inf_perturbation!)
__device__ __forceinline__ bool contains(const int64_t* __restrict__ a, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const int64_t v = a[mid];
        if (v == key) return true;
        if (v < key) lo = mid + 1; else hi = mid;
    }
    return false;
}

// body of a C entry point that launches one grid-stride elementwise kernel over tot entries (nothing when tot = 0)
#define B2_LAUNCH(who, kern, tot, ...) do {                                                                                        \
        if ((tot) == 0) return B2_OK;                                                                                              \
        cudaError_t e__ = ::b2::launch_pdl(kern, dim3(::b2::grid_elem(tot)), dim3(256), 0, ::b2::as_stream(stream), __VA_ARGS__);  \
        if (e__ != cudaSuccess) return ::b2::cuda_fail(e__, who, __FILE__, __LINE__);                                             \
        return B2_OK;                                                                                                              \
    } while (0)
#endif

// ---- programmatic dependent launch (PDL): the launch side.  The kernel side (pdl_trigger / pdl_wait / pdl_sync) and its rules
// are in ptx.cuh.
#ifdef __CUDACC__
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

// ---- conditional graph nodes (refine_loop.cu), shared by the refinement-loop and the inertia-correction graphs
// the CUDA errors by which a driver refuses conditional nodes (anything else is a fault and is reported as one)
bool conditional_unsupported(cudaError_t e);
// leave no capture open on the stream (a capture-to-graph's graph belongs to its owner) and clear the sticky error
void abort_capture(cudaStream_t st);
// solve_refine!'s stopping rule and the KKT type's inertia test after one refinement step, one thread; sets `cond` (a WHILE node)
cudaError_t launch_refine_test(cudaStream_t st, cudaGraphConditionalHandle cond, const double* norms, const b2_inertia_source& src,
                               int64_t expect_pos, int64_t expect_neg, int32_t max_iter, double tol, b2_refine_record* rec,
                               b2_refine_record* out);

}  // namespace b2
