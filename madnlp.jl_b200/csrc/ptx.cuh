// The inline-PTX primitives the kernels are built from: shared-window addresses, mbarriers and bulk copies, cp.async, ordered
// global accesses and the hand-off sentinel of the single-launch protocols, the bounded spin, the Newton reciprocal, named
// barriers, special registers and programmatic dependent launch.  Each is defined here and nowhere else.
#pragma once
#include <cuda_runtime.h>

namespace b2 {

// ---- shared-window address of a generic pointer into shared memory
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// ---- bounded spin: try ready(it) -- it = number of failed tries so far -- until it returns true, at most LIMIT times, with
// __nanosleep(SLEEP_NS) after each failed try (none when 0).  A wait that never ends would hang the device, so on time-out it
// sets *err and returns false instead.
template <unsigned LIMIT, unsigned SLEEP_NS, class Ready>
__device__ __forceinline__ bool bounded_spin(int* err, Ready ready) {
    for (unsigned it = 0; !ready(it);) {
        if (SLEEP_NS) __nanosleep(SLEEP_NS);
        if (++it >= LIMIT) {
            atomicExch(err, 1);
            return false;
        }
    }
    return true;
}

// ---- mbarrier in shared memory; the TMA unit completes a bulk copy on one by counting its bytes
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// makes the initialised barriers visible to the async proxy (the TMA unit); a __syncthreads() must follow before any thread uses them
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 1-D bulk copy global -> shared (16-byte aligned, a multiple of 16 bytes) that completes `bytes` on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// unbounded wait for the phase of the given parity to complete: the dense factorisation's hot loops, where the arrivals come
// from the same CTA
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
    unsigned done;
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return done != 0;
}
// bounded wait: at most LIMIT tries, then *err is set and the result is false
template <unsigned LIMIT>
__device__ __forceinline__ bool mbar_wait_bounded(unsigned long long* bar, unsigned parity, int* err) {
    return bounded_spin<LIMIT, 0>(err, [&](unsigned) { return mbar_try_wait(bar, parity); });
}

// ---- cp.async global -> shared: .ca caches in L1, .cg in L2 only (for data other CTAs of the same launch wrote)
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// !valid: writes 8 zero bytes and reads nothing (gsrc must still be a valid address)
__device__ __forceinline__ void cp_async8_zfill(void* smem_dst, const void* gsrc, bool valid) {
    const int sz = valid ? 8 : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async16_cg(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit_group() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ---- ordered global accesses at GPU scope (the cross-CTA protocols of the single-launch kernels)
__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int ld_relaxed(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// 8-byte loads and stores are single-copy atomic: a hand-off is one relaxed load of the value itself
__device__ __forceinline__ unsigned long long ld_relaxed_b64(const double* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
// two consecutive 8-byte words (16-byte aligned) in one access; each word is single-copy atomic on its own, not the pair
__device__ __forceinline__ void ld_relaxed_v2_b64(const double* p, unsigned long long& v0, unsigned long long& v1) {
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(v0), "=l"(v1) : "l"(p));
}
__device__ __forceinline__ void st_relaxed_v2_b64(double* p, unsigned long long v0, unsigned long long v1) {
    asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"(v0), "l"(v1) : "memory");
}
__device__ __forceinline__ void st_release(int* p, int v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_b64(double* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---- hand-off sentinel of the single-launch solves: a slot holds SLOT_EMPTY until its producer stores the value.  All ones -- a
// negative NaN with a full payload, which fp64 arithmetic never produces and a byte-wise cudaMemset(SLOT_EMPTY_BYTE) writes; a
// producer stores a value with that bit pattern (a NaN from the caller's right-hand side) as CANON_NAN instead.
constexpr int SLOT_EMPTY_BYTE = 0xff;
constexpr unsigned long long SLOT_EMPTY = ~0ull;
static_assert(SLOT_EMPTY == 0x0101010101010101ull * SLOT_EMPTY_BYTE, "a slot armed by cudaMemset(SLOT_EMPTY_BYTE) holds SLOT_EMPTY");
constexpr unsigned long long CANON_NAN = 0x7ff8000000000000ull;

// ---- 1 / x from the hardware reciprocal and two Newton corrections: within an ulp for normal x, and inline (the IEEE
// division's slow path is a call, which makes a kernel spill the registers live across it)
__device__ __forceinline__ double fast_rcp(double x) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    r = fma(r, fma(-x, r, 1.0), r);
    r = fma(r, fma(-x, r, 1.0), r);
    return r;
}

// ---- named barrier ID over the first N threads of the CTA
template <int ID, int N>
__device__ __forceinline__ void bar_sync() { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory"); }

// ---- special registers
__device__ __forceinline__ unsigned long long global_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ unsigned smid() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }

// ---- programmatic dependent launch (launch_pdl in common.cuh).  A kernel launched with the attribute may be scheduled while its
// predecessor in the stream is still running; it must not touch anything the predecessor produces before pdl_wait() returns (and
// must pass pdl_wait() before it exits, so that ITS completion implies the predecessor's).  Kernels with nothing to prefetch
// simply start with pdl_sync(): what overlaps is the launch latency.  Both are no-ops in a launch without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_trigger(); pdl_wait(); }

}  // namespace b2
