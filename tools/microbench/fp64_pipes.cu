// Per-SM issue rates that bound the small-front kernels on sm_90a: vector DFMA, 64-bit warp shuffles, LDS.64 broadcast,
// rcp.approx.f64, and the dependent-chain latency of DFMA / SHFL.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_pipes fp64_pipes.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void __launch_bounds__(256) k(double* out, int iters, double seed) {
    double a[16];
    for (int i = 0; i < 16; ++i) a[i] = seed * (threadIdx.x + i + 1);
    const double m = 1.0 + seed, c = seed * 0.5;
    __shared__ double sh[1024];
    for (int i = threadIdx.x; i < 1024; i += 256) sh[i] = seed * i;
    __syncthreads();
    for (int it = 0; it < iters; ++it) {
        if (MODE == 0) {            // 16 independent DFMA chains
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = fma(a[i], m, c);
        } else if (MODE == 1) {     // 16 independent 64-bit shuffles
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = __shfl_sync(0xffffffffu, a[i], (threadIdx.x + i + 1) & 31);
        } else if (MODE == 2) {     // dependent DFMA chain (latency)
#pragma unroll
            for (int i = 0; i < 16; ++i) a[0] = fma(a[0], m, c);
        } else if (MODE == 3) {     // dependent shuffle chain (latency)
#pragma unroll
            for (int i = 0; i < 16; ++i) a[0] = __shfl_sync(0xffffffffu, a[0], (threadIdx.x + 1) & 31);
        } else if (MODE == 4) {     // 16 LDS.64 broadcast loads + DFMA
#pragma unroll
            for (int i = 0; i < 16; ++i) a[i] = fma(a[i], sh[(it * 16 + i) & 1023], c);
        } else if (MODE == 5) {     // rcp.approx.ftz.f64 + 2 Newton steps, dependent
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                double r; asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(a[0]));
                r = fma(r, fma(-a[0], r, 1.0), r); r = fma(r, fma(-a[0], r, 1.0), r);
                a[0] = r + m;
            }
        } else if (MODE == 6) {     // 16 independent FFMA chains (fp32 reference point)
            float* fa = reinterpret_cast<float*>(a);
#pragma unroll
            for (int i = 0; i < 16; ++i) fa[i] = fmaf(fa[i], (float)m, (float)c);
        }
    }
    double s = 0; for (int i = 0; i < 16; ++i) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int MODE>
void run(const char* name, int sms, double clk_ghz) {
    double* out; cudaMalloc(&out, (size_t)sms * 8 * 256 * 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 2000;
    for (int warps = 1; warps <= 32; warps *= 2) {
        const int threads = warps >= 8 ? 256 : warps * 32, ctas = warps >= 8 ? warps / 8 : 1;
        k<MODE><<<sms * ctas, threads>>>(out, 10, 1e-9);
        cudaEventRecord(e0); k<MODE><<<sms * ctas, threads>>>(out, iters, 1e-9); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        const double cyc = ms * 1e-3 * clk_ghz * 1e9;
        const double warp_instr_per_clk_per_sm = (double)iters * 16 * warps / cyc;
        printf("%-28s %2d warps/SM: %.3f warp-instr/clk/SM  (%.1f clk per 16-instr iteration per warp)\n", name, warps, warp_instr_per_clk_per_sm, cyc / iters);
    }
    cudaFree(out);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int khz; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double ghz = khz * 1e-6;
    printf("%s, %d SMs, %.3f GHz nominal\n", p.name, p.multiProcessorCount, ghz);
    run<0>("DFMA independent", p.multiProcessorCount, ghz);
    run<2>("DFMA dependent chain", p.multiProcessorCount, ghz);
    run<1>("SHFL.64 independent", p.multiProcessorCount, ghz);
    run<3>("SHFL.64 dependent chain", p.multiProcessorCount, ghz);
    run<4>("LDS.64 broadcast + DFMA", p.multiProcessorCount, ghz);
    run<5>("rcp64 + 2 Newton dependent", p.multiProcessorCount, ghz);
    run<6>("FFMA independent", p.multiProcessorCount, ghz);
    return 0;
}
