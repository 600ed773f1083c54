// Throughput + fragment-layout check of the fp64 tensor-core shapes on sm_90a:
//   mma.sync.aligned.{m8n8k4, m16n8k4, m16n8k8, m16n8k16}.row.col.f64.f64.f64.f64
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_shapes dmma_shapes.cu ; run: ./dmma_shapes
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

template <int SHAPE> struct Frag;
template <> struct Frag<0> { static constexpr int M = 8, N = 8, K = 4, NA = 1, NB = 1, NC = 2; };
template <> struct Frag<1> { static constexpr int M = 16, N = 8, K = 4, NA = 2, NB = 1, NC = 4; };
template <> struct Frag<2> { static constexpr int M = 16, N = 8, K = 8, NA = 4, NB = 2, NC = 4; };
template <> struct Frag<3> { static constexpr int M = 16, N = 8, K = 16, NA = 8, NB = 4, NC = 4; };

template <int S>
__device__ __forceinline__ void mma(double* c, const double* a, const double* b) {
    if constexpr (S == 0)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    else if constexpr (S == 1)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (S == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// ---- layout check: one warp computes C = A(MxK) * B(KxN) with the assumed fragment layout; host compares
template <int S>
__global__ void k_check(const double* A, const double* B, double* C) {   // A row-major MxK, B: B[k*N+n], C row-major MxN
    using F = Frag<S>;
    const int lane = threadIdx.x, g = lane >> 2, q = lane & 3;
    double a[8], b[4], c[4] = {0, 0, 0, 0};
    if constexpr (S == 0) { a[0] = A[g * F::K + q]; b[0] = B[q * F::N + g]; }
    else {
        for (int i = 0; i < F::NA; ++i) a[i] = A[(g + 8 * (i & 1)) * F::K + q + 4 * (i >> 1)];
        for (int i = 0; i < F::NB; ++i) b[i] = B[(q + 4 * i) * F::N + g];
    }
    mma<S>(c, a, b);
    if constexpr (S == 0) { C[g * F::N + 2 * q] = c[0]; C[g * F::N + 2 * q + 1] = c[1]; }
    else for (int i = 0; i < 4; ++i) C[(g + 8 * (i >> 1)) * F::N + 2 * q + (i & 1)] = c[i];
}

// ---- throughput: every warp runs NACC independent accumulator chains, ITER times
template <int S, int NACC>
__global__ void __launch_bounds__(256) k_tput(double* out, int iters) {
    using F = Frag<S>;
    double a[8], b[4], c[NACC][4];
    for (int i = 0; i < 8; ++i) a[i] = 1e-3 * (threadIdx.x + i);
    for (int i = 0; i < 4; ++i) b[i] = 1e-3 * (threadIdx.x - i);
    for (int x = 0; x < NACC; ++x) for (int i = 0; i < 4; ++i) c[x][i] = 0.0;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int x = 0; x < NACC; ++x) mma<S>(c[x], a, b);
    }
    double s = 0;
    for (int x = 0; x < NACC; ++x) for (int i = 0; i < F::NC; ++i) s += c[x][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int S>
void run(int sms) {
    using F = Frag<S>;
    // layout check
    double hA[16 * 16], hB[16 * 8], hC[16 * 8], ref[16 * 8];
    for (int i = 0; i < F::M * F::K; ++i) hA[i] = (double)(rand() % 17 - 8);
    for (int i = 0; i < F::K * F::N; ++i) hB[i] = (double)(rand() % 13 - 6);
    for (int i = 0; i < F::M; ++i) for (int j = 0; j < F::N; ++j) { double s = 0; for (int k = 0; k < F::K; ++k) s += hA[i * F::K + k] * hB[k * F::N + j]; ref[i * F::N + j] = s; }
    double *dA, *dB, *dC; cudaMalloc(&dA, sizeof hA); cudaMalloc(&dB, sizeof hB); cudaMalloc(&dC, sizeof hC);
    cudaMemcpy(dA, hA, sizeof hA, cudaMemcpyHostToDevice); cudaMemcpy(dB, hB, sizeof hB, cudaMemcpyHostToDevice);
    k_check<S><<<1, 32>>>(dA, dB, dC); cudaMemcpy(hC, dC, sizeof hC, cudaMemcpyDeviceToHost);
    int bad = 0; for (int i = 0; i < F::M * F::N; ++i) bad += (hC[i] != ref[i]);
    // throughput, 2 CTAs of 8 warps per SM
    double* out; cudaMalloc(&out, (size_t)sms * 4 * 256 * 8);
    const int iters = 4000; constexpr int NACC = 8;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int ctas_per_sm = 1; ctas_per_sm <= 4; ctas_per_sm *= 2) {
        k_tput<S, NACC><<<sms * ctas_per_sm, 256>>>(out, 100);
        cudaEventRecord(e0); k_tput<S, NACC><<<sms * ctas_per_sm, 256>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        const double flops = 2.0 * F::M * F::N * F::K * NACC * (double)iters * 8 * sms * ctas_per_sm;
        printf("m%dn%dk%-2d layout_mismatches=%d  %d warps/SM: %.2f TFLOP/s\n", F::M, F::N, F::K, bad, 8 * ctas_per_sm, flops / (ms * 1e-3) / 1e12);
    }
    cudaError_t e = cudaGetLastError(); if (e != cudaSuccess) printf("cuda error %s\n", cudaGetErrorString(e));
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    printf("%s, %d SMs\n", p.name, p.multiProcessorCount);
    run<0>(p.multiProcessorCount); run<1>(p.multiProcessorCount); run<2>(p.multiProcessorCount); run<3>(p.multiProcessorCount);
    return 0;
}
