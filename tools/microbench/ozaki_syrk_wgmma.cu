// Micro-benchmark SURVEY.md section 7 asked for: the fp64 SYRK of BASELINE.json configs[1] (W = A' A, A = sqrt(D) .* J_ineq,
// K = ns = 2048 rows, n = 4096 columns) on the Hopper tensor cores.  wgmma has no fp64 kind, so fp64 is SLICED onto
// wgmma.mma_async s8 x s8 -> s32 (Ozaki scheme, int8 variant -- Ootomo/Ozaki/Yokota, "DGEMM on integer matrix multiplication unit", 2024):
//
//   1. per column m:  e_m = exponent of max_i |a_im|;  x = a_im * 2^-e_m in (-1, 1) is cut into S = 8 signed 7-bit digits
//      x = sum_s q_s 2^(-7(s+1))   (q_s int8, exact: 56 bits cover the fp64 mantissa of the column's largest entries)
//   2. G_d = sum_{s+t=d} Q_s' Q_t  for d = 0..S-1 : 36 EXACT int8 x int8 -> int32 GEMMs (|G_d| <= 8 * 2048 * 127^2 < 2^31),
//      the d-sums accumulate inside the wgmma register accumulators
//   3. W(m,n) = 2^(e_m + e_n - 14) * sum_d 2^(-7d) G_d(m,n)   evaluated in fp64 (Horner) by the epilogue
//
// Kernel (one 64 x 64 output tile per CTA, lower triangle only, 288 threads): see csrc/ozaki_kernels.cuh.
// Reported: max error relative to max|W| against cuBLAS DGEMM (parity gate 1e-13), time of the digit split and of the GEMM,
// int8 TOP/s, fp64-equivalent TFLOP/s, next to cuBLAS DGEMM/DSYRK on the same matrix.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o ozaki_syrk_wgmma ozaki_syrk_wgmma.cu -lcublas   (kernels: csrc/ozaki_kernels.cuh)
#include <cublas_v2.h>
#include <cudaTypedefs.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../../madnlp.jl_b200/csrc/ozaki_kernels.cuh"     // the kernels are the product's (b2d_condensed_assemble_ozaki)
using namespace ozk;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("{\"error\": \"%s at %s:%d\"}\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

// ------------------------------------------------------------------------------------------------ host
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    return (PFN_cuTensorMapEncodeTiled_v12000)fn;
}

static CUtensorMap make_map(PFN_cuTensorMapEncodeTiled_v12000 enc, const int8_t* Q, int K, int M) {
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)M, (cuuint64_t)S};
    cuuint64_t strides[2] = {(cuuint64_t)K, (cuuint64_t)K * M};        // bytes, dims 1 and 2
    cuuint32_t box[3] = {(cuuint32_t)BKB, (cuuint32_t)BM, (cuuint32_t)S};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)Q, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("{\"error\": \"cuTensorMapEncodeTiled failed: %d\"}\n", (int)r); exit(1); }
    return m;
}

int main(int argc, char** argv) {
    const int K = argc > 1 ? atoi(argv[1]) : 2048, M = argc > 2 ? atoi(argv[2]) : 4096;
    const int reps = argc > 3 ? atoi(argv[3]) : 10;
    if (K % BKB || M % BM) { printf("{\"error\": \"K must be a multiple of %d and M of %d\"}\n", BKB, BM); return 1; }
    // A = sqrt(D) .* J:  J ~ N(0,1)/sqrt(M),  D log-uniform in [1e-8, 1e8] per ROW (the contraction index) -- SURVEY 8d C2
    std::vector<double> hA((size_t)K * M);
    {
        std::mt19937_64 rng(1);
        std::normal_distribution<double> nd(0.0, 1.0);
        std::uniform_real_distribution<double> ud(-8.0, 8.0);
        std::vector<double> sd(K);
        for (int i = 0; i < K; ++i) sd[i] = sqrt(pow(10.0, ud(rng)));
        for (int m = 0; m < M; ++m)
            for (int i = 0; i < K; ++i) hA[(size_t)m * K + i] = sd[i] * nd(rng) / sqrt((double)M);
    }
    double *dA, *dC, *dRef;
    int8_t* dQ;
    int *dE, *dErr;
    CK(cudaMalloc(&dA, sizeof(double) * K * M));
    CK(cudaMalloc(&dC, sizeof(double) * M * M));
    CK(cudaMalloc(&dRef, sizeof(double) * M * M));
    CK(cudaMalloc(&dQ, (size_t)S * M * K));
    CK(cudaMalloc(&dE, sizeof(int) * M));
    CK(cudaMalloc(&dErr, sizeof(int)));
    CK(cudaMemset(dErr, 0, sizeof(int)));
    CK(cudaMemset(dC, 0, sizeof(double) * M * M));
    CK(cudaMemcpy(dA, hA.data(), sizeof(double) * K * M, cudaMemcpyHostToDevice));
    std::vector<int2> tiles;
    for (int bm = 0; bm < M / BM; ++bm)
        for (int bn = 0; bn <= bm; ++bn) tiles.push_back(make_int2(bm, bn));
    int2* dT;
    CK(cudaMalloc(&dT, sizeof(int2) * tiles.size()));
    CK(cudaMemcpy(dT, tiles.data(), sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice));
    auto enc = get_encode();
    CUtensorMap mapQ = make_map(enc, dQ, K, M);
    CK(cudaFuncSetAttribute(k_ozaki_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));

    cudaEvent_t e0, e1, e2;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    float ms_split = 1e30f, ms_gemm = 1e30f;
    for (int r = 0; r < reps + 2; ++r) {
        CK(cudaEventRecord(e0));
        k_ozaki_split<<<M, 256>>>(K, K, M, dA, (int64_t)K, nullptr, nullptr, dQ, dE);
        CK(cudaEventRecord(e1));
        k_ozaki_syrk<<<(int)tiles.size(), NTHREADS, SMEM_BYTES>>>(mapQ, K, M, dT, dE, dC, (int64_t)M, nullptr, 0, nullptr, 0, dErr);
        CK(cudaEventRecord(e2));
        CK(cudaEventSynchronize(e2));
        CK(cudaGetLastError());
        float a, b;
        CK(cudaEventElapsedTime(&a, e0, e1)); CK(cudaEventElapsedTime(&b, e1, e2));
        if (r >= 2) { ms_split = fminf(ms_split, a); ms_gemm = fminf(ms_gemm, b); }
    }
    int herr = 0;
    CK(cudaMemcpy(&herr, dErr, sizeof(int), cudaMemcpyDeviceToHost));
    // reference + library bars: cuBLAS DGEMM (what the reference calls, Dense/condensed.jl:171) and DSYRK
    cublasHandle_t hb;
    cublasCreate(&hb);
    const double one = 1.0, zero = 0.0;
    float ms_dgemm = 1e30f, ms_dsyrk = 1e30f;
    for (int r = 0; r < 4; ++r) {
        CK(cudaEventRecord(e0));
        cublasDgemm(hb, CUBLAS_OP_T, CUBLAS_OP_N, M, M, K, &one, dA, K, dA, K, &zero, dRef, M);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float a; CK(cudaEventElapsedTime(&a, e0, e1));
        if (r) ms_dgemm = fminf(ms_dgemm, a);
    }
    {
        double* dTmp;
        CK(cudaMalloc(&dTmp, sizeof(double) * M * M));
        for (int r = 0; r < 4; ++r) {
            CK(cudaEventRecord(e0));
            cublasDsyrk(hb, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_T, M, K, &one, dA, K, &zero, dTmp, M);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float a; CK(cudaEventElapsedTime(&a, e0, e1));
            if (r) ms_dsyrk = fminf(ms_dsyrk, a);
        }
        cudaFree(dTmp);
    }
    std::vector<double> hC((size_t)M * M), hR((size_t)M * M);
    CK(cudaMemcpy(hC.data(), dC, sizeof(double) * M * M, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hR.data(), dRef, sizeof(double) * M * M, cudaMemcpyDeviceToHost));
    double maxabs = 0.0, maxerr = 0.0;
    for (int n = 0; n < M; ++n)
        for (int m = n; m < M; ++m) {
            const double r = hR[(size_t)n * M + m];
            maxabs = fmax(maxabs, fabs(r));
            maxerr = fmax(maxerr, fabs(hC[(size_t)n * M + m] - r));
        }
    // exactness of the integer part on a sample: recompute W(m,n) from the fp64 definition in long double
    double maxerr_ld = 0.0;
    for (int q = 0; q < 64; ++q) {
        const int m = (q * 977 + 13) % M, n = (q * 131) % (m + 1);
        long double acc = 0.0L;
        for (int i = 0; i < K; ++i) acc += (long double)hA[(size_t)m * K + i] * (long double)hA[(size_t)n * K + i];
        maxerr_ld = fmax(maxerr_ld, fabs((double)(acc - (long double)hC[(size_t)n * M + m])));
    }
    const double flop = (double)M * (M + 1) * K;                                  // SYRK, lower triangle
    const double tile_ops = (double)tiles.size() * BM * BN * (double)K * 2.0 * (S * (S + 1) / 2);
    printf("{\"bench\": \"ozaki_int8_syrk_wgmma\", \"K\": %d, \"n\": %d, \"digits\": %d, \"bits_per_digit\": %d, \"int8_gemms\": %d, "
           "\"tile\": \"%dx%d, K block %d, %d stages\", \"tiles\": %d, \"err_flag\": %d, "
           "\"max_abs_err_vs_cublas_dgemm\": %.3e, \"max_abs_W\": %.3e, \"rel_err\": %.3e, \"rel_err_vs_long_double_sample\": %.3e, \"parity_gate_1e-13\": %s, "
           "\"ms_split\": %.4f, \"ms_gemm\": %.4f, \"ms_total\": %.4f, \"int8_tops\": %.1f, \"fp64_equiv_tflops\": %.2f, "
           "\"cublas_dgemm_ms\": %.4f, \"cublas_dsyrk_ms\": %.4f, \"cublas_dsyrk_tflops\": %.2f}\n",
           K, M, S, WB, S * (S + 1) / 2, BM, BN, BKB, STAGES, (int)tiles.size(), herr, maxerr, maxabs, maxerr / maxabs, maxerr_ld / maxabs,
           (maxerr / maxabs <= 1e-13 && herr == 0) ? "true" : "false", ms_split, ms_gemm, ms_split + ms_gemm, tile_ops / (ms_gemm * 1e-3) / 1e12,
           flop / ((ms_split + ms_gemm) * 1e-3) / 1e12, ms_dgemm, ms_dsyrk, flop / (ms_dsyrk * 1e-3) / 1e12);
    return 0;
}
