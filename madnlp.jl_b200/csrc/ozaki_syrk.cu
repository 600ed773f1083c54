// b2d_condensed_assemble_ozaki: build_kkt!(::DenseCondensedKKTSystem) (src/KKT/Dense/condensed.jl:157-186) with the J' D J
// contraction on the Hopper tensor cores (wgmma.mma_async s8 x s8 -> s32 + TMA) through the Ozaki digit scheme of
// ozaki_kernels.cuh, instead of the reference's cuBLAS mul!(W, jac_ineq', jac_ineq) (Dense/condensed.jl:171) / the DMMA SYRK of
// assembly.cu.  Same outputs: lower triangle of aug[0:n, 0:n] = J_I' D J_I + H + diag(pr[0:n]), then the equality rows.
#include <cudaTypedefs.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "ozaki_kernels.cuh"

using namespace b2;

struct b2d_ozaki_plan {
    int32_t n = 0, ns = 0, Kpad = 0, Mpad = 0, ntiles = 0;
    DevBuf<int8_t> Q;          // [S][Mpad][Kpad] digit planes (padding stays zero)
    DevBuf<int32_t> expo, err;
    DevBuf<int2> tiles;
    CUtensorMap mapQ;          // box (64 B of K, 64 rows, 8 digits): A and B tiles alike
};

extern "C" int b2d_condensed_assemble(int32_t n, int32_t m, int32_t ns, int32_t n_eq, const int64_t* ind_ineq_d, const int64_t* ind_eq_d,
                                      const double* hess_d, const double* jac_d, const double* pr_diag_d, const double* du_diag_d,
                                      double* diag_buffer_d, double* aug_d, void* stream);
// (internal, assembly.cu) diag_buffer + equality rows without the SYRK
int b2d_assemble_parts(int32_t n, int32_t m, int32_t ns, int32_t n_eq, const int64_t* ind_ineq_d, const int64_t* ind_eq_d,
                       const double* jac_d, const double* pr_diag_d, const double* du_diag_d, double* diag_buffer_d, double* aug_d,
                       bool before_syrk, cudaStream_t st);

static bool make_map(CUtensorMap* out, const int8_t* Q, int Kpad, int Mpad) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) { cudaGetLastError(); return false; }
    auto enc = (PFN_cuTensorMapEncodeTiled_v12000)fn;
    cuuint64_t dims[3] = {(cuuint64_t)Kpad, (cuuint64_t)Mpad, (cuuint64_t)ozk::S};
    cuuint64_t strides[2] = {(cuuint64_t)Kpad, (cuuint64_t)Kpad * Mpad};
    cuuint32_t box[3] = {(cuuint32_t)ozk::BKB, (cuuint32_t)ozk::BM, (cuuint32_t)ozk::S};
    cuuint32_t estr[3] = {1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)Q, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

extern "C" int b2d_ozaki_plan_create(int32_t n, int32_t ns, b2d_ozaki_plan** out) {
    if (!out || n <= 0 || ns <= 0) { set_error("b2d_ozaki_plan_create: invalid argument"); return B2_ERR_INVALID; }
    if (ns > 16384) { set_error("b2d_ozaki_plan_create: ns > 16384 would overflow the int32 accumulators"); return B2_ERR_INVALID; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); set_error("b2d_ozaki_plan_create: no CUDA device"); return B2_ERR_NO_DEVICE; }
    auto* p = new b2d_ozaki_plan();
    p->n = n; p->ns = ns;
    p->Kpad = (ns + ozk::BKB - 1) / ozk::BKB * ozk::BKB;
    p->Mpad = (n + ozk::BM - 1) / ozk::BM * ozk::BM;
    std::vector<int2> tiles;
    for (int bm = 0; bm < p->Mpad / ozk::BM; ++bm)
        for (int bn = 0; bn <= bm; ++bn) tiles.push_back(make_int2(bm, bn));
    p->ntiles = (int32_t)tiles.size();
    if (p->Q.alloc((size_t)ozk::S * p->Mpad * p->Kpad) != cudaSuccess || p->expo.alloc(p->Mpad) != cudaSuccess || p->err.alloc(1) != cudaSuccess ||
        p->tiles.upload(tiles.data(), tiles.size()) != cudaSuccess || cudaMemset(p->Q.p, 0, p->Q.bytes()) != cudaSuccess ||
        cudaMemset(p->expo.p, 0, p->expo.bytes()) != cudaSuccess || cudaMemset(p->err.p, 0, sizeof(int32_t)) != cudaSuccess) {
        delete p;
        return cuda_fail(cudaGetLastError(), "b2d_ozaki_plan_create alloc", __FILE__, __LINE__);
    }
    if (!make_map(&p->mapQ, p->Q.p, p->Kpad, p->Mpad) ||
        cudaFuncSetAttribute(ozk::k_ozaki_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, ozk::SMEM_BYTES) != cudaSuccess) {
        delete p;
        set_error("b2d_ozaki_plan_create: tensor map / kernel attribute setup failed");
        return B2_ERR_CUDA;
    }
    *out = p;
    return B2_OK;
}
extern "C" int b2d_ozaki_plan_destroy(b2d_ozaki_plan* p) { delete p; return B2_OK; }

extern "C" int b2d_condensed_assemble_ozaki(b2d_ozaki_plan* p, int32_t n, int32_t m, int32_t ns, int32_t n_eq, const int64_t* ind_ineq_d,
                                            const int64_t* ind_eq_d, const double* hess_d, const double* jac_d, const double* pr_diag_d,
                                            const double* du_diag_d, double* diag_buffer_d, double* aug_d, void* stream) {
    if (!p || p->n != n || p->ns != ns || m != ns + n_eq || !hess_d || !jac_d || !pr_diag_d || !aug_d || !diag_buffer_d || !ind_ineq_d) {
        set_error("b2d_condensed_assemble_ozaki: invalid argument");
        return B2_ERR_INVALID;
    }
    cudaStream_t st = as_stream(stream);
    const int N = n + n_eq;
    int rc = b2d_assemble_parts(n, m, ns, n_eq, ind_ineq_d, ind_eq_d, jac_d, pr_diag_d, du_diag_d, diag_buffer_d, aug_d, true, st);   // D
    if (rc != B2_OK) return rc;
    // digits of A = sqrt(D) .* jac[ind_ineq, :]  (one CTA per column of A = per variable)
    ozk::k_ozaki_split<<<n, 256, 0, st>>>(ns, p->Kpad, p->Mpad, jac_d, (int64_t)m, ind_ineq_d, diag_buffer_d, p->Q.p, p->expo.p);
    ozk::k_ozaki_syrk<<<p->ntiles, ozk::NTHREADS, ozk::SMEM_BYTES, st>>>(p->mapQ, p->Kpad, n, p->tiles.p, p->expo.p, aug_d, (int64_t)N, hess_d,
                                                                         (int64_t)n, pr_diag_d, 1, p->err.p);
    B2_CUDA(cudaGetLastError());
    return b2d_assemble_parts(n, m, ns, n_eq, ind_ineq_d, ind_eq_d, jac_d, pr_diag_d, du_diag_d, diag_buffer_d, aug_d, false, st);     // eq rows
}

// 1 if a pipeline wait of the tensor-core kernel ever timed out on this plan (bounded waits never hang; results are then invalid)
extern "C" int b2d_ozaki_plan_status(b2d_ozaki_plan* p, int32_t* timed_out, void* stream) {
    if (!p || !timed_out) return B2_ERR_INVALID;
    B2_CUDA(cudaMemcpyAsync(timed_out, p->err.p, sizeof(int32_t), cudaMemcpyDeviceToHost, as_stream(stream)));
    B2_CUDA(cudaStreamSynchronize(as_stream(stream)));
    return B2_OK;
}
