// KKT assembly kernels and their one-time symbolic plans (C-ABI in include/b200kkt.h).
//   b2_coo_to_csc / b2_transfer*    -- src/matrixtools.jl:55-95, kernels_sparse.jl:161-167 (rows A3/A4/A5 of SURVEY 8a)
//   b2_condensed_*                  -- src/KKT/Sparse/condensed.jl:201-366, gpu_sparse.jl:308-340 (rows A6/A7)
//   b2d_condensed_assemble          -- src/KKT/Dense/condensed.jl:120-186, kernels_dense.jl:81-119 (row A8)
//   b2d_aug_assemble, b2d_copy_diag -- src/KKT/Dense/augmented.jl:116-161, kernels_dense.jl:39-75
// All sparse kernels are "one thread per destination slot" gathers: race-free, no atomics, and the per-slot
// summation order equals the reference's sequential CPU loops, so results are bit-identical to them
// (adds and multiplies are issued with explicit rounding intrinsics so the compiler cannot contract them to FMA).
#include <algorithm>
#include <cstring>
#include <numeric>
#include <stdexcept>
#include <vector>

#include "common.cuh"
#include "condensed_plan.cuh"

using namespace b2;

// ---------------------------------------------------------------------------------------------------------
// COO -> CSC pattern + map (host, one-time)
// ---------------------------------------------------------------------------------------------------------
extern "C" int b2_coo_to_csc(int32_t m, int32_t n, int64_t nnz_coo, const int32_t* I_h, const int32_t* J_h,
                             int32_t* colptr_h, int32_t* rowval_h, int64_t* map_h, int64_t* nnz_csc) {
    if (m < 0 || n < 0 || nnz_coo < 0 || (nnz_coo && (!I_h || !J_h)) || !colptr_h || !rowval_h || !map_h) {
        set_error("b2_coo_to_csc: invalid argument");
        return B2_ERR_INVALID;
    }
    std::vector<int64_t> order(nnz_coo);
    std::iota(order.begin(), order.end(), (int64_t)0);
    for (int64_t k = 0; k < nnz_coo; ++k)
        if (I_h[k] < 0 || I_h[k] >= m || J_h[k] < 0 || J_h[k] >= n) { set_error("b2_coo_to_csc: index out of range"); return B2_ERR_INVALID; }
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
        if (J_h[a] != J_h[b]) return J_h[a] < J_h[b];
        return I_h[a] < I_h[b];
    });
    std::fill(colptr_h, colptr_h + n + 1, 0);
    int64_t slot = -1;
    int32_t li = -1, lj = -1;
    for (int64_t q = 0; q < nnz_coo; ++q) {
        const int64_t k = order[q];
        if (I_h[k] != li || J_h[k] != lj) {
            ++slot;
            li = I_h[k]; lj = J_h[k];
            rowval_h[slot] = li;
            colptr_h[lj + 1]++;
        }
        map_h[k] = slot;
    }
    for (int32_t j = 0; j < n; ++j) colptr_h[j + 1] += colptr_h[j];
    if (nnz_csc) *nnz_csc = slot + 1;
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// transfer!:  dst .= 0; dst[map[k]] += V[k]
// ---------------------------------------------------------------------------------------------------------
struct b2_transfer_plan {
    int64_t nnz_coo = 0, nnz_csc = 0;
    DevBuf<int32_t> ptr;   // [nnz_csc+1]
    DevBuf<int32_t> src;   // [nnz_coo] COO positions grouped by destination, ascending inside a group
};

__global__ void k_transfer(int64_t nslot, const int32_t* __restrict__ ptr, const int32_t* __restrict__ src,
                           const double* __restrict__ V, double* __restrict__ dst) {
    pdl_sync();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nslot; i += (int64_t)gridDim.x * blockDim.x) {
        const int a = ptr[i], b = ptr[i + 1];
        double acc = 0.0;
        for (int q = a; q < b; ++q) acc = __dadd_rn(acc, V[src[q]]);
        dst[i] = acc;
    }
}

extern "C" int b2_transfer_plan_create(int64_t nnz_coo, int64_t nnz_csc, const int64_t* map_h, b2_transfer_plan** out) {
    if (!out || nnz_coo < 0 || nnz_csc < 0 || (nnz_coo && !map_h) || nnz_coo >= (int64_t)1 << 31) {
        set_error("b2_transfer_plan_create: invalid argument");
        return B2_ERR_INVALID;
    }
    std::vector<int32_t> ptr(nnz_csc + 1, 0), src(nnz_coo);
    for (int64_t k = 0; k < nnz_coo; ++k) {
        if (map_h[k] < 0 || map_h[k] >= nnz_csc) { set_error("b2_transfer_plan_create: map out of range"); return B2_ERR_INVALID; }
        ptr[map_h[k] + 1]++;
    }
    for (int64_t i = 0; i < nnz_csc; ++i) ptr[i + 1] += ptr[i];
    std::vector<int32_t> pos(ptr.begin(), ptr.end() - 1);
    for (int64_t k = 0; k < nnz_coo; ++k) src[pos[map_h[k]]++] = (int32_t)k;   // ascending k inside each slot
    auto* p = new b2_transfer_plan();
    p->nnz_coo = nnz_coo; p->nnz_csc = nnz_csc;
    if (p->ptr.upload(ptr.data(), ptr.size()) != cudaSuccess || p->src.upload(src.data(), src.size()) != cudaSuccess) {
        delete p;
        return cuda_fail(cudaGetLastError(), "transfer plan upload", __FILE__, __LINE__);
    }
    *out = p;
    return B2_OK;
}

extern "C" int b2_transfer_plan_destroy(b2_transfer_plan* p) { delete p; return B2_OK; }

extern "C" int b2_transfer(b2_transfer_plan* p, double* dst_nz_d, const double* V_d, void* stream) {
    if (!p || (p->nnz_csc && (!dst_nz_d || !V_d))) { set_error("b2_transfer: invalid argument"); return B2_ERR_INVALID; }   // empty: may be null
    if (p->nnz_csc == 0) return B2_OK;
    const int grid = (int)std::min<int64_t>((p->nnz_csc + 255) / 256, 8 * sm_count());
    launch_pdl(k_transfer, dim3(grid), dim3(256), 0, as_stream(stream), p->nnz_csc, p->ptr.p, p->src.p, V_d, dst_nz_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// build_kkt!(::ScaledSparseKKTSystem) (scaled_augmented.jl:209-236): transfer! of V with every COO source scaled first, in one pass
// over the CSC slots of aug_com and in b2_transfer's summation order.  A slot at (row r, column c) of the lower triangle takes
//   c >= n_tot (du_diag)  : v            r >= n_tot (Jacobian, slack) : v * s[c]
//   r, c < n_tot          : v for a pr_diag source (COO index k < n_tot), (v * s[r]) * s[c] for a Hessian source
// so a diagonal slot that sums pr_diag and Hessian sources scales each on its own.  The column of a slot comes from colptr: the
// CTA finds the columns of its first and last slot, each thread bisects between them (a few steps: a CTA spans few columns).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t slot_column(const int32_t* __restrict__ colptr, int64_t lo, int64_t hi, int64_t slot) {
    while (lo < hi) {                                  // the last column c in [lo, hi] with colptr[c] <= slot
        const int64_t mid = (lo + hi + 1) >> 1;
        if (colptr[mid] <= slot) lo = mid; else hi = mid - 1;
    }
    return lo;
}
__global__ void k_scaled_transfer(int64_t nslot, int64_t ncol, int64_t n_tot, const int32_t* __restrict__ ptr, const int32_t* __restrict__ src,
                                  const int32_t* __restrict__ colptr, const int32_t* __restrict__ rowval, const double* __restrict__ sf,
                                  const double* __restrict__ V, double* __restrict__ dst) {
    __shared__ int64_t cspan[2];
    pdl_sync();
    const int64_t s0 = (int64_t)blockIdx.x * blockDim.x;
    if (threadIdx.x < 2) cspan[threadIdx.x] = slot_column(colptr, 0, ncol - 1, threadIdx.x ? std::min<int64_t>(s0 + blockDim.x, nslot) - 1 : s0);
    __syncthreads();
    const int64_t i = s0 + threadIdx.x;
    if (i >= nslot) return;
    const int64_t c = slot_column(colptr, cspan[0], cspan[1], i);
    const int64_t r = rowval[i];
    const int a = ptr[i], b = ptr[i + 1];
    double acc = 0.0;
    if (c >= n_tot) {
        for (int q = a; q < b; ++q) acc = __dadd_rn(acc, V[src[q]]);
    } else if (r >= n_tot) {
        const double sc = sf[c];
        for (int q = a; q < b; ++q) acc = __dadd_rn(acc, __dmul_rn(V[src[q]], sc));
    } else {
        const double sr = sf[r], sc = sf[c];
        for (int q = a; q < b; ++q) {
            const int k = src[q];
            const double v = V[k];
            acc = __dadd_rn(acc, k < n_tot ? v : __dmul_rn(__dmul_rn(v, sr), sc));
        }
    }
    dst[i] = acc;
}

extern "C" int b2_scaled_transfer(b2_transfer_plan* p, int64_t n, int64_t n_tot, const int32_t* colptr_d, const int32_t* rowval_d,
                                  const double* scaling_d, double* dst_nz_d, const double* V_d, void* stream) {
    B2_NEED(p && n >= 0 && n_tot >= 0 && n_tot <= n && (p->nnz_csc == 0 || (n > 0 && colptr_d && rowval_d && dst_nz_d && V_d)),
            "b2_scaled_transfer");
    B2_NEED(n_tot == 0 || p->nnz_csc == 0 || scaling_d, "b2_scaled_transfer");
    if (p->nnz_csc == 0) return B2_OK;
    launch_pdl(k_scaled_transfer, dim3((unsigned)((p->nnz_csc + 255) / 256)), dim3(256), 0, as_stream(stream), p->nnz_csc, n, n_tot,
               p->ptr.p, p->src.p, colptr_d, rowval_d, scaling_d, V_d, dst_nz_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// sparse condensed KKT:  aug = tril(H) + diag(pr_diag[1:n]) + tril(Jt * D * Jt')
// ---------------------------------------------------------------------------------------------------------
__global__ void k_diag_buffer(int64_t m, const double* __restrict__ Ss, const double* __restrict__ Sd, double* __restrict__ D) {
    pdl_sync();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
        D[i] = __ddiv_rn(Ss[i], __dsub_rn(1.0, __dmul_rn(Sd[i], Ss[i])));
}

__global__ void k_condensed(int64_t nslot, const int32_t* __restrict__ hsrc, const int32_t* __restrict__ dsrc,
                            const int32_t* __restrict__ tptr, const int4* __restrict__ trip,
                            const double* __restrict__ Hnz, const double* __restrict__ pr, const double* __restrict__ D,
                            const double* __restrict__ Jt, double* __restrict__ nz) {
    pdl_sync();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nslot; i += (int64_t)gridDim.x * blockDim.x) {
        double acc = 0.0;
        const int h = hsrc[i], dd = dsrc[i];
        if (h >= 0) acc = __dadd_rn(acc, Hnz[h]);
        if (dd >= 0) acc = __dadd_rn(acc, pr[dd]);
        // triples in batches of 4: index records first, then the 12 values, then the adds in the reference's order
        // (latency-bound gather: a slot holds 0-12 triples)
        const int a = tptr[i], b = tptr[i + 1];
        for (int q0 = a; q0 < b; q0 += 4) {
            int4 t[4]; double dv[4], j1[4], j2[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) t[u] = (q0 + u < b) ? trip[q0 + u] : make_int4(-1, 0, 0, 0);
#pragma unroll
            for (int u = 0; u < 4; ++u) { const bool ok = t[u].x >= 0; dv[u] = ok ? D[t[u].x] : 0.0; j1[u] = ok ? Jt[t[u].y] : 0.0; j2[u] = ok ? Jt[t[u].z] : 0.0; }
#pragma unroll
            for (int u = 0; u < 4; ++u) if (t[u].x >= 0) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(dv[u], j1[u]), j2[u]));
        }
        nz[i] = acc;
    }
}

extern "C" int b2_condensed_symbolic(int32_t n, int32_t m, const int32_t* Hc, const int32_t* Hr,
                                     const int32_t* Jc, const int32_t* Jr, b2_condensed_plan** out, int64_t* nnz_aug) {
    if (!out || n <= 0 || m < 0 || !Hc || !Jc) { set_error("b2_condensed_symbolic: invalid argument"); return B2_ERR_INVALID; }
    struct Ent { int32_t col, row, kind, s1, s2; };   // kind: -1 diag, 0 hess, >0: Jt column + 1
    const int64_t nnzH = Hc[n];
    int64_t nj = 0;
    for (int32_t i = 0; i < m; ++i) { const int64_t c = Jc[i + 1] - Jc[i]; nj += c * (c + 1) / 2; }
    std::vector<Ent> e;
    e.reserve((size_t)(n + nnzH + nj));
    for (int32_t i = 0; i < n; ++i) e.push_back({i, i, -1, i, 0});
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = Hc[j]; p < Hc[j + 1]; ++p) e.push_back({j, Hr[p], 0, p, 0});
    for (int32_t i = 0; i < m; ++i)
        for (int32_t j = Jc[i]; j < Jc[i + 1]; ++j)
            for (int32_t k = j; k < Jc[i + 1]; ++k) e.push_back({Jr[j], Jr[k], i + 1, j, k});   // (c1=Jr[j] col, c2=Jr[k] row)
    // stable sort by (col,row): preserves the reference's enumeration order inside a slot (condensed.jl:251)
    std::stable_sort(e.begin(), e.end(), [](const Ent& a, const Ent& b) {
        if (a.col != b.col) return a.col < b.col;
        return a.row < b.row;
    });
    auto* p = new b2_condensed_plan();
    p->n = n; p->m = m;
    p->colptr.assign(n + 1, 0);
    std::vector<int32_t> hsrc, dsrc, tptr;
    std::vector<int4> trip;
    trip.reserve(nj);
    int32_t lc = -1, lr = -1;
    for (const Ent& x : e) {
        if (x.row < x.col) { delete p; set_error("b2_condensed_symbolic: entry above the diagonal (H must be lower, Jt rows sorted)"); return B2_ERR_INVALID; }
        if (x.col != lc || x.row != lr) {
            lc = x.col; lr = x.row;
            p->rowval.push_back(x.row);
            p->colptr[x.col + 1]++;
            hsrc.push_back(-1); dsrc.push_back(-1);
            tptr.push_back((int32_t)trip.size());
        }
        if (x.kind == -1) { dsrc.back() = x.s1; p->n_dptr++; }
        else if (x.kind == 0) {
            if (hsrc.back() >= 0) { delete p; set_error("b2_condensed_symbolic: duplicate entry in H"); return B2_ERR_INVALID; }
            hsrc.back() = x.s1; p->n_hptr++;
        } else { trip.push_back(make_int4(x.kind - 1, x.s1, x.s2, 0)); p->n_jptr++; }
    }
    tptr.push_back((int32_t)trip.size());
    for (int32_t j = 0; j < n; ++j) p->colptr[j + 1] += p->colptr[j];
    p->nnz_aug = (int64_t)p->rowval.size();
    if (trip.empty()) trip.push_back(make_int4(0, 0, 0, 0));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0) {
        if (p->hsrc.upload(hsrc.data(), hsrc.size()) != cudaSuccess || p->dsrc.upload(dsrc.data(), dsrc.size()) != cudaSuccess ||
            p->tptr.upload(tptr.data(), tptr.size()) != cudaSuccess || p->trip.upload(trip.data(), trip.size()) != cudaSuccess) {
            delete p;
            return cuda_fail(cudaGetLastError(), "condensed plan upload", __FILE__, __LINE__);
        }
    } else {
        cudaGetLastError();   // pattern-only plan (host tooling); b2_condensed_assemble will refuse to run
    }
    *out = p;
    if (nnz_aug) *nnz_aug = p->nnz_aug;
    return B2_OK;
}

extern "C" int b2_condensed_pattern(b2_condensed_plan* p, int32_t* colptr_h, int32_t* rowval_h) {
    if (!p || !colptr_h || !rowval_h) return B2_ERR_INVALID;
    std::memcpy(colptr_h, p->colptr.data(), p->colptr.size() * sizeof(int32_t));
    std::memcpy(rowval_h, p->rowval.data(), p->rowval.size() * sizeof(int32_t));
    return B2_OK;
}

extern "C" int b2_condensed_plan_sizes(b2_condensed_plan* p, int64_t* n_dptr, int64_t* n_hptr, int64_t* n_jptr) {
    if (!p) return B2_ERR_INVALID;
    if (n_dptr) *n_dptr = p->n_dptr;
    if (n_hptr) *n_hptr = p->n_hptr;
    if (n_jptr) *n_jptr = p->n_jptr;
    return B2_OK;
}

extern "C" int b2_condensed_plan_destroy(b2_condensed_plan* p) { delete p; return B2_OK; }

extern "C" int b2_condensed_assemble(b2_condensed_plan* p, double* aug_nz_d, const double* pr_diag_d, const double* du_diag_d,
                                     const double* H_nz_d, const double* Jt_nz_d, double* diag_buffer_d, void* stream) {
    if (!p || !aug_nz_d || !pr_diag_d || (p->m && (!du_diag_d || !diag_buffer_d))) {   // m = 0: empty du_diag and diag_buffer may be null
        set_error("b2_condensed_assemble: invalid argument");
        return B2_ERR_INVALID;
    }
    if (!p->hsrc.p) { set_error("b2_condensed_assemble: plan has no device state (no CUDA device at creation)"); return B2_ERR_NO_DEVICE; }
    cudaStream_t st = as_stream(stream);
    if (p->m > 0) {
        const int g = (int)std::min<int64_t>((p->m + 255) / 256, 8 * sm_count());
        launch_pdl(k_diag_buffer, dim3(g), dim3(256), 0, st, p->m, pr_diag_d + p->n, du_diag_d, diag_buffer_d);
    }
    const int grid = (int)std::min<int64_t>((p->nnz_aug + 255) / 256, 8 * sm_count());
    launch_pdl(k_condensed, dim3(grid), dim3(256), 0, st, p->nnz_aug, p->hsrc.p, p->dsrc.p, p->tptr.p, p->trip.p, H_nz_d, pr_diag_d, diag_buffer_d,
                                      Jt_nz_d, aug_nz_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// dense condensed KKT (lower triangle):  aug[0:n,0:n] = J_I' D J_I + H + diag(pr[0:n]);  equality rows/diag below.
// The SYRK runs on the fp64 tensor pipe (mma.sync m16n8k4 -> DMMA; on H100 twice the issue rate of m8n8k4, measured with
// tools/microbench/dmma_shapes.cu): 128x64 tile per 256-thread CTA, k-chunks of 16
// double-buffered in shared memory; the sqrt(D) scaling of the reference's `jac_ineq` prologue kernel is folded into
// the B operand (D, not sqrt(D): one operand is scaled once), the +H +diag epilogue kernel into the store.
// ---------------------------------------------------------------------------------------------------------
constexpr int DT_M = 128, DT_N = 64, DT_K = 16;

__global__ void k_dense_diag_buffer(int64_t ns, const int64_t* __restrict__ ind_ineq, const double* __restrict__ Ss,
                                    const double* __restrict__ du, double* __restrict__ D) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += (int64_t)gridDim.x * blockDim.x)
        D[i] = Ss[i] / (1.0 - du[ind_ineq[i]] * Ss[i]);
}

__global__ void __launch_bounds__(256) k_dense_syrk(int n, int m, int ns, int N, const int64_t* __restrict__ ind_ineq,
                                                    const double* __restrict__ hess, const double* __restrict__ jac,
                                                    const double* __restrict__ pr, const double* __restrict__ D,
                                                    double* __restrict__ aug) {
    const int ti = blockIdx.x, tj = blockIdx.y;
    const int i0 = ti * DT_M, j0 = tj * DT_N;
    if (j0 > i0 + DT_M - 1) return;                       // tile entirely above the diagonal
    extern __shared__ double dsm[];
    typedef double (*ATile)[DT_K][DT_M + 4];
    typedef double (*BTile)[DT_K][DT_N + 4];
    ATile As = (ATile)dsm;
    BTile Bs = (BTile)(dsm + 2 * DT_K * (DT_M + 4));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int wi = (warp & 3) * 32, wj = (warp >> 2) * 32;   // 4x2 warps, each 32x32
    double c[4][4][2];
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 4; ++y) c[x][y][0] = c[x][y][1] = 0.0;
    const int nchunk = (ns + DT_K - 1) / DT_K;
    // loader mapping: k fastest (rows of J are contiguous in memory for a fixed column)
    const int lk = tid % DT_K, lc = tid / DT_K;            // 16 columns per pass
    double ra[DT_M / 16], rb[DT_N / 16];
    auto gload = [&](int ch) {
        const int k = ch * DT_K + lk;
        const bool kv = k < ns;
        const int64_t row = kv ? ind_ineq[k] : 0;
        const double dk = kv ? D[k] : 0.0;
#pragma unroll
        for (int cc = 0; cc < DT_M / 16; ++cc) {
            const int col = i0 + lc + 16 * cc;
            ra[cc] = (kv && col < n) ? jac[(size_t)col * m + row] : 0.0;
        }
#pragma unroll
        for (int cc = 0; cc < DT_N / 16; ++cc) {
            const int col = j0 + lc + 16 * cc;
            rb[cc] = (kv && col < n) ? dk * jac[(size_t)col * m + row] : 0.0;
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int cc = 0; cc < DT_M / 16; ++cc) As[buf][lk][lc + 16 * cc] = ra[cc];
#pragma unroll
        for (int cc = 0; cc < DT_N / 16; ++cc) Bs[buf][lk][lc + 16 * cc] = rb[cc];
    };
    if (nchunk > 0) { gload(0); sstore(0); }
    __syncthreads();
    for (int ch = 0; ch < nchunk; ++ch) {
        const int buf = ch & 1;
        if (ch + 1 < nchunk) gload(ch + 1);               // global loads in flight while the tensor pipe works
#pragma unroll
        for (int k0 = 0; k0 < DT_K; k0 += 4) {
            double af[4], bf[4];
#pragma unroll
            for (int x = 0; x < 4; ++x) af[x] = As[buf][k0 + q][wi + 8 * x + g];
#pragma unroll
            for (int y = 0; y < 4; ++y) bf[y] = Bs[buf][k0 + q][wj + 8 * y + g];
#pragma unroll
            for (int x = 0; x < 4; x += 2)                            // m16n8k4 = two m8n8k4 row blocks 8 apart sharing B
#pragma unroll
                for (int y = 0; y < 4; ++y)
                    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                                 : "+d"(c[x][y][0]), "+d"(c[x][y][1]), "+d"(c[x + 1][y][0]), "+d"(c[x + 1][y][1])
                                 : "d"(af[x]), "d"(af[x + 1]), "d"(bf[y]));
        }
        if (ch + 1 < nchunk) sstore(buf ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 4; ++y)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = i0 + wi + 8 * x + g;
                const int j = j0 + wj + 8 * y + 2 * q + e;
                if (i < n && j < n && i >= j) {
                    double v = c[x][y][e] + hess[(size_t)j * n + i];
                    if (i == j) v += pr[i];
                    aug[(size_t)j * N + i] = v;
                }
            }
}

// equality rows: aug[n+i, 0:n] = jac[ind_eq[i], :];  aug[n+i, n+j] = (i==j) ? du[ind_eq[i]] : 0  (j <= i)
__global__ void k_dense_eq_rows(int n, int m, int n_eq, int N, const int64_t* __restrict__ ind_eq,
                                const double* __restrict__ jac, const double* __restrict__ du, double* __restrict__ aug) {
    const int64_t total = (int64_t)n_eq * N;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(t % n_eq), j = (int)(t / n_eq);
        double v;
        if (j < n) v = jac[(size_t)j * m + ind_eq[i]];
        else {
            const int jj = j - n;
            if (jj > i) continue;
            v = (jj == i) ? du[ind_eq[i]] : 0.0;
        }
        aug[(size_t)j * N + n + i] = v;
    }
}

// the two cheap passes around the contraction: before_syrk -> diag_buffer D = Ss ./ (1 - Sd[ind_ineq] .* Ss); after -> equality rows
int b2d_assemble_parts(int32_t n, int32_t m, int32_t ns, int32_t n_eq, const int64_t* ind_ineq_d, const int64_t* ind_eq_d,
                       const double* jac_d, const double* pr_diag_d, const double* du_diag_d, double* diag_buffer_d, double* aug_d,
                       bool before_syrk, cudaStream_t st) {
    const int N = n + n_eq;
    if (before_syrk) {
        if (ns > 0) {
            const int g = std::min((ns + 255) / 256, 8 * sm_count());
            k_dense_diag_buffer<<<g, 256, 0, st>>>(ns, ind_ineq_d, pr_diag_d + n, du_diag_d, diag_buffer_d);
        }
    } else if (n_eq > 0) {
        const int64_t total = (int64_t)n_eq * N;
        const int g = (int)std::min<int64_t>((total + 255) / 256, 8 * sm_count());
        k_dense_eq_rows<<<g, 256, 0, st>>>(n, m, n_eq, N, ind_eq_d, jac_d, du_diag_d, aug_d);
    }
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_condensed_assemble(int32_t n, int32_t m, int32_t ns, int32_t n_eq, const int64_t* ind_ineq_d,
                                      const int64_t* ind_eq_d, const double* hess_d, const double* jac_d,
                                      const double* pr_diag_d, const double* du_diag_d, double* diag_buffer_d,
                                      double* aug_d, void* stream) {
    if (n <= 0 || m < 0 || ns < 0 || n_eq < 0 || ns + n_eq != m || !hess_d || !pr_diag_d || !aug_d || (m && !jac_d)) {
        set_error("b2d_condensed_assemble: invalid argument");
        return B2_ERR_INVALID;
    }
    cudaStream_t st = as_stream(stream);
    const int N = n + n_eq;
    int rc = b2d_assemble_parts(n, m, ns, n_eq, ind_ineq_d, ind_eq_d, jac_d, pr_diag_d, du_diag_d, diag_buffer_d, aug_d, true, st);
    if (rc != B2_OK) return rc;
    dim3 grid((n + DT_M - 1) / DT_M, (n + DT_N - 1) / DT_N);
    const size_t syrk_smem = (size_t)(2 * DT_K * (DT_M + 4) + 2 * DT_K * (DT_N + 4)) * sizeof(double);
    static bool attr_set = false;
    if (!attr_set) { B2_CUDA(cudaFuncSetAttribute(k_dense_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)syrk_smem)); attr_set = true; }
    k_dense_syrk<<<grid, 256, syrk_smem, st>>>(n, m, ns, N, ind_ineq_d, hess_d, jac_d, pr_diag_d, diag_buffer_d, aug_d);
    B2_CUDA(cudaGetLastError());
    return b2d_assemble_parts(n, m, ns, n_eq, ind_ineq_d, ind_eq_d, jac_d, pr_diag_d, du_diag_d, diag_buffer_d, aug_d, false, st);
}

// ---------------------------------------------------------------------------------------------------------
// dense augmented KKT (lower triangle), N = n + ns + m:
//   [ H + diag(pr_diag[0:n]) (diagonal: pr_diag + diag_hess)                ]
//   [ 0                        diag(pr_diag[n:n+ns])                        ]
//   [ J                        -1 at (ind_ineq[k], k)        diag(du_diag)  ]
// Column j of aug below the diagonal is one contiguous run, and so are the sources that fill it (column j of hess and of
// jac), so one CTA sweeps one column: coalesced reads and writes, every lower element written once (zeros included),
// nothing above the diagonal touched.  Pure copy: the only arithmetic is the diagonal's single add, in the reference's order.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dense_aug(int n, int m, int ns, const int64_t* __restrict__ ind_ineq,
                                                   const double* __restrict__ hess, const double* __restrict__ jac,
                                                   const double* __restrict__ pr, const double* __restrict__ du,
                                                   const double* __restrict__ dh, double* __restrict__ aug) {
    const int64_t nns = (int64_t)n + ns, N = nns + m;
    const int64_t j = blockIdx.x;
    double* __restrict__ col = aug + j * N;
    if (j < n) {
        const double* __restrict__ hc = hess + j * n;
        const double* __restrict__ jc = jac + j * m;
#pragma unroll 4
        for (int64_t i = j + threadIdx.x; i < N; i += blockDim.x)
            col[i] = i < n ? (i == j ? __dadd_rn(pr[i], dh[i]) : hc[i]) : (i < nns ? 0.0 : jc[i - nns]);
    } else if (j < nns) {
        const int64_t r = nns + ind_ineq[j - n];             // row of the slack's -1
#pragma unroll 4
        for (int64_t i = j + threadIdx.x; i < N; i += blockDim.x)
            col[i] = i == j ? pr[j] : (i == r ? -1.0 : 0.0);
    } else {
#pragma unroll 4
        for (int64_t i = j + threadIdx.x; i < N; i += blockDim.x)
            col[i] = i == j ? du[j - nns] : 0.0;
    }
}

__global__ void k_copy_diag(int n, int lda, const double* __restrict__ A, double* __restrict__ d) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        d[i] = A[i * lda + i];
}

extern "C" int b2d_aug_assemble(int32_t n, int32_t m, int32_t ns, const int64_t* ind_ineq_d,
                                const double* hess_d, const double* jac_d, const double* pr_diag_d,
                                const double* du_diag_d, const double* diag_hess_d, double* aug_d, void* stream) {
    const int64_t N = (int64_t)n + ns + m;
    if (n <= 0 || m < 0 || ns < 0 || ns > m || N > INT32_MAX || !hess_d || !pr_diag_d || !diag_hess_d || !aug_d ||
        (m && (!jac_d || !du_diag_d)) || (ns && !ind_ineq_d)) {
        set_error("b2d_aug_assemble: invalid argument");
        return B2_ERR_INVALID;
    }
    k_dense_aug<<<(unsigned)N, 256, 0, as_stream(stream)>>>(n, m, ns, ind_ineq_d, hess_d, jac_d, pr_diag_d, du_diag_d, diag_hess_d, aug_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_copy_diag(int32_t n, int32_t lda, const double* A_d, double* d_d, void* stream) {
    if (n < 0 || lda < n || (n && (!A_d || !d_d))) { set_error("b2d_copy_diag: invalid argument"); return B2_ERR_INVALID; }
    if (n == 0) return B2_OK;
    const int g = std::min((n + 255) / 256, 8 * sm_count());
    k_copy_diag<<<g, 256, 0, as_stream(stream)>>>(n, lda, A_d, d_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
