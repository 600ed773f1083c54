// Dense quasi-Newton Hessian updates of the dense KKT systems (MadNLP BFGS and DampedBFGS, src/quasi_newton.jl:71-201, 425-437).
// C ABI in include/b200kkt.h.
//
// Bk is the dense KKT system's `hess`: n x n, column-major, leading dimension n; only its lower triangle is read or written, as
// the reference's _symv!('L') / _syr!('L') do.  Every state value (is_instantiated, the last accept decision, the scalars) lives in
// device memory, and every entry point issues a fixed launch sequence with no host branch on data, so it can be captured in a CUDA
// graph.  The n-wide dot products are grid_sums (grid_reduce.cuh), as in lbfgs.cu: replays are bit-identical.
// update = [s'y, s's; decision] -> [diagonal on the first accepted call] -> b2d_symv_lower (bsk = B s) -> [s'bsk, theta, r, r's,
// alpha1, alpha2] -> one fused read-modify-write pass over the lower triangle that applies both rank-1 terms (the reference's
// symv + syr + syr read the half matrix five times; this reads it three times).
// Concurrent calls on one handle from two streams are not supported (one ticket per handle).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {
constexpr int QN_T = 256;          // threads of the reduction kernels
constexpr int QN_TILE = 64;        // the rank-2 pass works on 64 x 64 tiles of the lower triangle
constexpr int QN_RANK2_T = 256;    // 4 threads per tile row: each updates 16 columns of its row
constexpr int QN_COLS = QN_TILE * QN_TILE / QN_RANK2_T;

struct QnState {
    int32_t instantiated;   // is_instantiated
    int32_t accepted;       // the last update changed Bk
    int32_t set_diag;       // the last update is the first accepted one: the diagonal is rewritten to y's / s's
    double ys, ss, sBs, theta, alpha1, alpha2;
    double init_diag;       // init!: 2 rho0
    unsigned ticket;
};

// init! (quasi_newton.jl:425-437): norm_g0 = g0'g0; the last block stores 2 rho0.  `f0 ≈ 0` with isapprox's default tolerances
// holds for exactly +-0 only.
__global__ void __launch_bounds__(QN_T) k_qn_init(int64_t n, const double* __restrict__ g0, double f0, QnState* st, double* part) {
    __shared__ double out[1];
    auto f = [&](int, int64_t r) { return g0[r] * g0[r]; };
    if (!grid_sums<1>(n, 1, f, part, &st->ticket, out) || threadIdx.x != 0) return;
    const double norm_g0 = out[0];
    const double rho0 = norm_g0 < sqrt(2.220446049250313e-16) ? 1.0 : (f0 == 0.0 ? 1.0 / norm_g0 : fabs(f0) / norm_g0);
    st->init_diag = 2.0 * rho0;
}

// Bk[i, i] = v for the value chosen on the device: init!'s 2 rho0 (init = 1), or y's / s's on the first accepted update
__global__ void k_qn_diag(int64_t n, int init, const QnState* __restrict__ st, double* __restrict__ Bk) {
    if (!init && !st->set_diag) return;
    const double v = init ? st->init_diag : st->ys / st->ss;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        Bk[i + i * n] = v;
}

// update!, launch 1: y's and s's; the last block takes the decision.  BFGS skips when y's < 1e-8 (written as the reference
// writes it, so a NaN is not skipped); DampedBFGS never skips.  The first accepted call rewrites the diagonal (k_qn_diag).
__global__ void __launch_bounds__(QN_T) k_qn_pre(int64_t n, int kind, const double* __restrict__ s, const double* __restrict__ y,
                                                QnState* st, double* part) {
    __shared__ double out[2];
    auto f = [&](int q, int64_t r) { return q == 0 ? s[r] * y[r] : s[r] * s[r]; };
    if (!grid_sums<2>(n, 2, f, part, &st->ticket, out) || threadIdx.x != 0) return;
    const double ys = out[0], ss = out[1];
    const int acc = kind == 1 ? !(ys < 1e-8) : 1;
    st->ys = ys;
    st->ss = ss;
    st->accepted = acc;
    st->set_diag = acc && !st->instantiated;
    if (acc) st->instantiated = 1;
}

// update!, launch 4 (after bsk = B s): sBs = s'bsk, then alpha1 = 1 / sBs and
//   BFGS:        alpha2 = 1 / y's
//   DampedBFGS:  theta (Procedure 18.2), r = (0 + theta y) + (1 - theta) bsk (fill! + two axpy!), alpha2 = 1 / r's
// The last block forms r and r's alone (one n-wide pass, fixed order).
__global__ void __launch_bounds__(QN_T) k_qn_post(int64_t n, int kind, const double* __restrict__ s, const double* __restrict__ y,
                                                 const double* __restrict__ bsk, double* __restrict__ rk, QnState* st, double* part) {
    __shared__ double s_theta;
    __shared__ double out[1];
    auto f = [&](int, int64_t r) { return s[r] * bsk[r]; };
    if (!grid_sums<1>(n, 1, f, part, &st->ticket, out)) return;
    if (threadIdx.x == 0) {
        const double sBs = out[0], ys = st->ys;
        st->sBs = sBs;
        st->alpha1 = 1.0 / sBs;
        const double theta = kind == 2 && ys < 0.2 * sBs ? 0.8 * sBs / (sBs - ys) : 1.0;
        st->theta = theta;
        s_theta = theta;
        if (kind == 1) st->alpha2 = 1.0 / ys;
    }
    __syncthreads();
    if (kind != 2) return;
    const double theta = s_theta, omt = 1.0 - theta;
    double a = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const double r = __dadd_rn(__dadd_rn(0.0, __dmul_rn(theta, y[i])), __dmul_rn(omt, bsk[i]));
        rk[i] = r;
        a += r * s[i];
    }
    a = block_sum(a);
    if (threadIdx.x == 0) st->alpha2 = 1.0 / a;
}

// Tile index e of the lower triangle (row-wise: (0,0), (1,0), (1,1), (2,0), ...) -> (tile row a >= tile column b)
__device__ __forceinline__ void tile_decode(int64_t e, int64_t& a, int64_t& b) {
    a = (int64_t)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
    while (a * (a + 1) / 2 > e) --a;
    while ((a + 1) * (a + 2) / 2 <= e) ++a;
    b = e - a * (a + 1) / 2;
}

// update!, launch 5, on accepted calls only: the two rank-1 terms in one read-modify-write pass over the lower triangle.  Per
// element (i >= j), netlib dsyr's statement order applied twice, in the reference's order, with no contraction:
//   a = a + b_i ((-alpha1) b_j) ;  a = a + v_i (alpha2 v_j)        (v = y for BFGS, r for DampedBFGS)
// One CTA per 64 x 64 tile; a warp covers 32 consecutive rows of one column per access, so every load and store is coalesced.
__global__ void __launch_bounds__(QN_RANK2_T) k_qn_rank2(int64_t n, const QnState* __restrict__ st, const double* __restrict__ b,
                                                        const double* __restrict__ v, double* __restrict__ Bk) {
    __shared__ double t1[QN_TILE], t2[QN_TILE];
    if (!st->accepted) return;
    int64_t ti, tj;
    tile_decode(blockIdx.x, ti, tj);
    const int64_t r0 = ti * QN_TILE, c0 = tj * QN_TILE;
    const int t = threadIdx.x;
    if (t < QN_TILE) {
        const int64_t j = c0 + t;
        const double na1 = -st->alpha1, a2 = st->alpha2;
        t1[t] = j < n ? __dmul_rn(na1, b[j]) : 0.0;
        t2[t] = j < n ? __dmul_rn(a2, v[j]) : 0.0;
    }
    __syncthreads();
    const int64_t i = r0 + (t & (QN_TILE - 1));
    if (i >= n) return;
    const double bi = b[i], vi = v[i];
    const int jc0 = (t / QN_TILE) * QN_COLS;          // this thread's first column within the tile
    double* col = Bk + i + (c0 + jc0) * n;
    double a[QN_COLS];
#pragma unroll
    for (int k = 0; k < QN_COLS; ++k) {
        const int64_t j = c0 + jc0 + k;
        a[k] = (j <= i) ? col[k * n] : 0.0;
    }
#pragma unroll
    for (int k = 0; k < QN_COLS; ++k) {
        const int64_t j = c0 + jc0 + k;
        if (j <= i) {
            double x = __dadd_rn(a[k], __dmul_rn(bi, t1[jc0 + k]));
            x = __dadd_rn(x, __dmul_rn(vi, t2[jc0 + k]));
            col[k * n] = x;
        }
    }
}

}  // namespace

struct b2d_qn {
    int64_t n = 0;
    int kind = 1;
    int nb = 1;
    DevBuf<QnState> st;
    DevBuf<double> bsk, rk, part;
};

// ---------------------------------------------------------------------------------------------------------------------- C ABI
extern "C" int b2d_qn_create(int64_t n, int32_t kind, b2d_qn** out) {
    if (!out || n < 1 || n > INT32_MAX || (kind != B2_QN_BFGS && kind != B2_QN_DAMPED_BFGS)) {
        set_error("b2d_qn_create: invalid argument (1 <= n <= 2^31 - 1, kind 1 = BFGS or 2 = DampedBFGS)");
        return B2_ERR_INVALID;
    }
    auto* h = new b2d_qn();
    h->n = n; h->kind = kind; h->nb = grid_sums_blocks(n);
    cudaError_t e = cudaSuccess;
    auto A = [&](auto& buf, size_t cnt) { if (e == cudaSuccess) e = buf.alloc(cnt); if (e == cudaSuccess) e = cudaMemset(buf.p, 0, buf.bytes()); };
    A(h->st, 1); A(h->bsk, (size_t)n); A(h->rk, (size_t)n); A(h->part, (size_t)h->nb * 2);
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "b2d_qn_create", __FILE__, __LINE__); }
    *out = h;
    return B2_OK;
}

extern "C" int b2d_qn_destroy(b2d_qn* h) { delete h; return B2_OK; }

extern "C" int b2d_qn_init(b2d_qn* h, double* Bk_d, const double* g0_d, double f0, void* stream) {
    if (!h || !Bk_d || !g0_d) { set_error("b2d_qn_init: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    k_qn_init<<<h->nb, QN_T, 0, st>>>(h->n, g0_d, f0, h->st.p, h->part.p);
    k_qn_diag<<<grid_elem(h->n), 256, 0, st>>>(h->n, 1, h->st.p, Bk_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_qn_update(b2d_qn* h, double* Bk_d, const double* sk_d, const double* yk_d, void* stream) {
    if (!h || !Bk_d || !sk_d || !yk_d) { set_error("b2d_qn_update: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    const int64_t n = h->n;
    k_qn_pre<<<h->nb, QN_T, 0, st>>>(n, h->kind, sk_d, yk_d, h->st.p, h->part.p);
    k_qn_diag<<<grid_elem(n), 256, 0, st>>>(n, 0, h->st.p, Bk_d);
    B2_CUDA(cudaGetLastError());
    const int rc = b2d_symv_lower((int32_t)n, (int32_t)n, Bk_d, sk_d, h->bsk.p, 1.0, 0.0, stream);
    if (rc != B2_OK) return rc;
    k_qn_post<<<h->nb, QN_T, 0, st>>>(n, h->kind, sk_d, yk_d, h->bsk.p, h->rk.p, h->st.p, h->part.p);
    const int64_t nt = (n + QN_TILE - 1) / QN_TILE;
    k_qn_rank2<<<(unsigned)(nt * (nt + 1) / 2), QN_RANK2_T, 0, st>>>(n, h->st.p, h->bsk.p, h->kind == B2_QN_BFGS ? yk_d : h->rk.p,
                                                                     Bk_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_qn_rank2(b2d_qn* h, double* Bk_d, const double* yk_d, void* stream) {
    if (!h || !Bk_d || (h->kind == B2_QN_BFGS && !yk_d)) { set_error("b2d_qn_rank2: invalid argument"); return B2_ERR_INVALID; }
    const int64_t nt = (h->n + QN_TILE - 1) / QN_TILE;
    k_qn_rank2<<<(unsigned)(nt * (nt + 1) / 2), QN_RANK2_T, 0, as_stream(stream)>>>(h->n, h->st.p, h->bsk.p,
                                                                                    h->kind == B2_QN_BFGS ? yk_d : h->rk.p, Bk_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_qn_state(b2d_qn* h, int32_t* instantiated, int32_t* accepted, double* scalars, void* stream) {
    if (!h || !instantiated || !accepted || !scalars) { set_error("b2d_qn_state: invalid argument"); return B2_ERR_INVALID; }
    QnState s;
    B2_CUDA(cudaMemcpyAsync(&s, h->st.p, sizeof(s), cudaMemcpyDeviceToHost, as_stream(stream)));
    B2_CUDA(cudaStreamSynchronize(as_stream(stream)));
    *instantiated = s.instantiated; *accepted = s.accepted;
    const double v[6] = {s.ys, s.ss, s.sBs, s.theta, s.alpha1, s.alpha2};
    std::copy(v, v + 6, scalars);
    return B2_OK;
}

extern "C" int b2d_qn_debug_vectors(b2d_qn* h, double* bsk_h, double* rk_h, void* stream) {
    if (!h || !bsk_h || !rk_h) { set_error("b2d_qn_debug_vectors: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemcpyAsync(bsk_h, h->bsk.p, h->n * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaMemcpyAsync(rk_h, h->rk.p, h->n * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    return B2_OK;
}
