// Restarted GMRES preconditioned on the right by the KKT solve (KrylovIterator, madnlp.jl_b200/krylov.py): the vector passes of one
// Arnoldi step and of a cycle close.  The host layer runs solve_kkt! and mul! of the KKT type in between; everything else -- the
// basis V, the preconditioned vectors Z, H, the Givens rotations, g, y and the per-iteration record -- is device memory owned by
// the handle.  Reductions are the fixed-order grid_reduce (last CTA by ticket), max norms are integer atomicMax on the bits of
// non-negative doubles: no floating-point atomics, so replays are bit-identical.  No entry allocates or synchronises, so every
// sequence can be captured in a CUDA graph.
#include <cmath>

#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

constexpr int KR_LDH = B2_KRYLOV_MAX_RESTART + 1;       // rows of H (column-major, column k at st + B2_KRYLOV_H + k * KR_LDH)

struct b2_krylov {
    int64_t n = 0;
    int restart = 0;
    DevBuf<double> V;          // (restart + 1) x n: the Arnoldi basis
    DevBuf<double> Z;          // restart x n: z_k = M^-1 v_k
    DevBuf<double> st;         // B2_KRYLOV_STATE_LEN doubles: H, rotations, g, y, the divisor of the next scale pass, the record
    DevBuf<double> part;       // grid_reduce partials
    DevBuf<unsigned> ticket;
};

// NaN-propagating max of non-negative doubles, committed as integers
__device__ __forceinline__ void kr_max_commit(double mx, double* out) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, mx, o); if (t > mx || t != t) mx = t; }
    if ((threadIdx.x & 31) == 0) atomicMax((unsigned long long*)out, (unsigned long long)__double_as_longlong(mx));
}

// start of a cycle.  first: x = 0, w = b, rec[NORM_B] = ||b||_inf.  Then beta = ||w||_2 (w holds r = b - K x), g = beta e_1 and
// the divisor of the next scale pass is beta; first: rec[NORM_B2] = beta.
__global__ void k_krylov_begin(int64_t n, int first, const double* __restrict__ b, double* __restrict__ x, double* __restrict__ w,
                               double* __restrict__ st, double* __restrict__ part, unsigned* ticket) {
    double v[1] = {0.0}, out[1];
    double mx = 0.0;
    GRID_STRIDE(i, n) {
        double wi;
        if (first) {
            wi = b[i];
            w[i] = wi;
            x[i] = 0.0;
            const double a = fabs(wi);
            if (a > mx || a != a) mx = a;
        } else {
            wi = w[i];
        }
        v[0] += wi * wi;
    }
    if (first) kr_max_commit(mx, st + B2_KRYLOV_REC + B2_KRYLOV_REC_NORM_B);
    if (!grid_reduce<R_SUM, 1>(v, 0.0, part, ticket, out)) return;
    if (threadIdx.x == 0) {
        const double beta = sqrt(out[0]);
        for (int j = 0; j < KR_LDH; ++j) st[B2_KRYLOV_G + j] = 0.0;
        st[B2_KRYLOV_G] = beta;
        st[B2_KRYLOV_SCALE] = beta;
        if (first) st[B2_KRYLOV_REC + B2_KRYLOV_REC_NORM_B2] = beta;
    }
}

// v_k = w / s and z_k = v_k (the copy solve_kkt! overwrites in place), s = the divisor left by the previous pass (beta or h_{k,k-1});
// s = 0 (b = 0) writes zeros
__global__ void k_krylov_scale(int64_t n, const double* __restrict__ w, double* __restrict__ vk, double* __restrict__ zk,
                               const double* __restrict__ st) {
    const double s = st[B2_KRYLOV_SCALE];
    GRID_STRIDE(i, n) {
        const double t = s != 0.0 ? w[i] / s : 0.0;
        vk[i] = t;
        zk[i] = t;
    }
}

// modified Gram-Schmidt pass i of Arnoldi step k (w = K z_k on entry of pass 0).  Pass i first applies the previous projection
// w -= h_{i-1,k} v_{i-1}, then reduces <v_i, w> (i <= k, written to h_{i,k}) or ||w||_2^2 (i = k + 1).  After the norm the last CTA
// applies the stored rotations to column k, forms the new one, updates g and writes the record (|g_{k+1}|, h_{k+1,k}); h_{k+1,k}
// is also the divisor of the next scale pass.
__global__ void k_krylov_mgs(int64_t n, int64_t ld, int k, int i, const double* __restrict__ V, double* __restrict__ w,
                             double* __restrict__ st, double* __restrict__ part, unsigned* ticket) {
    double* h = st + B2_KRYLOV_H + (int64_t)k * KR_LDH;
    const double hp = i > 0 ? h[i - 1] : 0.0;
    const double* vp = V + (int64_t)(i > 0 ? i - 1 : 0) * ld;
    const double* vi = V + (int64_t)(i <= k ? i : 0) * ld;
    double v[1] = {0.0}, out[1];
    GRID_STRIDE(t, n) {
        double wt = w[t];
        if (i > 0) {
            wt -= hp * vp[t];
            w[t] = wt;
        }
        v[0] += (i <= k ? vi[t] : wt) * wt;
    }
    if (!grid_reduce<R_SUM, 1>(v, 0.0, part, ticket, out)) return;
    if (threadIdx.x != 0) return;
    if (i <= k) {
        h[i] = out[0];
        return;
    }
    double* cs = st + B2_KRYLOV_CS;
    double* sn = st + B2_KRYLOV_SN;
    double* g = st + B2_KRYLOV_G;
    const double hk1 = sqrt(out[0]);
    for (int j = 0; j < k; ++j) {
        const double a = h[j], c = h[j + 1];
        h[j] = cs[j] * a + sn[j] * c;
        h[j + 1] = -sn[j] * a + cs[j] * c;
    }
    const double d = hypot(h[k], hk1);
    const double c = d != 0.0 ? h[k] / d : 1.0, s = d != 0.0 ? hk1 / d : 0.0;
    cs[k] = c;
    sn[k] = s;
    h[k] = d;
    h[k + 1] = 0.0;
    const double gk = g[k];
    g[k] = c * gk;
    g[k + 1] = -s * gk;
    st[B2_KRYLOV_SCALE] = hk1;
    st[B2_KRYLOV_REC + B2_KRYLOV_REC_EST] = fabs(g[k + 1]);
    st[B2_KRYLOV_REC + B2_KRYLOV_REC_H] = hk1;
}

// y = R^-1 g over m = k + 1 columns (upper triangular, m <= 16) by one warp: R is staged in shared memory, lane j holds y_j, and
// row i's sum over j > i is an xor-tree warp reduction; y goes to the state, where the close pass reads it
__global__ void k_krylov_y(int m, double* __restrict__ st) {
    __shared__ double R[B2_KRYLOV_MAX_RESTART][B2_KRYLOV_MAX_RESTART];
    const int lane = threadIdx.x;
    for (int e = lane; e < m * m; e += 32) {
        const int i = e % m, j = e / m;
        R[i][j] = st[B2_KRYLOV_H + i + j * KR_LDH];
    }
    __syncwarp();
    double y = 0.0;
    for (int i = m - 1; i >= 0; --i) {
        double t = (lane > i && lane < m) ? R[i][lane] * y : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == i) y = (st[B2_KRYLOV_G + i] - t) / R[i][i];
    }
    if (lane < m) st[B2_KRYLOV_Y + lane] = y;
}

// cycle close over m = k + 1 columns: x += Z y (columns in index order, y from k_krylov_y), w = b and rec[NORM_X] = ||x||_inf
__global__ void k_krylov_close(int64_t n, int64_t ld, int m, const double* __restrict__ Z, const double* __restrict__ b,
                               double* __restrict__ x, double* __restrict__ w, double* __restrict__ st) {
    __shared__ double y[B2_KRYLOV_MAX_RESTART];
    if (threadIdx.x < m) y[threadIdx.x] = st[B2_KRYLOV_Y + threadIdx.x];
    __syncthreads();
    double mx = 0.0;
    GRID_STRIDE(t, n) {
        double xt = x[t];
        for (int j = 0; j < m; ++j) xt += y[j] * Z[(int64_t)j * ld + t];
        x[t] = xt;
        w[t] = b[t];
        const double a = fabs(xt);
        if (a > mx || a != a) mx = a;
    }
    kr_max_commit(mx, st + B2_KRYLOV_REC + B2_KRYLOV_REC_NORM_X);
}

extern "C" int b2_krylov_create(int64_t n, int32_t restart, b2_krylov** out) {
    if (!out || n <= 0 || restart < 1 || restart > B2_KRYLOV_MAX_RESTART) {
        set_error("b2_krylov_create: invalid argument (n >= 1, 1 <= restart <= 16)");
        return B2_ERR_INVALID;
    }
    auto* h = new b2_krylov();
    h->n = n;
    h->restart = restart;
    cudaError_t e = cudaSuccess;
    auto A = [&](auto& buf, size_t cnt) { if (e == cudaSuccess) e = buf.alloc(cnt); if (e == cudaSuccess) e = cudaMemset(buf.p, 0, buf.bytes()); };
    A(h->V, (size_t)(restart + 1) * n); A(h->Z, (size_t)restart * n); A(h->st, B2_KRYLOV_STATE_LEN);
    A(h->part, B2_RED_BLOCKS); A(h->ticket, 1);
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "b2_krylov_create", __FILE__, __LINE__); }
    *out = h;
    return B2_OK;
}

extern "C" int b2_krylov_destroy(b2_krylov* h) { delete h; return B2_OK; }

extern "C" int b2_krylov_buffers(b2_krylov* h, double** V, double** Z, double** state) {
    if (!h || !V || !Z || !state) { set_error("b2_krylov_buffers: invalid argument"); return B2_ERR_INVALID; }
    *V = h->V.p; *Z = h->Z.p; *state = h->st.p;
    return B2_OK;
}

extern "C" int b2_krylov_begin(b2_krylov* h, int32_t first, const double* b_d, double* x_d, double* w_d, void* stream) {
    if (!h || !w_d || (first && (!b_d || !x_d))) { set_error("b2_krylov_begin: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    if (first) B2_CUDA(cudaMemsetAsync(h->st.p + B2_KRYLOV_REC, 0, B2_KRYLOV_REC_LEN * sizeof(double), st));
    k_krylov_begin<<<grid_red(h->n), 256, 0, st>>>(h->n, first ? 1 : 0, b_d, x_d, w_d, h->st.p, h->part.p, h->ticket.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_krylov_scale(b2_krylov* h, int32_t k, const double* w_d, void* stream) {
    if (!h || !w_d || k < 0 || k >= h->restart) { set_error("b2_krylov_scale: invalid argument"); return B2_ERR_INVALID; }
    k_krylov_scale<<<grid_elem(h->n), 256, 0, as_stream(stream)>>>(h->n, w_d, h->V.p + (int64_t)k * h->n, h->Z.p + (int64_t)k * h->n,
                                                                     h->st.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_krylov_orthogonalize(b2_krylov* h, int32_t k, double* w_d, void* stream) {
    if (!h || !w_d || k < 0 || k >= h->restart) { set_error("b2_krylov_orthogonalize: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    for (int i = 0; i <= k + 1; ++i)
        k_krylov_mgs<<<grid_red(h->n), 256, 0, st>>>(h->n, h->n, k, i, h->V.p, w_d, h->st.p, h->part.p, h->ticket.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_krylov_close(b2_krylov* h, int32_t m, const double* b_d, double* x_d, double* w_d, void* stream) {
    if (!h || !b_d || !x_d || !w_d || m < 1 || m > h->restart) { set_error("b2_krylov_close: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemsetAsync(h->st.p + B2_KRYLOV_REC + B2_KRYLOV_REC_NORM_W, 0, 2 * sizeof(double), st));   // NORM_W, NORM_X
    k_krylov_y<<<1, 32, 0, st>>>(m, h->st.p);
    k_krylov_close<<<grid_elem(h->n), 256, 0, st>>>(h->n, h->n, m, h->Z.p, b_d, x_d, w_d, h->st.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
