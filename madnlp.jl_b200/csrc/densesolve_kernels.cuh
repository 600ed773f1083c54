// Dense triangular solves  x <- (L D L')^{-1} x  in ONE launch: a dataflow over the 128-wide block rows of the factor.
//
// The launch-per-block sweeps (bigsolve_kernels.cuh) cost 2 * N/128 dependent launches (64 at N = 4096, for a job whose
// HBM time is tens of microseconds).  Here CTA k OWNS block row k of the forward sweep and block column k of the backward sweep:
//
//   forward :  t_k = b_k - sum_{c<k} L(k,c) y_c   accumulated as the y_c become available,  y_k = Linv_k t_k
//   diagonal:  z_k = y_k ./ d_k
//   backward:  s_k = z_k - sum_{c>k} L(c,k)' x_c  accumulated as the x_c become available,  x_k = Linv_k' s_k
//
// Hand-off between CTAs goes through two small global vectors (ybuf, xbuf) whose entries start as SLOT_EMPTY
// (ptx.cuh: all ones, a NaN no arithmetic produces) -- a consumer polls the 128 values themselves, so a block costs ONE L2 round trip
// on the critical path instead of flag + data, and needs no fence (8-byte stores are single-copy atomic).  The factor block a
// CTA needs next is loaded into registers BEFORE it polls, so the chain per block is: poll -> 16 FMAs + shared-memory reduction
// (off-diagonal block) -> 16 FMAs + reduction (inverted diagonal block) -> 128 stores.  Every CTA of the grid must be
// resident (grid = N/128 <= number of SMs, 1024 threads each); polls are bounded and report through `err`.
// Deterministic: fixed summation order, no atomics.
#pragma once
#include "bigsolve_kernels.cuh"
#include "ptx.cuh"

namespace b2 {

constexpr int DS_NT = 1024;
constexpr unsigned DS_SPIN_MAX = 1u << 22;

__device__ __forceinline__ double ds_poll(const double* p, int* err) {
    unsigned long long v;
    if (!bounded_spin<DS_SPIN_MAX, 0>(err, [&](unsigned) { return (v = ld_relaxed_b64(p)) != SLOT_EMPTY; })) return 0.0;
    return __longlong_as_double((long long)v);
}

// L: N x N column-major factor (unit lower, D on the diagonal), Linv: inverted 128 x 128 diagonal blocks (ld 128),
// dvec: D, x: right-hand side in / solution out, ybuf/xbuf: [nblk*128] hand-off vectors preset to SLOT_EMPTY.
// Registers hold ONE 128 x 128 block of L (16 doubles per thread, 1024 threads); its load is issued BEFORE the poll of the
// vector it multiplies, so on the critical path (the newest y_c / x_c) the block is already there.  The CTA's own inverted
// diagonal block sits in shared memory (cp.async at kernel start, padded rows: both the plain and the transposed apply are
// bank-conflict free).
constexpr int DS_LDI = BS + 1;
constexpr size_t DS_SMEM = (size_t)(BS * DS_LDI + 2 * BS + 2 * 8 * BS + BS) * sizeof(double);

// BK (Bunch-Kaufman factor, dense_bk.cu): L is the unit-lower factor of A(perm, perm), so x is gathered through perm on entry and
// scattered through it on exit, and D is block diagonal: evec[i] != 0 marks a 2 x 2 block on rows (i, i+1), which may straddle two
// 128-row blocks -- its partner value is then polled from ybuf like any other hand-off (the block after publishes it once its own
// forward sweep, which needs only this block's y, is done).  The 2 x 2 solve is dsytrs's.
template <bool BK>
__global__ void __launch_bounds__(DS_NT, 1) k_dense_solve_flow(int N, const double* __restrict__ L, const double* __restrict__ Linv,
                                                              const double* __restrict__ dvec, double* __restrict__ x,
                                                              double* ybuf, double* xbuf, int* err,
                                                              const int32_t* __restrict__ perm, const double* __restrict__ evec) {
    extern __shared__ __align__(16) double ds_sm[];
    double* Ls = ds_sm;                                   // [BS][DS_LDI]: Ls[c*DS_LDI + r] = Linv_k(r, c)
    double (*vec)[BS] = (double (*)[BS])(Ls + BS * DS_LDI);                  // [2][BS] the block vector being applied
    double (*part)[8][BS] = (double (*)[8][BS])(Ls + BS * DS_LDI + 2 * BS);  // [2][8][BS] partial sums of the 8 groups
    double* tk = Ls + BS * DS_LDI + 2 * BS + 2 * 8 * BS;                     // [BS]
    const int k = blockIdx.x, kb = k * BS;
    const int nblk = gridDim.x;
    const int nb = min(BS, N - kb);
    const int tid = threadIdx.x, r = tid & (BS - 1), g = tid >> 7;           // r: row (fwd) / column (bwd) inside the block
    {
        const double* Li = Linv + (size_t)k * BS * BS;
        for (int e = tid; e < BS * BS; e += DS_NT) cp_async8(Ls + (e >> 7) * DS_LDI + (e & (BS - 1)), Li + e);
        cp_async_commit_group();
    }
    // ---------------- forward
    double t = (g == 0 && r < nb) ? x[BK ? perm[kb + r] : kb + r] : 0.0;     // group 0 carries the accumulator
    double v[16];
    for (int c = 0; c < k; ++c) {
        {                                                                     // L(kb + r, c*BS + g*16 + q), issued before the poll
            const double* p = L + (size_t)(c * BS + g * 16) * N + kb + min(r, nb - 1);
#pragma unroll
            for (int q = 0; q < 16; ++q) v[q] = (r < nb) ? p[(size_t)q * N] : 0.0;
        }
        const int b = c & 1;
        if (tid < BS) vec[b][tid] = ds_poll(ybuf + (size_t)c * BS + tid, err);
        __syncthreads();
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < 16; ++q) acc = fma(v[q], vec[b][g * 16 + q], acc);
        part[b][g][r] = acc;
        __syncthreads();
        if (g == 0) {
            double sum = 0.0;
#pragma unroll
            for (int u = 0; u < 8; ++u) sum += part[b][u][r];
            t -= sum;
        }
    }
    cp_async_wait_all();
    if (g == 0) tk[r] = t;
    __syncthreads();
    {                                                                         // y_k = Linv_k t_k   (Linv(r, c) = 0 for c > r)
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < 16; ++q) { const int c = g * 16 + q; acc = fma((c <= r) ? Ls[c * DS_LDI + r] : 0.0, tk[c], acc); }
        part[0][g][r] = acc;
    }
    __syncthreads();
    double yk = 0.0;
    if (g == 0) {
#pragma unroll
        for (int u = 0; u < 8; ++u) yk += part[0][u][r];
        if (r >= nb) yk = 0.0;
        ybuf[(size_t)k * BS + r] = yk;                                        // publish y_k (consumers: the block rows below)
    }
    // ---------------- diagonal + backward
    // s_k(j) -= sum_i L(cb + i, kb + j) x_c(i): a warp owns 4 columns j, its lanes stride the rows i (each load instruction reads
    // 32 consecutive rows of one column: coalesced), column sums meet through shuffles; `sacc` lives in the threads tid < BS
    double s = (g == 0 && r < nb) ? yk / dvec[kb + r] : 0.0;
    if constexpr (BK) {
        const int i = kb + r;
        const bool first = g == 0 && r < nb && evec[i] != 0.0, second = g == 0 && r < nb && i > 0 && evec[i - 1] != 0.0;
        if (first || second) {
            const int i0 = first ? i : i - 1;
            const double y0 = first ? yk : ds_poll(ybuf + i0, err), y1 = first ? ds_poll(ybuf + i0 + 1, err) : yk;
            const double akm1k = evec[i0], akm1 = dvec[i0] / akm1k, ak = dvec[i0 + 1] / akm1k;
            const double denom = akm1 * ak - 1.0, bkm1 = y0 / akm1k, bk = y1 / akm1k;
            s = first ? (ak * bkm1 - bk) / denom : (akm1 * bk - bkm1) / denom;
        }
    }
    const int warp = tid >> 5, lane = tid & 31;
    for (int c = nblk - 1; c > k; --c) {
        const int cb = c * BS, ncb = min(BS, N - cb);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int j = warp * 4 + q;
            const double* p = L + (size_t)(kb + min(j, nb - 1)) * N + cb;
#pragma unroll
            for (int u = 0; u < 4; ++u) v[q * 4 + u] = (j < nb && lane + 32 * u < ncb) ? p[lane + 32 * u] : 0.0;
        }
        const int b = c & 1;
        if (tid < BS) vec[b][tid] = ds_poll(xbuf + (size_t)c * BS + tid, err);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double acc = 0.0;
#pragma unroll
            for (int u = 0; u < 4; ++u) acc = fma(v[q * 4 + u], vec[b][lane + 32 * u], acc);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) part[b][0][warp * 4 + q] = acc;
        }
        __syncthreads();
        if (g == 0) s -= part[b][0][r];
    }
    __syncthreads();
    if (g == 0) tk[r] = s;
    __syncthreads();
    {                                                                         // x_k = Linv_k' s_k : sum_{i >= r} Linv(i, r) s_i
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < 16; ++q) { const int i = g * 16 + q; acc = fma((i >= r) ? Ls[r * DS_LDI + i] : 0.0, tk[i], acc); }
        part[1][g][r] = acc;
    }
    __syncthreads();
    if (g == 0) {
        double xk = 0.0;
#pragma unroll
        for (int u = 0; u < 8; ++u) xk += part[1][u][r];
        if (r >= nb) xk = 0.0;
        xbuf[(size_t)k * BS + r] = xk;                                        // publish x_k (consumers: the block columns before)
        if (r < nb) x[BK ? perm[kb + r] : kb + r] = xk;
    }
}

}  // namespace b2
