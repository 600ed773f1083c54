// Multi-CTA triangular solves for HBM-resident fronts (order > 64) and the dense solver.
//
// The pivot columns of a front are cut into blocks of BS = 128 whose unit-lower diagonal blocks are available INVERTED
// (k_big_diag128 for the big fronts, k_big_inv for the shared-memory class).  A sweep is one launch per block:
//   forward  block b: every CTA reads y_b (128 values) and updates its own 128 rows below:
//                     y_i -= sum_k L(i,k) y_b(k)  (coalesced stream of the panel); the CTA that owns the rows of block
//                     b+1 then forms y_{b+1} = Linv_{b+1} * rhs_{b+1} for the next launch.
//   backward block b: every CTA reads x_b and updates one earlier block of 128 pivot columns:
//                     t_j -= sum_i L(b_i, j) x_b(i)  (one warp per column: right-looking, deterministic, no cross-CTA
//                     reduction); the CTA of block b-1 then forms x_{b-1} = Linv_{b-1}' * t_{b-1}.
// so the 128 KB inverse block is read by ONE CTA per launch and the sweep is bounded by streaming L once.
#pragma once
#include "solve_kernels.cuh"

namespace b2 {

constexpr int BS = 128;

struct BigSolveArgs {
    SolveArgs s;
    const double* Linv;          // inverted diagonal blocks, BS*BS doubles each (column-major, ld BS)
    const int64_t* linv_off;     // per supernode: offset of its first block in Linv (-1: not a big front)
    double* side;                // [n] solved pivot blocks are parked here: CTA 0 must not overwrite the block's right-hand
                                 // side in xp while the other CTAs of the same launch are still reading it
};

// ---- inversion of the unit-lower diagonal blocks (once per factorisation); grid (max blocks, nfronts), 128 threads
__global__ void __launch_bounds__(BS) k_big_inv(const FrontDesc* desc, const int32_t* __restrict__ list, const double* __restrict__ L,
                                                double* __restrict__ Linv, const int64_t* __restrict__ linv_off) {
    extern __shared__ double T[];                 // [BS][BS+1], T[i*(BS+1)+j] = row i, col j
    const int s = list[blockIdx.y];
    const FrontDesc d = desc[s];
    const int kb = blockIdx.x * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb), f = d.f, tid = threadIdx.x;
    const double* Lp = L + d.lp_off;
    for (int c = 0; c < nb; ++c) {                // coalesced over rows
        if (tid < nb) T[tid * (BS + 1) + c] = (tid > c) ? Lp[(size_t)(kb + c) * f + kb + tid] : (tid == c ? 1.0 : 0.0);
    }
    __syncthreads();
    // in-place inversion, columns from the last to the first: X(i,j) = -( L(i,j) + sum_{j<k<i} X(i,k) L(k,j) )
    for (int j = nb - 2; j >= 0; --j) {
        double v = 0.0;
        if (tid > j && tid < nb) {
            v = T[tid * (BS + 1) + j];
            for (int k = j + 1; k < tid; ++k) v = fma(T[tid * (BS + 1) + k], T[k * (BS + 1) + j], v);
        }
        __syncthreads();
        if (tid > j && tid < nb) T[tid * (BS + 1) + j] = -v;
        __syncthreads();
    }
    double* out = Linv + linv_off[s] + (size_t)blockIdx.x * BS * BS;
    for (int c = 0; c < BS; ++c) out[(size_t)c * BS + tid] = (tid < nb && c < nb) ? T[tid * (BS + 1) + c] : 0.0;
}

// location of entry i (0..f) of the front's solve vector: pivots live in xp, the rest in the contribution vector
__device__ __forceinline__ double* yptr(const SolveArgs& a, const FrontDesc& d, int64_t cbv0, int i) {
    return (i < d.w) ? a.xp + d.col0 + i : a.cbv + cbv0 + (i - d.w);
}

// ---- forward init: zero the contribution vector, pull the children (ascending id); one CTA per front
__global__ void __launch_bounds__(1024) k_bs_fwd_init(BigSolveArgs b, const int32_t* __restrict__ list) {
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.x];
    const FrontDesc d = a.desc[s];
    const int64_t cbv0 = a.cbv_off[s];
    const int r = d.f - d.w, tid = threadIdx.x;
    for (int i = tid; i < r; i += 1024) a.cbv[cbv0 + i] = 0.0;
    __syncthreads();
    for (int c = 0; c < d.nchild; ++c) {
        const int cs = a.child_idx[d.child_off + c];
        const FrontDesc dc = a.desc[cs];
        const int rc = dc.f - dc.w;
        const int32_t* rl = a.rel + dc.rel_off;
        const double* cv = a.cbv + a.cbv_off[cs];
        for (int i = tid; i < rc; i += 1024) *yptr(a, d, cbv0, rl[i]) += cv[i];
        __syncthreads();
    }
}

// Every launch of a sweep is a link of a dependent chain, so what matters is its LATENCY: 1024 threads per CTA, every
// thread issues all of its (<= 16) loads before the first use -- one memory round trip per phase.
constexpr int BS_NT = 1024;
constexpr int BS_KG = BS_NT / BS;         // 8 k-groups of 16 columns

// ---- y = Linv_b * rhs (forward) or x = Linv_b' * t (backward) of one diagonal block; sm >= (1 + BS_KG) * BS doubles
__device__ __forceinline__ void bs_block_apply(const double* __restrict__ Li, const double* rhs, int nb, bool transpose, double* out,
                                               double* sm, int tid) {
    __syncthreads();
    if (tid < BS) sm[tid] = (tid < nb) ? rhs[tid] : 0.0;
    __syncthreads();
    if (!transpose) {
        const int r = tid & (BS - 1), g = tid >> 7;               // BS_KG groups of 16 columns; Linv(r, c) = 0 for c > r
        double v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) { const int c = g * 16 + k; v[k] = (c <= r) ? Li[(size_t)c * BS + r] : 0.0; }
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 16; ++k) acc = fma(v[k], sm[g * 16 + k], acc);
        sm[BS + tid] = acc;
        __syncthreads();
        if (tid < nb) {
            double tot = 0.0;
#pragma unroll
            for (int q = 0; q < BS_KG; ++q) tot += sm[BS + q * BS + tid];
            out[tid] = tot;
        }
    } else {
        const int warp = tid >> 5, lane = tid & 31;               // 32 warps x 4 columns; a column is contiguous over the rows
        double v[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int c = warp * 4 + q, r = lane + 32 * u;
                v[q][u] = (r >= c) ? Li[(size_t)c * BS + r] : 0.0;
            }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double acc = 0.0;
#pragma unroll
            for (int u = 0; u < 4; ++u) acc = fma(v[q][u], sm[lane + 32 * u], acc);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0 && warp * 4 + q < nb) out[warp * 4 + q] = acc;
        }
    }
}

// ---- head of a sweep: block `blk` of every front (blk < 0: each front's own LAST block); one CTA per front
__global__ void __launch_bounds__(BS_NT) k_bs_head(BigSolveArgs b, const int32_t* __restrict__ list, int blk, int transpose) {
    __shared__ double sm[(1 + BS_KG) * BS];
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.x];
    const FrontDesc d = a.desc[s];
    if (blk < 0) blk = (d.w - 1) / BS;
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb);
    bs_block_apply(b.Linv + b.linv_off[s] + (size_t)blk * BS * BS, a.xp + d.col0 + kb, nb, transpose != 0, b.side + d.col0 + kb, sm, threadIdx.x);
}

constexpr int BSF_ROWS = 128;    // rows per CTA in the forward update (x BS_KG k-groups = 1024 threads)
__global__ void __launch_bounds__(BS_NT) k_bs_fwd(BigSolveArgs b, const int32_t* __restrict__ list, int blk) {
    __shared__ double sm[(1 + BS_KG) * BS];                        // y_b | partial sums
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb), f = d.f, tid = threadIdx.x;
    const int row0 = kb + nb + blockIdx.x * BSF_ROWS;
    if (row0 >= f) return;
    if (tid < BS) sm[tid] = (tid < nb) ? b.side[d.col0 + kb + tid] : 0.0;
    const int ir = tid & (BSF_ROWS - 1), g = tid >> 7;
    const int i = row0 + ir;
    double v[16];
    {
        const double* col = a.L + d.lp_off + (size_t)(kb + g * 16) * f + min(i, f - 1);
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = (i < f && g * 16 + k < nb) ? col[(size_t)k * f] : 0.0;
    }
    __syncthreads();
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 16; ++k) acc = fma(v[k], sm[g * 16 + k], acc);
    sm[BS + tid] = acc;
    __syncthreads();
    if (g == 0 && i < f) {
        double tot = 0.0;
#pragma unroll
        for (int q = 0; q < BS_KG; ++q) tot += sm[BS + q * BS + ir];
        *yptr(a, d, a.cbv_off[s], i) -= tot;
    }
    // the rows of this CTA are the pivots of the next block: its right-hand side is final now
    if (blockIdx.x == 0 && kb + BS < d.w)
        bs_block_apply(b.Linv + b.linv_off[s] + (size_t)(blk + 1) * BS * BS, a.xp + d.col0 + kb + BS, min(BS, d.w - kb - BS), false,
                       b.side + d.col0 + kb + BS, sm, tid);
}

// ---- backward init: t_j = y_j / d_j - sum_{i >= w} L(i,j) x(rows_i)  (y_j parked in `side` by the forward sweep);
//      one warp per pivot column (lanes stride the rows: coalesced stream of the column), grid (ceil(w/8), nfronts)
__global__ void __launch_bounds__(256) k_bs_bwd_init(BigSolveArgs b, const int32_t* __restrict__ list) {
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= d.w) return;
    const int f = d.f;
    const double* __restrict__ col = a.L + d.lp_off + (size_t)j * f;
    const int32_t* __restrict__ rows = a.rows + d.rows_off;
    double acc = 0.0;
    int i = d.w + lane;
    for (; i + 96 < f; i += 128) {
        double l[4], x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { l[u] = col[i + 32 * u]; x[u] = a.xp[rows[i + 32 * u]]; }
#pragma unroll
        for (int u = 0; u < 4; ++u) acc = fma(l[u], x[u], acc);
    }
    for (; i < f; i += 32) acc = fma(col[i], a.xp[rows[i]], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) a.xp[d.col0 + j] = b.side[d.col0 + j] / a.dvec[d.col0 + j] - acc;
}

constexpr int BSB_COLS = BS;     // earlier pivot columns per CTA in the backward update: exactly one block
__global__ void __launch_bounds__(BS_NT) k_bs_bwd(BigSolveArgs b, const int32_t* __restrict__ list, int blk) {
    __shared__ double sm[(1 + BS_KG) * BS];                        // x_b
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb), f = d.f, tid = threadIdx.x;
    const int t = blockIdx.x;                                      // block of columns served by this CTA, t < blk
    if (t >= blk) return;
    if (tid < BS) sm[tid] = (tid < nb) ? b.side[d.col0 + kb + tid] : 0.0;
    const int warp = tid >> 5, lane = tid & 31;                   // 32 warps x 4 columns: rows [kb, kb+nb) of a column are contiguous
    double v[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const double* col = a.L + d.lp_off + (size_t)(t * BS + warp * 4 + q) * f + kb;
#pragma unroll
        for (int u = 0; u < 4; ++u) v[q][u] = (lane + 32 * u < nb) ? col[lane + 32 * u] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        double acc = 0.0;
#pragma unroll
        for (int u = 0; u < 4; ++u) acc = fma(v[q][u], sm[lane + 32 * u], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) a.xp[d.col0 + t * BS + warp * 4 + q] -= acc;
    }
    // block blk-1 has received its last update: form x_{blk-1} for the next launch
    if (t == blk - 1)
        bs_block_apply(b.Linv + b.linv_off[s] + (size_t)t * BS * BS, a.xp + d.col0 + t * BS, BS, true, b.side + d.col0 + t * BS, sm, tid);
}

// ---- end of a front's backward sweep: solved pivots from `side` back into xp; grid (ceil(w/256), nfronts)
__global__ void __launch_bounds__(256) k_bs_bwd_finish(BigSolveArgs b, const int32_t* __restrict__ list) {
    const FrontDesc d = b.s.desc[list[blockIdx.y]];
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j < d.w) b.s.xp[d.col0 + j] = b.side[d.col0 + j];
}

// ------------------------------------------------------------------------------------------------ NR right-hand sides
// The same sweeps for NR right-hand sides in one launch (b2_solve's level-launch block solve): xp, cbv and side hold NR interleaved
// columns, entry i of column q at [i * NR + q].  Every panel element and Linv entry is loaded once and applied to all NR columns, and
// column q goes through exactly the operations of the one-column kernel in the same order, so it is bit-identical to a one-column
// solve.  (Separate from the one-column kernels: an NR = 1 instance of these bodies does not compile to the same code.)

// yptr for NR interleaved columns: the entry of column 0
template <int NR>
__device__ __forceinline__ double* yptr_block(const SolveArgs& a, const FrontDesc& d, int64_t cbv0, int i) {
    return (i < d.w) ? a.xp + (d.col0 + i) * NR : a.cbv + (cbv0 + (i - d.w)) * NR;
}

// ---- forward init: zero the contribution vector, pull the children (ascending id); one CTA per front
template <int NR>
__device__ __forceinline__ void bs_fwd_init(const BigSolveArgs& b, const int32_t* __restrict__ list) {
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.x];
    const FrontDesc d = a.desc[s];
    const int64_t cbv0 = a.cbv_off[s];
    const int r = d.f - d.w, tid = threadIdx.x;
    for (int i = tid; i < r * NR; i += 1024) a.cbv[cbv0 * NR + i] = 0.0;
    __syncthreads();
    for (int c = 0; c < d.nchild; ++c) {
        const int cs = a.child_idx[d.child_off + c];
        const FrontDesc dc = a.desc[cs];
        const int rc = dc.f - dc.w;
        const int32_t* rl = a.rel + dc.rel_off;
        const double* cv = a.cbv + a.cbv_off[cs] * NR;
        for (int i = tid; i < rc; i += 1024) {
            double* y = yptr_block<NR>(a, d, cbv0, rl[i]);
#pragma unroll
            for (int q = 0; q < NR; ++q) y[q] += cv[i * NR + q];
        }
        __syncthreads();
    }
}
template <int NR>
__global__ void __launch_bounds__(1024) k_bs_fwd_init_block(BigSolveArgs b, const int32_t* __restrict__ list) { bs_fwd_init<NR>(b, list); }

// shared memory of the forward kernels: NR planes of BS right-hand-side values, then NR planes of BS_NT partial sums; the backward
// kernels use the first NR * BS doubles only
template <int NR>
constexpr int bs_smem_doubles() { return NR * (BS + BS_NT); }

// ---- y = Linv_b * rhs (forward) or x = Linv_b' * t (backward) of one diagonal block; sm >= bs_smem_doubles<NR>()
template <int NR>
__device__ __forceinline__ void bs_block_apply_block(const double* __restrict__ Li, const double* rhs, int nb, bool transpose, double* out,
                                               double* sm, int tid) {
    __syncthreads();
    if (tid < BS) {
#pragma unroll
        for (int q = 0; q < NR; ++q) sm[q * BS + tid] = (tid < nb) ? rhs[tid * NR + q] : 0.0;
    }
    __syncthreads();
    if (!transpose) {
        const int r = tid & (BS - 1), g = tid >> 7;               // BS_KG groups of 16 columns; Linv(r, c) = 0 for c > r
        double v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) { const int c = g * 16 + k; v[k] = (c <= r) ? Li[(size_t)c * BS + r] : 0.0; }
        double* part = sm + NR * BS;
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 16; ++k) acc = fma(v[k], sm[q * BS + g * 16 + k], acc);
            part[q * BS_NT + tid] = acc;
        }
        __syncthreads();
        if (tid < nb) {
#pragma unroll
            for (int q = 0; q < NR; ++q) {
                double tot = 0.0;
#pragma unroll
                for (int kg = 0; kg < BS_KG; ++kg) tot += part[q * BS_NT + kg * BS + tid];
                out[tid * NR + q] = tot;
            }
        }
    } else {
        const int warp = tid >> 5, lane = tid & 31;               // 32 warps x 4 columns; a column is contiguous over the rows
        double v[4][4];
#pragma unroll
        for (int cq = 0; cq < 4; ++cq)
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int c = warp * 4 + cq, r = lane + 32 * u;
                v[cq][u] = (r >= c) ? Li[(size_t)c * BS + r] : 0.0;
            }
#pragma unroll 1
        for (int q = 0; q < NR; ++q) {                            // (one column at a time: 64 registers at 1024 threads)
#pragma unroll
            for (int cq = 0; cq < 4; ++cq) {
                double acc = 0.0;
#pragma unroll
                for (int u = 0; u < 4; ++u) acc = fma(v[cq][u], sm[q * BS + lane + 32 * u], acc);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (lane == 0 && warp * 4 + cq < nb) out[(warp * 4 + cq) * NR + q] = acc;
            }
        }
    }
}

// ---- head of a sweep: block `blk` of every front (blk < 0: each front's own LAST block); one CTA per front
template <int NR>
__device__ __forceinline__ void bs_head(const BigSolveArgs& b, const int32_t* __restrict__ list, int blk, int transpose, double* sm) {
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.x];
    const FrontDesc d = a.desc[s];
    if (blk < 0) blk = (d.w - 1) / BS;
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb);
    bs_block_apply_block<NR>(b.Linv + b.linv_off[s] + (size_t)blk * BS * BS, a.xp + (d.col0 + kb) * NR, nb, transpose != 0,
                       b.side + (d.col0 + kb) * NR, sm, threadIdx.x);
}
template <int NR>
__global__ void __launch_bounds__(BS_NT) k_bs_head_block(BigSolveArgs b, const int32_t* __restrict__ list, int blk, int transpose) {
    extern __shared__ double smd[];
    bs_head<NR>(b, list, blk, transpose, smd);
}

template <int NR>
__device__ __forceinline__ void bs_fwd(const BigSolveArgs& b, const int32_t* __restrict__ list, int blk, double* sm) {
    const SolveArgs& a = b.s;                                      // sm: y_b | partial sums
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb), f = d.f, tid = threadIdx.x;
    const int row0 = kb + nb + blockIdx.x * BSF_ROWS;
    if (row0 >= f) return;
    if (tid < BS) {
#pragma unroll
        for (int q = 0; q < NR; ++q) sm[q * BS + tid] = (tid < nb) ? b.side[(d.col0 + kb + tid) * NR + q] : 0.0;
    }
    const int ir = tid & (BSF_ROWS - 1), g = tid >> 7;
    const int i = row0 + ir;
    double v[16];
    {
        const double* col = a.L + d.lp_off + (size_t)(kb + g * 16) * f + min(i, f - 1);
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = (i < f && g * 16 + k < nb) ? col[(size_t)k * f] : 0.0;
    }
    __syncthreads();
    double* part = sm + NR * BS;
#pragma unroll
    for (int q = 0; q < NR; ++q) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 16; ++k) acc = fma(v[k], sm[q * BS + g * 16 + k], acc);
        part[q * BS_NT + tid] = acc;
    }
    __syncthreads();
    if (g == 0 && i < f) {
        double* y = yptr_block<NR>(a, d, a.cbv_off[s], i);
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            double tot = 0.0;
#pragma unroll
            for (int kg = 0; kg < BS_KG; ++kg) tot += part[q * BS_NT + kg * BS + ir];
            y[q] -= tot;
        }
    }
    // the rows of this CTA are the pivots of the next block: its right-hand side is final now
    if (blockIdx.x == 0 && kb + BS < d.w)
        bs_block_apply_block<NR>(b.Linv + b.linv_off[s] + (size_t)(blk + 1) * BS * BS, a.xp + (d.col0 + kb + BS) * NR, min(BS, d.w - kb - BS),
                           false, b.side + (d.col0 + kb + BS) * NR, sm, tid);
}
template <int NR>
__global__ void __launch_bounds__(BS_NT) k_bs_fwd_block(BigSolveArgs b, const int32_t* __restrict__ list, int blk) {
    extern __shared__ double smd[];
    bs_fwd<NR>(b, list, blk, smd);
}

// ---- backward init: t_j = y_j / d_j - sum_{i >= w} L(i,j) x(rows_i)  (y_j parked in `side` by the forward sweep);
//      one warp per pivot column (lanes stride the rows: coalesced stream of the column), grid (ceil(w/8), nfronts)
template <int NR>
__device__ __forceinline__ void bs_bwd_init(const BigSolveArgs& b, const int32_t* __restrict__ list) {
    const SolveArgs& a = b.s;
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= d.w) return;
    const int f = d.f;
    const double* __restrict__ col = a.L + d.lp_off + (size_t)j * f;
    const int32_t* __restrict__ rows = a.rows + d.rows_off;
    double acc[NR];
#pragma unroll
    for (int q = 0; q < NR; ++q) acc[q] = 0.0;
    int i = d.w + lane;
    for (; i + 96 < f; i += 128) {
        double l[4], x[4][NR];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            l[u] = col[i + 32 * u];
            const double* xr = a.xp + rows[i + 32 * u] * NR;
#pragma unroll
            for (int q = 0; q < NR; ++q) x[u][q] = xr[q];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int q = 0; q < NR; ++q) acc[q] = fma(l[u], x[u][q], acc[q]);
    }
    for (; i < f; i += 32) {
        const double* xr = a.xp + rows[i] * NR;
#pragma unroll
        for (int q = 0; q < NR; ++q) acc[q] = fma(col[i], xr[q], acc[q]);
    }
#pragma unroll
    for (int q = 0; q < NR; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < NR; ++q) a.xp[(d.col0 + j) * NR + q] = b.side[(d.col0 + j) * NR + q] / a.dvec[d.col0 + j] - acc[q];
    }
}
template <int NR>
__global__ void __launch_bounds__(256) k_bs_bwd_init_block(BigSolveArgs b, const int32_t* __restrict__ list) { bs_bwd_init<NR>(b, list); }

template <int NR>
__device__ __forceinline__ void bs_bwd(const BigSolveArgs& b, const int32_t* __restrict__ list, int blk, double* sm) {
    const SolveArgs& a = b.s;                                      // sm: x_b
    const int s = list[blockIdx.y];
    const FrontDesc d = a.desc[s];
    const int kb = blk * BS;
    if (kb >= d.w) return;
    const int nb = min(BS, d.w - kb), f = d.f, tid = threadIdx.x;
    const int t = blockIdx.x;                                      // block of columns served by this CTA, t < blk
    if (t >= blk) return;
    if (tid < BS) {
#pragma unroll
        for (int q = 0; q < NR; ++q) sm[q * BS + tid] = (tid < nb) ? b.side[(d.col0 + kb + tid) * NR + q] : 0.0;
    }
    const int warp = tid >> 5, lane = tid & 31;                   // 32 warps x 4 columns: rows [kb, kb+nb) of a column are contiguous
    double v[4][4];
#pragma unroll
    for (int cq = 0; cq < 4; ++cq) {
        const double* col = a.L + d.lp_off + (size_t)(t * BS + warp * 4 + cq) * f + kb;
#pragma unroll
        for (int u = 0; u < 4; ++u) v[cq][u] = (lane + 32 * u < nb) ? col[lane + 32 * u] : 0.0;
    }
    __syncthreads();
#pragma unroll 1
    for (int q = 0; q < NR; ++q) {                                // (one column at a time: 64 registers at 1024 threads)
#pragma unroll
        for (int cq = 0; cq < 4; ++cq) {
            double acc = 0.0;
#pragma unroll
            for (int u = 0; u < 4; ++u) acc = fma(v[cq][u], sm[q * BS + lane + 32 * u], acc);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) a.xp[(d.col0 + t * BS + warp * 4 + cq) * NR + q] -= acc;
        }
    }
    // block blk-1 has received its last update: form x_{blk-1} for the next launch
    if (t == blk - 1)
        bs_block_apply_block<NR>(b.Linv + b.linv_off[s] + (size_t)t * BS * BS, a.xp + (d.col0 + t * BS) * NR, BS, true,
                           b.side + (d.col0 + t * BS) * NR, sm, tid);
}
template <int NR>
__global__ void __launch_bounds__(BS_NT) k_bs_bwd_block(BigSolveArgs b, const int32_t* __restrict__ list, int blk) {
    extern __shared__ double smd[];
    bs_bwd<NR>(b, list, blk, smd);
}

// ---- end of a front's backward sweep: solved pivots from `side` back into xp; grid (ceil(w/256), nfronts)
template <int NR>
__device__ __forceinline__ void bs_bwd_finish(const BigSolveArgs& b, const int32_t* __restrict__ list) {
    const FrontDesc d = b.s.desc[list[blockIdx.y]];
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j < d.w) {
#pragma unroll
        for (int q = 0; q < NR; ++q) b.s.xp[(d.col0 + j) * NR + q] = b.side[(d.col0 + j) * NR + q];
    }
}
template <int NR>
__global__ void __launch_bounds__(256) k_bs_bwd_finish_block(BigSolveArgs b, const int32_t* __restrict__ list) { bs_bwd_finish<NR>(b, list); }

}  // namespace b2
