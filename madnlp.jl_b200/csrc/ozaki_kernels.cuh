// Ozaki-scheme fp64 SYRK on the Hopper tensor cores: W = A' A with A (K x n) cut into S = 8 signed 7-bit digits per entry, the
// 36 digit-pair products run as EXACT int8 GEMMs on wgmma.mma_async (s8 x s8 -> s32, accumulators in registers), operands staged
// by TMA (cp.async.bulk.tensor, 64-byte swizzle), fp64 reconstruction in the epilogue.  See tools/microbench/ozaki_syrk_wgmma.cu
// for the stand-alone measurement and DESIGN.md section 3 for the error analysis; used by b2d_condensed_assemble_ozaki
// (build_kkt!(::DenseCondensedKKTSystem), src/KKT/Dense/condensed.jl:157-186, in place of cuBLAS mul!(W, J', J)).
//
//   1. per column m:  e_m = exponent of max_i |a_im|;  x = a_im * 2^-e_m in (-1, 1) is cut into S = 8 signed 7-bit digits
//      x = sum_s q_s 2^(-7(s+1))   (q_s int8, exact: 56 bits cover the fp64 mantissa of the column's largest entries)
//   2. G_d = sum_{s+t=d} Q_s' Q_t  for d = 0..S-1 : 36 exact int8 x int8 -> int32 GEMMs (|G_d| <= 8 * K * 127^2 < 2^31 for
//      K <= 16384), the d-sums accumulate inside the wgmma accumulators
//   3. W(m,n) = 2^(e_m + e_n - 14) * sum_d 2^(-7d) G_d(m,n)   evaluated in fp64 (Horner) by the epilogue
//   A column holding a NaN or an Inf makes its row and column of W NaN (the fp64 contraction is non-finite there).
//   Error (DESIGN.md section 3, checked entry by entry in tests/test_dense_assembly_entrywise_oracle.py):
//   |W^ - W| <= 2^-51 ns 2^(e_m + e_n) before the final rounding -- truncation below 2^-56 of the column max (2^-55), the
//   dropped digit pairs s + t >= 8 (127^2 sum_{d>=8} (15 - d) 2^(-7(d+2)) = 2^-53.2) and the Horner sum (~2^-53), per term
//
// Kernel (one 64 x 64 output tile per CTA, 288 threads):
//   warp 8 lane 0 : TMA producer  -- the 8 A-digit tiles and 8 B-digit tiles of a 64-deep K block into a 3-stage ring
//   warps 0..7    : two consumer warpgroups; each owns 4 of the 8 accumulators G_d (4 x m64n64 s32 = 128 registers a thread:
//                   all 8 would not fit the register file), split so that both issue 18 digit pairs = 36 wgmma m64n64k32 per
//                   K block.  Epilogue: both park their accumulators in shared memory, then all 256 threads run the Horner
//                   sum over d, the scaling and coalesced column-major stores.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cfloat>
#include <cstdint>

#include "ptx.cuh"

namespace ozk {

constexpr int S = 8;             // digits
constexpr int WB = 7;            // bits per digit
constexpr int BM = 64, BN = 64;  // output tile
constexpr int BKB = 64;          // K bytes (= int8 elements) per pipeline stage: one 64-byte swizzle row
constexpr int STAGES = 3;
constexpr int A_TILE = BM * BKB, B_TILE = BN * BKB;                 // bytes of one digit tile
constexpr int STAGE_BYTES = S * (A_TILE + B_TILE);                  // 64 KiB
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;             // + alignment slack
constexpr int NTHREADS = 288;
constexpr int GLD = BM + 4;                                         // int32 row stride of the parked accumulators (no bank conflicts)
static_assert(S * BN * GLD * 4 <= STAGES * STAGE_BYTES, "the parked accumulators reuse the operand ring");
constexpr uint32_t SPIN_MAX = 1u << 22;                             // tries of a bounded mbarrier wait

// ------------------------------------------------------------------------------------------------ digit split
// expo[m] of a column that holds a NaN or an Inf: the epilogue writes NaN wherever row m or column m of W is read, as the fp64
// contraction would give a non-finite value there (frexp exponents of finite doubles lie in [-1073, 1024])
constexpr int EXPO_NONFINITE = 1 << 20;

// one CTA per column m of the operand A (K x M): a(i, m) = (scale ? sqrt(scale[i]) : 1) * src[m*lds + (rows ? rows[i] : i)];
// exponent of the column, then S int8 digits per element into Q[s][m][i] (row length Kpad, rows beyond K stay zero)
__global__ void __launch_bounds__(256) k_ozaki_split(int K, int Kpad, int Mpad, const double* __restrict__ src, int64_t lds,
                                                     const int64_t* __restrict__ rows, const double* __restrict__ scale,
                                                     int8_t* __restrict__ Q, int* __restrict__ expo) {
    const int m = blockIdx.x;
    const double* col = src + (size_t)m * lds;
    __shared__ double red[256];
    double mx = 0.0;
    int bad = 0;
    for (int i = threadIdx.x; i < K; i += 256) {
        const double a = fabs(col[rows ? rows[i] : i] * (scale ? sqrt(scale[i]) : 1.0));
        mx = fmax(mx, a);                           // (fmax drops a NaN: the flag catches it)
        bad |= !(a <= DBL_MAX);
    }
    red[threadIdx.x] = mx;
    bad = __syncthreads_or(bad);
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]); __syncthreads(); }
    mx = red[0];
    int e = 0;
    if (bad) e = EXPO_NONFINITE;
    else if (mx > 0.0) frexp(mx, &e);               // mx = f * 2^e, f in [0.5, 1)  ->  |a| * 2^-e < 1 (subnormal mx included)
    if (threadIdx.x == 0) expo[m] = e;
    for (int i = threadIdx.x; i < K; i += 256) {
        double x = bad ? 0.0 : ldexp(col[rows ? rows[i] : i] * (scale ? sqrt(scale[i]) : 1.0), -e);    // exact scaling
#pragma unroll
        for (int s = 0; s < S; ++s) {
            x *= (double)(1 << WB);                 // exact
            const double q = trunc(x);              // |q| <= 127
            Q[((size_t)s * Mpad + m) * Kpad + i] = (int8_t)(int)q;
            x -= q;                                 // exact
        }
    }
}

// ------------------------------------------------------------------------------------------------ PTX helpers
// (mbarriers, the shared-window address and the named barrier: ptx.cuh)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, unsigned long long* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(b2::smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(b2::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// wgmma shared-memory descriptor of a K-major operand tile with 64-byte swizzle: rows of 64 bytes, 8-row groups 512 bytes
// apart (stride byte offset), leading byte offset unused (1), layout type 2 = SWIZZLE_64B
__device__ __forceinline__ uint64_t gmma_desc_k_sw64(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;
    return d;
}
// D(64 x 64, s32) += A(64 x 32, s8, K-major) * B(32 x 64, s8, K-major), both operands from shared memory
__device__ __forceinline__ void wgmma_s8(int (&d)[32], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
          "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
          "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]),
          "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(adesc), "l"(bdesc));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// 2^e for -1022 <= e <= 1023 (exponent field only)
__device__ __forceinline__ double pow2i(int e) { return __longlong_as_double((long long)(e + 1023) << 52); }

// accumulators of consumer warpgroup G: {0, 1, 6, 7} and {2, 3, 4, 5} -- d has d + 1 digit pairs, 18 pairs each
__host__ __device__ constexpr int acc_digit(int G, int j) { return G == 0 ? (j < 2 ? j : j + 4) : j + 2; }

// one K block of warpgroup G: every digit pair (s, t = d - s) of its accumulators, two k32 steps each
template <int G>
__device__ __forceinline__ void mma_kblock(int (&acc)[4][32], uint64_t ad0, uint64_t bd0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int d = acc_digit(G, j);
#pragma unroll
        for (int s = 0; s <= d; ++s)
#pragma unroll
            for (int k2 = 0; k2 < BKB / 32; ++k2)
                wgmma_s8(acc[j], ad0 + (uint64_t)((s * A_TILE + k2 * 32) >> 4), bd0 + (uint64_t)(((d - s) * B_TILE + k2 * 32) >> 4));
    }
}

// ------------------------------------------------------------------------------------------------ the GEMM
// tile list: tiles[t] = (bm, bn) with bn <= bm (touches the lower triangle); A and B tiles are both boxes of the digit planes
// epilogue: C(m, n) = W(m, n) [+ hess(m, n)] [+ pr(m) on the diagonal] for m, n < nvalid (and m >= n when lower_only); ld = ldc / ldh
__global__ void __launch_bounds__(NTHREADS, 1) k_ozaki_syrk(const __grid_constant__ CUtensorMap mapQ, int K, int nvalid,
                                                            const int2* __restrict__ tiles, const int* __restrict__ expo,
                                                            double* __restrict__ C, int64_t ldc, const double* __restrict__ hess, int64_t ldh,
                                                            const double* __restrict__ pr, int lower_only, int* err) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    __shared__ unsigned long long full_bar[STAGES], empty_bar[STAGES];
    // warp index through a shuffle: the compiler then knows it is warp-uniform and does not serialise the wgmma sequence
    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int bm = tiles[blockIdx.x].x, bn = tiles[blockIdx.x].y;
    const int nkb = K / BKB;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { b2::mbar_init(&full_bar[s], 1); b2::mbar_init(&empty_bar[s], 2); }
        b2::mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ---------------- TMA producer
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int st = kb % STAGES;
                if (kb >= STAGES && !b2::mbar_wait_bounded<SPIN_MAX>(&empty_bar[st], ((kb / STAGES) - 1) & 1, err)) break;
                uint8_t* sa = smem + (size_t)st * STAGE_BYTES;
                uint8_t* sb = sa + S * A_TILE;
                b2::mbar_expect_tx(&full_bar[st], STAGE_BYTES);
                tma_load_3d(sa, &mapQ, &full_bar[st], kb * BKB, bm * BM, 0);      // box (64 B of K, 64 rows, 8 digits)
                tma_load_3d(sb, &mapQ, &full_bar[st], kb * BKB, bn * BN, 0);
            }
        }
        return;
    }

    // ---------------- consumers: warpgroup g = warp / 4
    const int g = warp >> 2;
    int acc[4][32];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0;
    bool ok = true;
    for (int kb = 0; kb < nkb; ++kb) {
        const int st = kb % STAGES;
        ok = __all_sync(0xffffffffu, b2::mbar_wait_bounded<SPIN_MAX>(&full_bar[st], (kb / STAGES) & 1, err));
        if (!ok) break;
        const uint32_t sa = b2::smem_u32(smem + (size_t)st * STAGE_BYTES);
        const uint64_t ad0 = gmma_desc_k_sw64(sa), bd0 = gmma_desc_k_sw64(sa + S * A_TILE);
        wgmma_fence();
        if (g == 0) mma_kblock<0>(acc, ad0, bd0);
        else mma_kblock<1>(acc, ad0, bd0);
        wgmma_commit();
        wgmma_wait_all();
        if ((threadIdx.x & 127) == 0) b2::mbar_arrive(&empty_bar[st]);    // this warpgroup has read the stage
    }
    wgmma_wait_all();

    // ---------------- epilogue: park G_d(m, n) at Gs[d][n][m] (over the operand ring, which every wgmma has finished reading)
    b2::bar_sync<1, 256>();                               // warps 0..7 only
    int32_t* Gs = reinterpret_cast<int32_t*>(smem);
    {
        const int w = warp & 3;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int32_t* Gd = Gs + (size_t)acc_digit(g, j) * BN * GLD;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int r = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);     // wgmma accumulator fragment: row, column
                const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
                Gd[c * GLD + r] = acc[j][i];
            }
        }
    }
    b2::bar_sync<1, 256>();                               // warps 0..7 only
    if (!ok) return;
    const int ml = threadIdx.x & (BM - 1);
    const int m = bm * BM + ml;
    const int em = expo[m];
#pragma unroll 4
    for (int nl = threadIdx.x >> 6; nl < BN; nl += 256 / BM) {
        const int n = bn * BN + nl;
        double h = 0.0;
#pragma unroll
        for (int d = S - 1; d >= 0; --d) h = fma(h, 1.0 / (1 << WB), (double)Gs[((size_t)d * BN + nl) * GLD + ml]);
        if (n < nvalid && m < nvalid && (!lower_only || m >= n)) {
            const int en = expo[n], E = em + en - 2 * WB;
            // h * 2^E rounded once (the bits of ldexp, without its branches), so W underflows and overflows where the fp64
            // contraction does: h = 0 or 2^-49 <= |h| < 2^29, so h * 2^A is exact, and the second product rounds
            const int A = min(max(E, -970), 990);
            double v = (h * pow2i(A)) * pow2i(min(max(E - A, -1022), 1023));
            if (em == EXPO_NONFINITE || en == EXPO_NONFINITE) v = __longlong_as_double(0x7ff8000000000000LL);
            if (hess) v += hess[(size_t)n * ldh + m];
            if (pr && m == n) v += pr[m];
            C[(size_t)n * ldc + m] = v;
        }
    }
}


}  // namespace ozk
