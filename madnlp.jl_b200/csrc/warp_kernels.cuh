// Latency-oriented kernels for small fronts (order f <= 64): ONE WARP PER FRONT.
//
// On AC-OPF-like KKT systems every front is tiny (<= ~50) and the factorisation holds only ~2e7 flops: wall time is
// the dependent-latency chain, not bandwidth or flops.  These kernels therefore
//   * keep a front private to one warp (shared memory slice + registers), so a pivot step costs one __syncwarp
//     instead of two __syncthreads;
//   * take the reciprocal of each pivot with rcp.approx + 2 Newton steps (the only division on the critical path);
//   * carry the triangular-solve recurrences through warp shuffles (chain per pivot: SHFL + DFMA) with the factor
//     entries prefetched from shared memory, independent of the recurrence;
//   * run through a STAGED schedule: a CTA owns a list of stages (local levels of an elimination subtree); its warps
//     sweep the fronts of a stage, __syncthreads(), next stage.  Whole bottom subtrees thus execute inside one
//     kernel launch; data handed from child to parent front travels through global memory (same SM, ordered by
//     the barrier), so no pointer in here is const/__restrict__ for buffers written by these kernels.
#pragma once
#include "common.cuh"
#include "front_kernels.cuh"
#include "ptx.cuh"
#include "solve_kernels.cuh"

namespace b2 {

constexpr int FW_WARPS = 4;

struct ChildRec {          // one per (parent, child) edge, contiguous per parent, ascending child id
    int64_t cb_off;        // child's update block in the workspace (ld = rc)
    int64_t rel_off;       // child's relative indices into the parent front
    int64_t cbv_off;       // child's contribution vector (solve)
    int32_t rc;            // order of the child's update block
    int32_t sn;
};
static_assert(sizeof(ChildRec) == 32, "ChildRec must be 32 bytes");

struct WarpSched {
    const int32_t* cta_ptr;     // [nCTA+1] stage ranges
    const int32_t* stage_off;   // [nstage] offset into list
    const int32_t* stage_cnt;   // [nstage]
    const int32_t* list;        // supernode ids
};

// ------------------------------------------------------------------------------------------------ factor
// A front is owned by a TEAM of NW warps (NW = 1: order <= 32, NW = 2: order <= 64; NW = 4: order <= 96, PAIRS only, whose pivot
// loop runs in shared memory); thread `tid` of the team owns
// ROW tid of the front and keeps it in registers as a sliding window: after pivot k, a[j] holds column k+1+j.
// Per pivot the only shared-memory traffic is the broadcast of the pivot column (double-buffered, one team barrier).
// Global loads are issued in independent batches (memory-level parallelism instead of one L2 round trip per element).
#define B2_STAMP(idx) do { if (prof) { team_sync<NW>(team); if (tid == 0) prof[idx] = clock64(); } } while (0)

template <int NW>
__device__ __forceinline__ void team_sync(int team) {
    if (NW == 1) __syncwarp();
    else asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "r"(NW * 32) : "memory");
}

// Split team barrier of the pivot loop (front_factor_team): every warp ARRIVES on its own named barrier and WAITS on its
// partner's, ids alternating with the pivot parity -- bar.arrive + bar.sync by disjoint warps, 64 threads per barrier.  A warp
// can only arrive for pivot k+2 after its partner has left the wait of pivot k, so two ids per warp are enough.
// ids: 1..2 = team_sync; 3 + team*4 + warp*2 + parity (<= 10 of the 16 hardware barriers).
template <int NW>
__device__ __forceinline__ void team_arrive(int team, int warp, int parity) {
    static_assert(NW <= 2, "split barrier is written for one- and two-warp teams");
    if (NW == 2) asm volatile("bar.arrive %0, 64;" ::"r"(3 + team * 4 + warp * 2 + parity) : "memory");
}
template <int NW>
__device__ __forceinline__ void team_wait(int team, int warp, int parity) {
    if (NW == 1) __syncwarp();
    else asm volatile("bar.sync %0, 64;" ::"r"(3 + team * 4 + (warp ^ 1) * 2 + parity) : "memory");
}

// shared-memory slice of one team:
//   F[maxf*maxf] assembly area, later the finished panel | colbuf[4][FMAX+4] | rel[MAXC][FMAX] ints | recs[MAXC] |
//   stage[STAGE] children's update blocks landed by cp.async
constexpr int MAXC = 8;                                // children staged per round
template <int NW>
struct TeamSmem {
    static constexpr int FMAX = 32 * NW;
    static constexpr int STAGE = (NW == 1) ? 1024 : 4096;   // doubles; one child always fits (rc^2 <= (FMAX-1)^2)
    static __host__ __device__ int fsize(int maxf) { return (maxf * maxf + 1) & ~1; }   // keeps `stage` 16-byte aligned
    // the four-warp class (PAIRS fronts of order 65..96) sizes its stage by its largest front: a child's block has rc <= f - 1 of its
    // parent, so one child still always fits, and a launch whose fronts stop at order 66 needs 78 KB instead of 156 KB
    static __host__ __device__ int stage(int maxf) { return NW <= 2 ? STAGE : fsize(maxf); }
    static __host__ __device__ int doubles(int maxf) {
        return fsize(maxf) + 4 * (FMAX + 4) + (MAXC * FMAX) / 2 + MAXC * 4 + stage(maxf);
    }
};

// dependency flags of the single-launch factorisation (k_factor_dep): zeroed before the launch, a flag is ready when it holds 1
// (stored with st_release by the front that finishes); a wait polls at most DEP_SPIN_MAX times, DEP_SPIN_SLEEP_NS apart
constexpr unsigned DEP_SPIN_MAX = 1u << 24, DEP_SPIN_SLEEP_NS = 32;

// Hand-off slots of the single-launch solve: the value is its own flag.  A slot holds SLOT_EMPTY (ptx.cuh) until its one producer
// stores the value; its one consumer polls the value itself (no flag, no release fence, one L2 round trip per hand-off) and stores
// SLOT_EMPTY back once it has it, which arms the slot for the next launch.
__device__ __forceinline__ void slot_put(double* p, double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    st_relaxed_b64(p, b == SLOT_EMPTY ? CANON_NAN : b);
}
// take the slots p[c] with bit c of `need` set: poll them all at once until none is empty, then re-arm each.  Bounded like the flag polls:
// a slot still empty at the time-out sets *err (the solve then writes NaN into x) and reads as NaN.
template <int K>
__device__ __forceinline__ void slot_take(double* const (&p)[K], unsigned need, double (&v)[K], int* err) {
    unsigned long long b[K];
#pragma unroll
    for (int c = 0; c < K; ++c) b[c] = (need >> c & 1u) ? ld_relaxed_b64(p[c]) : 0ull;
    unsigned it = 0;
    for (;;) {
        unsigned pend = 0;
#pragma unroll
        for (int c = 0; c < K; ++c) pend |= ((need >> c & 1u) && b[c] == SLOT_EMPTY) ? 1u << c : 0u;
        if (!pend) break;
        if (++it >= DEP_SPIN_MAX) {          // never hang the device, report instead
            atomicExch(err, 1);
            break;
        }
        __nanosleep(DEP_SPIN_SLEEP_NS);
#pragma unroll
        for (int c = 0; c < K; ++c) if (pend >> c & 1u) b[c] = ld_relaxed_b64(p[c]);
    }
#pragma unroll
    for (int c = 0; c < K; ++c) {
        v[c] = __longlong_as_double((long long)b[c]);
        if ((need >> c & 1u) && b[c] != SLOT_EMPTY) st_relaxed_b64(p[c], SLOT_EMPTY);
    }
}

// Block hand-offs of the single-launch solve with NR right-hand sides (k_solve_dep_block): a slot index owns NR consecutive words,
// word c for column c, and each word keeps the rule above -- the producer never stores SLOT_EMPTY, the consumer polls the words
// themselves.  A consumer accepts a slot once none of its NR words is SLOT_EMPTY and then re-arms all of them.  NR = 1 is slot_put /
// slot_take.
template <int NR>
__device__ __forceinline__ void slot_put_block(double* p, const double (&v)[NR]) {
    if constexpr (NR == 1) {
        slot_put(p, v[0]);
    } else {
        static_assert(NR % 2 == 0, "block slots are accessed in 16-byte pairs");
        unsigned long long b[NR];
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            b[q] = (unsigned long long)__double_as_longlong(v[q]);
            b[q] = b[q] == SLOT_EMPTY ? CANON_NAN : b[q];
        }
#pragma unroll
        for (int q = 0; q < NR; q += 2) st_relaxed_v2_b64(p + q, b[q], b[q + 1]);
    }
}
// slot_take over K block slots: a slot still incomplete at the time-out reads as NaN where it is empty and is not re-armed here (the
// launch's time-out path re-arms every slot once all its CTAs are done)
template <int K, int NR>
__device__ __forceinline__ void slot_take_block(double* const (&p)[K], unsigned need, double (&v)[K][NR], int* err) {
    if constexpr (NR == 1) {
        double u[K];
        slot_take(p, need, u, err);
#pragma unroll
        for (int c = 0; c < K; ++c) v[c][0] = u[c];
    } else {
        static_assert(NR % 2 == 0, "block slots are accessed in 16-byte pairs");
        unsigned long long b[K][NR];
#pragma unroll
        for (int c = 0; c < K; ++c)
#pragma unroll
            for (int q = 0; q < NR; q += 2) {
                if (need >> c & 1u) ld_relaxed_v2_b64(p[c] + q, b[c][q], b[c][q + 1]);
                else b[c][q] = b[c][q + 1] = 0ull;
            }
        unsigned it = 0, pend;
        for (;;) {
            pend = 0;
#pragma unroll
            for (int c = 0; c < K; ++c) {
                bool empty = false;
#pragma unroll
                for (int q = 0; q < NR; ++q) empty |= b[c][q] == SLOT_EMPTY;
                pend |= ((need >> c & 1u) && empty) ? 1u << c : 0u;
            }
            if (!pend) break;
            if (++it >= DEP_SPIN_MAX) {
                atomicExch(err, 1);
                break;
            }
            __nanosleep(DEP_SPIN_SLEEP_NS);
#pragma unroll
            for (int c = 0; c < K; ++c)
                if (pend >> c & 1u)
#pragma unroll
                    for (int q = 0; q < NR; q += 2) ld_relaxed_v2_b64(p[c] + q, b[c][q], b[c][q + 1]);
        }
#pragma unroll
        for (int c = 0; c < K; ++c) {
#pragma unroll
            for (int q = 0; q < NR; ++q) v[c][q] = __longlong_as_double((long long)b[c][q]);
            if ((need >> c & 1u) && !(pend >> c & 1u))
#pragma unroll
                for (int q = 0; q < NR; q += 2) st_relaxed_v2_b64(p[c] + q, SLOT_EMPTY, SLOT_EMPTY);
        }
    }
}

// One pivot of front_factor_team's software-pipelined loop, for a window of NB live 8-column blocks: the latency chain of pivot k
// (d_k -> reciprocal (approx + 2 Newton steps) -> l_k -> column k+1 -> publish -> arrive) and the pending row update of pivot k-1,
// as one branch-free block.  The publish is a predicated st.shared + bar.arrive in ONE asm without a memory clobber, so that most
// of the pending update (which reads the OTHER column buffers) follows the arrive and overlaps the partner warp's barrier latency.
// The empty volatile asm statements (B2_TIE) keep NVVM from sinking the whole chain below the update; ptxas then issues the six tied
// FMA pairs under the latency of the d_k load and runs the chain contiguously.  (Measured: forcing a
// finer interleave with real data dependencies -- one LOP3 per link -- costs more issue slots than the latency it hides.)
struct PivotCtx { const double* cb; const double* pb; double* nb; double* Fk; double eps; int tid, k, f, team; };
#define B2_TIE(c, x, y) asm volatile("" : "+d"(c), "+d"(x), "+d"(y))
template <int NW, int P>
__device__ __forceinline__ void pending_pair(double (&av)[32 * NW + 1], double lp, const double2* up) {
    const double2 u = up[P];
    av[2 * P - 1] = fma(-lp, u.x, av[2 * P]);
    av[2 * P] = fma(-lp, u.y, av[2 * P + 1]);
}
template <int NW, int P0, int P1>
struct PendingRange {
    static __device__ __forceinline__ void run(double (&av)[32 * NW + 1], double lp, const double2* up) {
        if constexpr (P0 < P1) { pending_pair<NW, P0>(av, lp, up); PendingRange<NW, P0 + 1, P1>::run(av, lp, up); }
    }
};
template <int NW, int NB>
__device__ __forceinline__ void pivot_iter(double (&av)[32 * NW + 1], double& lp, const PivotCtx& c, int& nneg, int& npert) {
    constexpr int NP = 4 * NB;                          // pending pairs 1 .. NP-1 (pair 0 is column k+1, handled with the chain)
    double dk = c.cb[1];
    const double u0 = c.cb[2];
    const double2* up = reinterpret_cast<const double2*>(c.pb + 2);
    const bool tiny = !(fabs(dk) >= c.eps), neg = dk < 0.0;
    dk = tiny ? (neg ? -c.eps : c.eps) : dk;
    npert += (c.tid == 0 && tiny) ? 1 : 0;
    nneg += (c.tid == 0 && !tiny && neg) ? 1 : 0;
    double a1 = fma(-lp, up[0].y, av[1]);               // column k+1 with pivot k-1 applied
    double r, e;
    asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(dk));
    if constexpr (NP > 1) { pending_pair<NW, 1>(av, lp, up); B2_TIE(r, av[1], av[2]); }
    e = fma(-dk, r, 1.0);
    if constexpr (NP > 2) { pending_pair<NW, 2>(av, lp, up); B2_TIE(e, av[3], av[4]); }
    r = fma(r, e, r);
    if constexpr (NP > 3) { pending_pair<NW, 3>(av, lp, up); B2_TIE(r, av[5], av[6]); }
    e = fma(-dk, r, 1.0);
    if constexpr (NP > 4) { pending_pair<NW, 4>(av, lp, up); B2_TIE(e, av[7], av[8]); }
    r = fma(r, e, r);
    if constexpr (NP > 5) { pending_pair<NW, 5>(av, lp, up); B2_TIE(r, av[9], av[10]); }
    double l = av[0] * r;
    if constexpr (NP > 6) { pending_pair<NW, 6>(av, lp, up); B2_TIE(l, av[11], av[12]); }
    // column k+1 with pivot k applied -- the value the next pivot waits for (junk, unused, when k+1 = f)
    double nx = fma(-l, u0, a1);
    double* dst = c.nb + (c.tid - c.k);                // row tid of column k+1 at nb[tid - (k+1) + 1]
    if (NW == 1) {
        if (c.tid > c.k) *dst = nx;
    } else {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.gt.s32 p, %2, %3;\n\t@p st.shared.f64 [%0], %1;\n\tbar.arrive %4, 64;\n\t}"
                     ::"r"(smem_u32(dst)), "d"(nx), "r"(c.tid), "r"(c.k),
                       "r"(3 + c.team * 4 + (c.tid >> 5) * 2 + ((c.k + 1) & 1)));
    }
    if (c.tid < c.f) c.Fk[c.tid] = (c.tid == c.k) ? dk : l;   // finished column k of the panel (rows < k: scratch)
    av[0] = nx;
    PendingRange<NW, 7, NP>::run(av, lp, up);
    lp = l;
}

// B2_SPARSE_PIVOT_PAIRS (DESIGN.md section 3): bit j of the 128-bit mask[2s] | mask[2s+1] << 64 marks a candidate 2 x 2 pivot (j, j+1)
// of front s; the factorisation writes each pivot's kind (B2_PIVOT_*) and D's subdiagonal (b at the first index of a 2 x 2 block,
// else 0), permuted order
struct PairArgs {
    const unsigned long long* mask = nullptr;
    double* dsub = nullptr;
    int8_t* kind = nullptr;
};
constexpr double PAIR_ALPHA = 0.6403882032022076;    // (1 + sqrt(17)) / 8, Bunch-Kaufman's growth bound

template <int NW, bool DEP = false, bool PAIRS = false>
__device__ __forceinline__ void front_factor_team(const FactorArgs& a, const ChildRec* childrec, int s, double* sm_team,
                                                  int tid, int team, int maxf, int& nneg, int& npert, long long* prof = nullptr,
                                                  int* done = nullptr, int* err = nullptr, PairArgs pa = PairArgs()) {
    static_assert(NW <= 2 || (DEP && PAIRS), "the four-warp class runs the single-launch PAIRS factorisation only");
    constexpr int FMAX = 32 * NW, TEAM = 32 * NW;
    const int STAGE = TeamSmem<NW>::stage(maxf);
    double* F = sm_team;
    constexpr int CBS = FMAX + 4;                      // four pivot-column buffers
    double* colbuf = F + TeamSmem<NW>::fsize(maxf);    // [4][CBS]
    int* relst = (int*)(colbuf + 4 * CBS);             // [MAXC][FMAX]
    ChildRec* recs = (ChildRec*)(relst + MAXC * FMAX); // [MAXC]
    double* stage = (double*)(recs + MAXC);            // [STAGE]
    B2_STAMP(0);
    if (a.ftrace && tid == 0) a.ftrace[3 * (size_t)s] = global_ns();
    const FrontDesc d = a.desc[s];
    const int f = d.f, w = d.w, r = f - w;
    B2_STAMP(1);
    for (int i = tid; i < f * f; i += TEAM) F[i] = 0.0;
    for (int i = tid; i < 4 * CBS; i += TEAM) colbuf[i] = 0.0;
    team_sync<NW>(team);
    B2_STAMP(2);
    {   // original matrix entries: panel layout pos + col*f == assembly-area layout
        const int32_t* src = a.amap_src + d.amap_off;
        const int32_t* dst = a.amap_dst + d.amap_off;
        for (int t0 = 0; t0 < d.amap_cnt; t0 += 4 * TEAM) {
            int sd[4], dd[4]; double v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int t = t0 + tid + u * TEAM;
                sd[u] = (t < d.amap_cnt) ? src[t] : -1;
                dd[u] = (t < d.amap_cnt) ? dst[t] : 0;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = (sd[u] >= 0) ? __ldg(a.A + sd[u]) : 0.0;
#pragma unroll
            for (int u = 0; u < 4; ++u) if (sd[u] >= 0) F[dd[u]] = v[u];
        }
    }
    team_sync<NW>(team);
    B2_STAMP(3);
    // ---- extend-add of the children (ascending id): rounds of <= MAXC children whose update blocks fit the stage;
    //      every block of a round is landed in shared memory by cp.async in ONE memory round trip.
    // Dependency-driven schedule: the children are still added in ascending id (the summation order is part of the result), but a
    // round does not wait for all of them -- it waits for the next child and takes along those behind it that have ALREADY finished,
    // so a parent whose last child is late has staged and added the others by then (the tree's critical path pays one round, not
    // the whole extend-add: tools/trace_sparse.py).
    int* nready_sh = relst + FMAX - 1;                 // (row 0 of relst holds at most FMAX - 1 indices: this slot is free)
    for (int c0 = 0; c0 < d.nchild;) {
        const int cb0 = (c0 / MAXC) * MAXC;            // children are fetched in blocks of MAXC records
        const int ro = c0 - cb0;                       // first record of this round inside the block
        if (ro == 0) {
            if (tid < min(MAXC, d.nchild - cb0)) recs[tid] = childrec[d.child_off + cb0 + tid];
            team_sync<NW>(team);
        }
        int nrec = min(MAXC, d.nchild - cb0) - ro;
        if (DEP) {
            if (tid < 32) {
                // lane c polls child ro + c's flag: the round starts once child ro has finished (its update block is in L2) and
                // takes along the finished prefix behind it, read in the same poll -- no second, dependent round trip for the
                // children behind the one it waited for
                const int* fl = done + recs[ro + (tid < nrec ? tid : 0)].sn;
                unsigned m, it = 0;
                for (;;) {
                    const int v = (tid < nrec) ? ld_acquire(fl) : 0;
                    m = __ballot_sync(0xffffffffu, v != 0);
                    if (m & 1u) break;
                    if (++it >= DEP_SPIN_MAX) {                              // never hang the device, report instead
                        if (tid == 0) atomicExch(err, 1);
                        __threadfence();
                        m = 1u;
                        break;
                    }
                    __nanosleep(DEP_SPIN_SLEEP_NS);
                }
                if (tid == 0) *nready_sh = __ffs(~m) - 1;                  // length of the finished prefix (>= 1)
            }
            team_sync<NW>(team);
            nrec = *nready_sh;
        }
        const ChildRec* rrec = recs + ro;
        int nc = 0, tot = 0;
        while (nc < nrec) {
            const int sz = (rrec[nc].rc * rrec[nc].rc + 1) & ~1;
            if (nc > 0 && tot + sz > STAGE) break;
            tot += sz; ++nc;
        }
        int off = 0;
        for (int c = 0; c < nc; ++c) {
            const int rc = rrec[c].rc;
            const double* CB = a.ws + rrec[c].cb_off;          // 16-byte aligned, padded to an even count
            const int sz = (rc * rc + 1) & ~1;
            if (DEP) { for (int e = 2 * tid; e < sz; e += 2 * TEAM) cp_async16_cg(stage + off + e, CB + e); }
            else { for (int e = tid; e < rc * rc; e += TEAM) cp_async8(stage + off + e, CB + e); }
            if (tid < rc) cp_async4(relst + c * FMAX + tid, a.rel + rrec[c].rel_off + tid);
            off += sz;
        }
        cp_async_wait_all();
        team_sync<NW>(team);
        off = 0;
        for (int c = 0; c < nc; ++c) {
            const int rc = rrec[c].rc;
            const int* rl = relst + c * FMAX;
            const double* cs = stage + off;
            if (tid < rc) {
                const int ri = rl[tid];
                for (int j0 = 0; j0 <= tid; j0 += 8) {         // row tid of the child block, 8 columns per batch
                    double v[8], g[8]; int ix[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int j = j0 + u; ix[u] = (j <= tid) ? ri + rl[j] * f : -1; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int j = j0 + u; v[u] = (ix[u] >= 0) ? cs[j * rc + tid] : 0.0; g[u] = (ix[u] >= 0) ? F[ix[u]] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) if (ix[u] >= 0) F[ix[u]] = g[u] + v[u];
                }
            }
            team_sync<NW>(team);
            off += (rc * rc + 1) & ~1;
        }
        c0 += nc;
    }
    B2_STAMP(4);
    if (a.ftrace && tid == 0) a.ftrace[3 * (size_t)s + 1] = global_ns();
    double av[NW <= 2 ? FMAX + 1 : 1];                 // (four warps: a row of up to 96 doubles would spill; it stays in F)
    if constexpr (PAIRS) {
        // Pivots with candidate 2 x 2 blocks, right-looking in shared memory (thread = row): pivot k's column (and k+1's for a block)
        // is snapshotted in colbuf, then every row below updates itself.  Rule at a candidate pair with a = F(k,k), b = F(k+1,k),
        // c = F(k+1,k+1): a 2 x 2 block when |a| < alpha |b| and d1 = (a / |b|) c - |b| < 0 (indefinite: one negative and one
        // positive eigenvalue, the count of the reference's num_neg_ev, never perturbed); otherwise k is a 1 x 1 pivot (perturbed to
        // +-eps when |a| < eps, as the static path does) and k+1 an ordinary one.  The multipliers of a block are dsytf2's.
        const unsigned long long pm = pa.mask[2 * s], pm_hi = (NW > 2) ? pa.mask[2 * s + 1] : 0ull;
        double* u1 = colbuf;
        double* u2 = colbuf + CBS;
        for (int k = 0; k < w;) {
            team_sync<NW>(team);
            const double av_ = F[k + k * f];
            bool two = false;
            double b_ = 0.0, c_ = 0.0;
            if (((NW <= 2 || k < 64) ? pm >> k : pm_hi >> (k - 64)) & 1ull) {
                b_ = F[k + 1 + k * f];
                c_ = F[(k + 1) * (f + 1)];
                const double t = fabs(b_);
                two = fabs(av_) < PAIR_ALPHA * t && (av_ / t) * c_ - t < 0.0;
            }
            if (!two) {
                const bool tiny = !(fabs(av_) >= a.eps), neg = av_ < 0.0;
                const double dk = tiny ? (neg ? -a.eps : a.eps) : av_;
                npert += (tid == 0 && tiny) ? 1 : 0;
                nneg += (tid == 0 && !tiny && neg) ? 1 : 0;
                if (tid > k && tid < f) u1[tid] = F[tid + k * f];
                team_sync<NW>(team);
                if (tid > k && tid < f) {
                    const double l = u1[tid] / dk;
                    for (int j = k + 1; j <= tid; ++j) F[tid + j * f] = fma(-l, u1[j], F[tid + j * f]);
                    F[tid + k * f] = l;
                }
                if (tid == 0) {
                    F[k + k * f] = dk;
                    pa.kind[d.col0 + k] = tiny ? 1 : 0;
                    pa.dsub[d.col0 + k] = 0.0;
                }
                k += 1;
            } else {
                nneg += (tid == 0) ? 1 : 0;
                if (tid > k + 1 && tid < f) { u1[tid] = F[tid + k * f]; u2[tid] = F[tid + (k + 1) * f]; }
                team_sync<NW>(team);
                if (tid > k + 1 && tid < f) {
                    const double d11 = c_ / b_, d22 = av_ / b_, t = 1.0 / (d11 * d22 - 1.0), d21 = t / b_;
                    const double x1 = u1[tid], x2 = u2[tid];
                    const double l1 = d21 * (d11 * x1 - x2), l2 = d21 * (d22 * x2 - x1);
                    for (int j = k + 2; j <= tid; ++j) F[tid + j * f] = fma(-l2, u2[j], fma(-l1, u1[j], F[tid + j * f]));
                    F[tid + k * f] = l1;
                    F[tid + (k + 1) * f] = l2;
                }
                if (tid == 0) {
                    F[k + 1 + k * f] = 0.0;                // L11(k+1, k) of a block; D keeps a, b, c
                    pa.kind[d.col0 + k] = 2;
                    pa.kind[d.col0 + k + 1] = 3;
                    pa.dsub[d.col0 + k] = b_;
                    pa.dsub[d.col0 + k + 1] = 0.0;
                }
                k += 2;
            }
        }
        team_sync<NW>(team);
        if constexpr (NW <= 2) {
#pragma unroll
            for (int j = 0; j < FMAX; ++j) av[j] = (w + j < f && tid < f) ? F[tid + (w + j) * f] : 0.0;
        }
    } else {
    // row `tid` of the front into registers: a[j] = F(tid, j)
#pragma unroll
    for (int j = 0; j < FMAX; ++j) av[j] = (j < f && tid < f) ? F[tid + j * f] : 0.0;
    av[FMAX] = 0.0;
    // Pivot loop, software-pipelined by one pivot.  The pivot column is published WINDOW-RELATIVE in one of four buffers --
    // cb[1] = d_k, cb[2 + j] = u(k+1+j) -- so that the register window lines up with 16-byte pairs whatever the parity of k: one
    // LDS.128 feeds two FMAs (shared-memory issue, not the FP64 pipe, bounds a lone warp: tools/microbench/fp64_pipes.cu).
    // A pivot has a latency chain (barrier -> d_k -> reciprocal -> l_k -> the one FMA that makes column k+1 -> publish) and a
    // throughput part (the other f-k-2 FMAs of the row).  Iteration k runs the chain of pivot k TOGETHER with the throughput
    // part of pivot k-1 (`pending`: multiplier lp, buffer pb), as straight-line code per number of live 8-column blocks so that
    // ptxas interleaves the two; the team barrier is split (arrive after the publish, wait at the top of the next iteration).
    // Every element still receives the pivots' updates in ascending order, one fma each: bit-identical to the plain loop.
    //   top of iteration k:  av[0] = column k (final), av[j] = column k+j with pivot k-1's update pending (j >= 1)
    //   four buffers: a warp past wait(k) reads (k-1)%4 and k%4 and writes (k+1)%4; its partner, at most one pivot ahead (it has
    //   this warp's arrive(k+1) but not arrive(k+2)), writes (k+2)%4.
    colbuf[tid + 1] = av[0];                           // column 0
    team_arrive<NW>(team, tid >> 5, 0);
    double lp = 0.0;                                   // multiplier of the pending pivot (none yet: the pass only shifts)
    int kb = 0, pbi = 3;
    for (int k = 0; k < w; ++k) {
        const double* cb = colbuf + kb * CBS;
        const double* pb = colbuf + pbi * CBS;
        pbi = kb;
        kb = (kb + 1) & 3;
        double* nb = colbuf + kb * CBS;
        double* Fk = F + k * f;
        const int nblk = (f - k + 7) >> 3;              // live 8-column blocks of the window (team-uniform, >= 1)
        team_wait<NW>(team, tid >> 5, k & 1);
        PivotCtx c{cb, pb, nb, Fk, a.eps, tid, k, f, team};
        switch (nblk) {
            case 1: pivot_iter<NW, 1>(av, lp, c, nneg, npert); break;
            case 2: pivot_iter<NW, 2>(av, lp, c, nneg, npert); break;
            case 3: pivot_iter<NW, 3>(av, lp, c, nneg, npert); break;
            case 4: pivot_iter<NW, 4>(av, lp, c, nneg, npert); break;
            case 5: pivot_iter<NW, (NW > 1 ? 5 : 4)>(av, lp, c, nneg, npert); break;
            case 6: pivot_iter<NW, (NW > 1 ? 6 : 4)>(av, lp, c, nneg, npert); break;
            case 7: pivot_iter<NW, (NW > 1 ? 7 : 4)>(av, lp, c, nneg, npert); break;
            default: pivot_iter<NW, (NW > 1 ? 8 : 4)>(av, lp, c, nneg, npert); break;
        }
    }
    team_wait<NW>(team, tid >> 5, w & 1);              // pairs with the last iteration's (unconditional) arrive
    {   // the last pivot's pending update (no shift): av[j] = column w+j, j >= 1; av[0] = column w is final
        const double2* up = reinterpret_cast<const double2*>(colbuf + pbi * CBS + 2);
        av[1] = fma(-lp, up[0].y, av[1]);
#pragma unroll
        for (int j0 = 0; j0 < FMAX; j0 += 8) {
            if (w + j0 < f) {
#pragma unroll
                for (int j = (j0 ? j0 : 2); j < j0 + 8; j += 2) {
                    const double2 u = up[j >> 1];
                    av[j] = fma(-lp, u.x, av[j]);
                    av[j + 1] = fma(-lp, u.y, av[j + 1]);
                }
            }
        }
    }
    }   // !PAIRS
    B2_STAMP(5);
    // update block first (it is all the parent waits for): av[j] holds column w+j of row tid -- registers only, no barrier needed
    // (four warps: straight from row tid of F, which only thread tid has written since the pivot loop's last barrier)
    if (tid >= w && tid < f) {
        double* CBo = a.ws + d.cb_off;
        const int ir = tid - w;
        if constexpr (NW <= 2) {
#pragma unroll
            for (int j = 0; j < FMAX; ++j) if (j <= ir) CBo[(size_t)j * r + ir] = av[j];
        } else {
            for (int j = 0; j <= ir; ++j) CBo[(size_t)j * r + ir] = F[tid + (w + j) * f];
        }
    }
    // hand-off: the team barrier orders every thread's stores before thread 0's st.release.gpu (release is cumulative over the
    // barrier's synchronises-with edge -- the CUTLASS semaphore pattern), so no team-wide __threadfence() is needed.  The same
    // barrier completes the pivot loop's writes of the panel columns into F.
    team_sync<NW>(team);
    if (DEP && tid == 0) st_release(done + s, 1);
    if (a.ftrace && tid == 0) a.ftrace[3 * (size_t)s + 2] = global_ns();
    B2_STAMP(6);
    // panel, off the tree's critical path: column-major (forward solve, parent-independent) and row-major copy (backward solve)
    {
        double* Lp = a.L + d.lp_off;
        for (int e = tid; e < f * w; e += TEAM) Lp[e] = F[e];
        if (tid < f) {
            double* Lt = a.Lt + d.lp_off + (size_t)tid * w;
            for (int k = 0; k < w; ++k) Lt[k] = F[tid + k * f];
        }
        if (tid < w) a.dvec[d.col0 + tid] = F[tid + tid * f];
    }
    team_sync<NW>(team);                               // (a team of the staged kernels reuses F for its next front)
    B2_STAMP(7);
}

// debug: re-factor ONE front with clock64() stamps at the phase boundaries (children's update blocks must be valid)
template <int NW>
__global__ void k_factor_team_profile(FactorArgs a, const ChildRec* childrec, int sn, int maxf, long long* prof, int reps) {
    extern __shared__ __align__(16) double sm[];
    int nneg = 0, npert = 0;
    for (int r = 0; r < reps; ++r) front_factor_team<NW>(a, childrec, sn, sm, threadIdx.x, 0, maxf, nneg, npert, prof + 8 * r);
}

// a team's pivot counts into the factorisation's counters (negative pivots, perturbed pivots)
__device__ __forceinline__ void flush_counters(int* counters, int nneg, int npert) {
    if (nneg) atomicAdd(counters + 0, nneg);
    if (npert) atomicAdd(counters + 1, npert);
}

// teams per CTA: FW_WARPS one-warp teams, or ONE two-warp team (its staging area is large)
template <int NW> struct TeamsPerCta { static constexpr int value = (NW == 1) ? FW_WARPS : 1; };

template <int NW>
__global__ void __launch_bounds__(TeamsPerCta<NW>::value * NW * 32) k_factor_warp(FactorArgs a, const ChildRec* childrec, WarpSched ws, int maxf) {
    extern __shared__ __align__(16) double sm[];
    constexpr int NTEAM = TeamsPerCta<NW>::value;
    const int team = threadIdx.x / (32 * NW), tid = threadIdx.x % (32 * NW);
    double* smt = sm + (size_t)team * TeamSmem<NW>::doubles(maxf);
    const int s0 = ws.cta_ptr[blockIdx.x], s1 = ws.cta_ptr[blockIdx.x + 1];
    int nneg = 0, npert = 0;
    for (int st = s0; st < s1; ++st) {
        const int off = ws.stage_off[st], cnt = ws.stage_cnt[st];
        for (int q = team; q < cnt; q += NTEAM) front_factor_team<NW>(a, childrec, ws.list[off + q], smt, tid, team, maxf, nneg, npert);
        if (s1 - s0 > 1) __syncthreads();
    }
    if (tid == 0) flush_counters(a.counters, nneg, npert);
}

// ------------------------------------------------------------------------------------------------ solves
// Programmatic dependent launch: a level's kernel is launched while the previous level still runs.  Everything that is
// CONSTANT during a solve (descriptors, index lists, the factor panels) is fetched before pdl_wait(); only the values the
// previous levels produce (xp, cbv) are read after it.  Both calls are no-ops for a launch without the attribute.
// (pdl_trigger / pdl_wait: ptx.cuh)

// A front's solve is three memory round trips, whatever its number of children or pivots:
//   (1) descriptor;  (2) child records + the whole panel (cp.async into shared memory, in flight while (3) runs) + own
//   right-hand side;  (3) every child's relative indices and contribution vector at once.
// Forward:  thread = row i of the front; y_i in a register; the recurrence y_i -= L(i,k) y_k reads L from the staged
//           column-major panel and y_k from a shuffle (one-warp teams) or a double-buffered shared slot (two-warp teams).
// Backward: thread = pivot column j; t_j in a register; L(i,j) comes from the staged ROW-major copy `Lt`.
// With NR right-hand sides (k_solve_dep_block) everything a front stages is fetched once and applied to all NR columns; a thread holds
// NR values in registers, and ys/xs hold one FMAX plane per column.
template <int NW, int NR = 1>
struct SolveSmem {
    static constexpr int FMAX = 32 * NW;
    // ys/xs [NR][FMAX] | slots [16] | recs [MAXC] (4 doubles each) | panel [FMAX*FMAX]
    static constexpr int doubles = NR * FMAX + 16 + 4 * MAXC + FMAX * FMAX;
    // the same slice with the panel sized by the largest front it holds (the four-warp class: FMAX^2 would be 128 KB)
    static __host__ __device__ constexpr int doubles_panel(int maxf) { return NR * FMAX + 16 + 4 * MAXC + maxf * maxf; }
};

// DEP: the front runs inside the single-launch solve (k_solve_dep).  It reads its right-hand side straight from the caller's
// x[perm[j]] and takes its children's contribution vectors from their `up` slots; it puts its own contribution vector into its `up`
// slots and its forward result into its `ypiv` slots (for its own backward task).  The backward sweep takes the ancestor values
// from its `down` slots and its forward result from `ypiv`, writes its solution into x[perm[j]] and puts each child's ancestor
// values into that child's `down` slots.  Without DEP (level-launch solve) the values go through xp and cbv instead.
// NR > 1 with DEP: NR right-hand sides in one walk, column q at x + q * ldx, the first ncol of them live (the others are computed
// on zeros and never touch x).  NR > 1 without DEP (k_fwd_warp2_block): xp and cbv hold NR interleaved columns, entry i of column q
// at [i * NR + q].  Either way each column goes through exactly the operations of NR = 1, in the same order.
template <int NW, bool DEP = false, int NR = 1>
__device__ __forceinline__ void front_fwd_team(const SolveArgs& a, const ChildRec* childrec, int s, double* sm_team, int tid, int team,
                                               int* err = nullptr, int ncol = 1, int64_t ldx = 0) {
    static_assert(NW <= 2 || DEP, "the four-warp class runs in the single-launch solve only");
    constexpr int FMAX = 32 * NW, TEAM = 32 * NW;
    double* ys = sm_team;                              // [NR][FMAX] assembly of the front's rhs
    double* yb = ys + NR * FMAX;                       // [2][8] broadcast slots
    ChildRec* recs = (ChildRec*)(yb + 16);             // [MAXC]
    double* P = (double*)(recs + MAXC);                // panel, column-major, ld f
    if (DEP && a.strace && tid == 0) a.strace[6 * (size_t)s] = global_ns();
    const FrontDesc d = a.desc[s];
    const int f = d.f, w = d.w;
    {
        const double* Lp = a.L + d.lp_off;
        for (int e = tid; e < f * w; e += TEAM) cp_async8(P + e, Lp + e);
    }
    const int pj = (a.x && tid < w) ? a.perm[d.col0 + tid] : 0;
    const int64_t cvo = a.cbv_off[s];                  // (loaded early: the address of the hand-off at the end)
    for (int c0 = 0; c0 < max(d.nchild, 1); c0 += MAXC) {
        const int nc = min(MAXC, d.nchild - c0);
        if (tid < nc) recs[tid] = childrec[d.child_off + c0 + tid];
        team_sync<NW>(team);
        int tg[MAXC]; double vv[MAXC][NR];
#pragma unroll
        for (int c = 0; c < MAXC; ++c) tg[c] = (c < nc && tid < recs[c].rc) ? a.rel[recs[c].rel_off + tid] : -1;
        if (c0 == 0) {                                  // (constant data is in flight; now the values of the levels below)
            if (!DEP) pdl_wait();
#pragma unroll
            for (int q = 0; q < NR; ++q)
                ys[q * FMAX + tid] = (tid < w) ? (a.x ? (q < ncol ? a.x[q * ldx + pj] : 0.0) : a.xp[DEP ? d.col0 + tid : (d.col0 + tid) * NR + q]) : 0.0;
        }
        if (DEP) {                                      // every child's slots at once: one L2 round trip once the last one lands
            double* p[MAXC];
            unsigned need = 0;
#pragma unroll
            for (int c = 0; c < MAXC; ++c) {
                p[c] = a.up + (tg[c] >= 0 ? recs[c].cbv_off + tid : 0) * NR;
                need |= (tg[c] >= 0) ? 1u << c : 0u;
            }
            slot_take_block(p, need, vv, err);
        } else {
#pragma unroll
            for (int c = 0; c < MAXC; ++c) {
#pragma unroll
                for (int q = 0; q < NR; ++q) vv[c][q] = (tg[c] >= 0) ? a.cbv[(recs[c].cbv_off + tid) * NR + q] : 0.0;
            }
        }
        if (c0 == 0) team_sync<NW>(team);
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {               // ascending child order: deterministic sums
            if (c < nc) {
                if (tg[c] >= 0) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) ys[q * FMAX + tg[c]] += vv[c][q];
                }
                team_sync<NW>(team);
            }
        }
    }
    if (DEP && a.strace && tid == 0) a.strace[6 * (size_t)s + 1] = global_ns();
    cp_async_wait_all();
    team_sync<NW>(team);
    double y[NR];
#pragma unroll
    for (int q = 0; q < NR; ++q) y[q] = ys[q * FMAX + tid];
    if (NW == 1) {
        for (int k0 = 0; k0 < w; k0 += 8) {
            double l[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int k = k0 + u; l[u] = (k < w && tid > k && tid < f) ? P[k * f + tid] : 0.0; }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int k = k0 + u;
                if (k < w) {                                                        // team-uniform
#pragma unroll
                    for (int q = 0; q < NR; ++q) y[q] = fma(-l[u], __shfl_sync(0xffffffffu, y[q], k), y[q]);
                }
            }
        }
    } else if (NW == 2) {
        // two-warp team, blocked by warp: warp 0 eliminates pivots 0..31 among its own rows with shuffles and publishes
        // them; warp 1 applies them in one parallel pass, then eliminates pivots 32.. among its rows -- two barriers per
        // front instead of one per pivot
        const int w0 = min(w, 32);
        if (tid < 32) {
            for (int k0 = 0; k0 < w0; k0 += 8) {
                double l[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int k = k0 + u; l[u] = (k < w0 && tid > k && tid < f) ? P[k * f + tid] : 0.0; }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int k = k0 + u;
                    if (k < w0) {
#pragma unroll
                        for (int q = 0; q < NR; ++q) y[q] = fma(-l[u], __shfl_sync(0xffffffffu, y[q], k), y[q]);
                    }
                }
            }
            if (tid < w0) {
#pragma unroll
                for (int q = 0; q < NR; ++q) ys[q * FMAX + tid] = y[q];
            }
        }
        team_sync<NW>(team);
        if (tid >= 32) {
            if (tid < f) {
                double acc[NR];
#pragma unroll
                for (int q = 0; q < NR; ++q) acc[q] = 0.0;
#pragma unroll 8
                for (int k = 0; k < w0; ++k) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) acc[q] = fma(P[k * f + tid], ys[q * FMAX + k], acc[q]);
                }
#pragma unroll
                for (int q = 0; q < NR; ++q) y[q] -= acc[q];
            }
            for (int k0 = 32; k0 < w; k0 += 8) {
                double l[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int k = k0 + u; l[u] = (k < w && tid > k && tid < f) ? P[k * f + tid] : 0.0; }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int k = k0 + u;
                    if (k < w) {
#pragma unroll
                        for (int q = 0; q < NR; ++q) y[q] = fma(-l[u], __shfl_sync(0xffffffffu, y[q], k - 32), y[q]);
                    }
                }
            }
        }
    } else {
        // four-warp team, blocked by warp as above: in round b, warp b (which has applied blocks < b) eliminates pivots
        // [32b, 32b+32) among its own rows with shuffles and publishes them; every warp below applies them in one pass
        const int wp = tid >> 5;
        for (int kb = 0; kb < w; kb += 32) {
            const int ke = min(w, kb + 32);
            if (wp == kb >> 5) {
                for (int k0 = kb; k0 < ke; k0 += 8) {
                    double l[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int k = k0 + u; l[u] = (k < ke && tid > k && tid < f) ? P[k * f + tid] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const int k = k0 + u;
                        if (k < ke) {
#pragma unroll
                            for (int q = 0; q < NR; ++q) y[q] = fma(-l[u], __shfl_sync(0xffffffffu, y[q], k - kb), y[q]);
                        }
                    }
                }
                if (tid < ke) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) ys[q * FMAX + tid] = y[q];
                }
            }
            team_sync<NW>(team);
            if (wp > (kb >> 5) && tid < f) {
                double acc[NR];
#pragma unroll
                for (int q = 0; q < NR; ++q) acc[q] = 0.0;
#pragma unroll 8
                for (int k = kb; k < ke; ++k) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) acc[q] = fma(P[k * f + tid], ys[q * FMAX + k], acc[q]);
                }
#pragma unroll
                for (int q = 0; q < NR; ++q) y[q] -= acc[q];
            }
        }
    }
    if (DEP) {
        if constexpr (NR == 1) {
            if (tid < f) slot_put(tid < w ? a.ypiv + d.col0 + tid : a.up + cvo + tid - w, y[0]);
        } else {
            if (tid < f) slot_put_block(tid < w ? a.ypiv + (d.col0 + tid) * NR : a.up + (cvo + tid - w) * NR, y);
        }
        if (a.strace) { team_sync<NW>(team); if (tid == 0) a.strace[6 * (size_t)s + 2] = global_ns(); }
    } else {
        if (tid < f) {
#pragma unroll
            for (int q = 0; q < NR; ++q) { if (tid < w) a.xp[(d.col0 + tid) * NR + q] = y[q]; else a.cbv[(cvo + tid - w) * NR + q] = y[q]; }
        }
        team_sync<NW>(team);
    }
}

// PAIRS (DEP only): D^-1 over the 2 x 2 blocks that dsub marks (PairArgs), by dsytrs's formula
template <int NW, bool DEP = false, bool PAIRS = false>
__device__ __forceinline__ void front_bwd_team(const SolveArgs& a, int s, double* sm_team, int tid, int team,
                                               const ChildRec* childrec = nullptr, int* err = nullptr, const double* dsub = nullptr) {
    static_assert(NW <= 2 || DEP, "the four-warp class runs in the single-launch solve only");
    constexpr int FMAX = 32 * NW, TEAM = 32 * NW;
    double* xs = sm_team;                              // [FMAX] gathered ancestor values at [xa, xa + r)
    double* xb = xs + FMAX;                            // [2][8]
    ChildRec* recs = (ChildRec*)(xb + 16);             // [MAXC] (DEP: the children, whose `down` slots this front fills)
    double* P = xb + 16 + 4 * MAXC;                    // row-major f x w panel (same slice layout as the forward sweep)
    if (DEP && a.strace && tid == 0) a.strace[6 * (size_t)s + 3] = global_ns();
    const FrontDesc d = a.desc[s];
    const int f = d.f, w = d.w, r = f - w;
    // DEP: xs is the whole front vector -- own pivots' x at [0, w), the ancestors' at [w, f) -- from which the children's
    // hand-offs are gathered
    const int xa = DEP ? w : 0;
    {
        const double* Lt = a.Lt + d.lp_off;
        for (int e = tid; e < f * w; e += TEAM) cp_async8(P + e, Lt + e);
    }
    const int32_t* rows = a.rows + d.rows_off + w;
    const int myrow = (!DEP && tid < r) ? rows[tid] : 0;
    const int pj = (a.x && tid < w) ? a.perm[d.col0 + tid] : 0;
    const double dinv = (tid < w) ? fast_rcp(a.dvec[d.col0 + tid]) : 0.0;
    const int nc0 = min(MAXC, d.nchild);
    int tg[MAXC];                                      // DEP: row of the front that child c's slot `tid` takes
    double t;
    if (DEP) {
        // the children's records and relative indices are constant: fetched before the wait, so that the hand-off to the
        // children follows the back-substitution directly
        if (tid < nc0) recs[tid] = childrec[d.child_off + tid];
        team_sync<NW>(team);
#pragma unroll
        for (int c = 0; c < MAXC; ++c) tg[c] = (c < nc0 && tid < recs[c].rc) ? a.rel[recs[c].rel_off + tid] : -1;
        // ancestor values (the parent's hand-off) and own forward result, at once
        double* const p[2] = {a.down + a.cbv_off[s] + tid, a.ypiv + d.col0 + tid};
        double v[2];
        slot_take(p, (tid < r ? 1u : 0u) | (tid < w ? 2u : 0u), v, err);
        if (tid < r) xs[xa + tid] = v[0];
        t = (tid < w) ? v[1] * dinv : 0.0;
        if constexpr (PAIRS) {
            // a block's partner row is in the same front: its forward value through xs[0, w), free until the back-substitution
            if (tid < w) xs[tid] = v[1];
            team_sync<NW>(team);
            const int i = d.col0 + tid;
            const bool first = tid < w && dsub[i] != 0.0, second = tid < w && tid > 0 && dsub[i - 1] != 0.0;
            if (first || second) {
                const int i0 = first ? i : i - 1, k0 = first ? tid : tid - 1;
                const double akm1k = dsub[i0], akm1 = a.dvec[i0] / akm1k, ak = a.dvec[i0 + 1] / akm1k;
                const double denom = akm1 * ak - 1.0, bkm1 = xs[k0] / akm1k, bk = xs[k0 + 1] / akm1k;
                t = first ? (ak * bkm1 - bk) / denom : (akm1 * bk - bkm1) / denom;
            }
        }
    } else {
        pdl_wait();
        if (tid < r) xs[xa + tid] = a.xp[myrow];
        t = (tid < w) ? a.xp[d.col0 + tid] * dinv : 0.0;
    }
    cp_async_wait_all();
    team_sync<NW>(team);
    if (DEP && a.strace && tid == 0) a.strace[6 * (size_t)s + 4] = global_ns();
    {   // t_j -= sum_{i >= w} L(i,j) x_i : no recurrence
        double acc = 0.0;
        if (tid < w) {
#pragma unroll 8
            for (int i = 0; i < r; ++i) acc = fma(P[(w + i) * w + tid], xs[xa + i], acc);
        }
        t -= acc;
    }
    // back-substitution with L11': x_k final -> t_j -= L(k,j) x_k for j < k
    if (NW == 1) {
        for (int k0 = w - 1; k0 >= 1; k0 -= 8) {
            double l[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int k = k0 - u;
                if (k >= 1) t = fma(-l[u], __shfl_sync(0xffffffffu, t, k), t);
            }
        }
    } else if (NW == 2) {
        // blocked by warp (see the forward sweep): warp 1 finishes columns 32.. with shuffles and publishes them in
        // xs[32..w) (the gathered ancestors occupy xs[0 .. f-w) with f - w < 32 here, or xs[w .. f) with DEP); warp 0 applies
        // them in one pass
        if (w > 32) {
            if (tid >= 32) {
                for (int k0 = w - 1; k0 >= 33; k0 -= 8) {
                    double l[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 33 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const int k = k0 - u;
                        if (k >= 33) t = fma(-l[u], __shfl_sync(0xffffffffu, t, k - 32), t);
                    }
                }
                if (tid < w) xs[tid] = t;
            }
            team_sync<NW>(team);
            if (tid < 32) {
                double acc = 0.0;
#pragma unroll 8
                for (int k = 32; k < w; ++k) acc = fma(P[k * w + tid], xs[k], acc);
                t -= acc;
            }
        }
        if (tid < 32) {
            for (int k0 = min(w, 32) - 1; k0 >= 1; k0 -= 8) {
                double l[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int k = k0 - u;
                    if (k >= 1) t = fma(-l[u], __shfl_sync(0xffffffffu, t, k), t);
                }
            }
        }
    } else {
        // four-warp team, last block first: in round b, warp b (which has applied blocks > b) finishes columns [32b, 32b+32) with
        // shuffles and publishes them in xs[32b..) (own pivots' region: the ancestors are at xs[w .. f)); every warp above applies
        // them in one pass
        const int wp = tid >> 5;
        for (int kb = ((w - 1) >> 5) * 32; kb >= 0; kb -= 32) {
            const int ke = min(w, kb + 32);
            if (wp == kb >> 5) {
                for (int k0 = ke - 1; k0 >= kb + 1; k0 -= 8) {
                    double l[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= kb + 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const int k = k0 - u;
                        if (k >= kb + 1) t = fma(-l[u], __shfl_sync(0xffffffffu, t, k - kb), t);
                    }
                }
                if (kb > 0 && tid < w) xs[tid] = t;
            }
            if (kb > 0) {
                team_sync<NW>(team);
                if (wp < (kb >> 5)) {
                    double acc = 0.0;
#pragma unroll 8
                    for (int k = kb; k < ke; ++k) acc = fma(P[k * w + tid], xs[k], acc);
                    t -= acc;
                }
            }
        }
    }
    if (DEP) {
        if (tid < w) { xs[tid] = t; a.x[pj] = t; }
        team_sync<NW>(team);
        // hand-off to the children: slot i of child c takes the front's value at row rel_c[i]
#pragma unroll
        for (int c = 0; c < MAXC; ++c) if (tg[c] >= 0) slot_put(a.down + recs[c].cbv_off + tid, xs[tg[c]]);
        for (int c0 = MAXC; c0 < d.nchild; c0 += MAXC) {          // (fronts with more than MAXC children)
            const int nc = min(MAXC, d.nchild - c0);
            team_sync<NW>(team);
            if (tid < nc) recs[tid] = childrec[d.child_off + c0 + tid];
            team_sync<NW>(team);
            for (int c = 0; c < nc; ++c)
                if (tid < recs[c].rc) slot_put(a.down + recs[c].cbv_off + tid, xs[a.rel[recs[c].rel_off + tid]]);
        }
        if (a.strace) { team_sync<NW>(team); if (tid == 0) a.strace[6 * (size_t)s + 5] = global_ns(); }
    } else {
        if (tid < w) a.xp[d.col0 + tid] = t;
        team_sync<NW>(team);
    }
}

// front_bwd_team<NW, DEP, PAIRS> for NR > 1 right-hand sides, as front_fwd_team<NW, DEP, NR>: every column goes through the one-column
// operations in the same order.  DEP: k_solve_dep_block; without DEP: k_bwd_warp2_block, on NR interleaved columns of xp.  (A separate
// function: an NR parameter on front_bwd_team changes the code ptxas emits for the existing one-column kernels.)
template <int NW, bool PAIRS, int NR, bool DEP = true>
__device__ __forceinline__ void front_bwd_block(const SolveArgs& a, int s, double* sm_team, int tid, int team, const ChildRec* childrec,
                                                int* err, const double* dsub, int ncol, int64_t ldx) {
    static_assert(NR % 2 == 0, "block slots are accessed in 16-byte pairs");
    static_assert(DEP || !PAIRS, "pair factors are solved on the single-launch schedule only");
    static_assert(NW <= 2 || (DEP && PAIRS), "the four-warp class holds PAIRS fronts on the single-launch schedule only");
    constexpr int FMAX = 32 * NW, TEAM = 32 * NW;
    double* xs = sm_team;                              // [NR][FMAX] gathered ancestor values at [xa, xa + r)
    double* xb = xs + NR * FMAX;                       // [2][8]
    ChildRec* recs = (ChildRec*)(xb + 16);             // [MAXC] the children, whose `down` slots this front fills
    double* P = xb + 16 + 4 * MAXC;                    // row-major f x w panel (same slice layout as the forward sweep)
    const FrontDesc d = a.desc[s];
    const int f = d.f, w = d.w, r = f - w;
    // DEP: xs is the whole front vector -- own pivots' x at [0, w), the ancestors' at [w, f) -- from which the children's hand-offs are
    // gathered
    const int xa = DEP ? w : 0;
    {
        const double* Lt = a.Lt + d.lp_off;
        for (int e = tid; e < f * w; e += TEAM) cp_async8(P + e, Lt + e);
    }
    const int myrow = (!DEP && tid < r) ? a.rows[d.rows_off + w + tid] : 0;
    const int pj = (DEP && tid < w) ? a.perm[d.col0 + tid] : 0;
    const double dinv = (tid < w) ? fast_rcp(a.dvec[d.col0 + tid]) : 0.0;
    const int nc0 = min(MAXC, d.nchild);
    int tg[MAXC];                                      // row of the front that child c's slot `tid` takes
    double t[NR];
    if constexpr (!DEP) {
        pdl_wait();
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            if (tid < r) xs[q * FMAX + tid] = a.xp[myrow * NR + q];
            t[q] = (tid < w) ? a.xp[(d.col0 + tid) * NR + q] * dinv : 0.0;
        }
    } else {
        // the children's records and relative indices are constant: fetched before the wait, so that the hand-off to the
        // children follows the back-substitution directly
        if (tid < nc0) recs[tid] = childrec[d.child_off + tid];
        team_sync<NW>(team);
#pragma unroll
        for (int c = 0; c < MAXC; ++c) tg[c] = (c < nc0 && tid < recs[c].rc) ? a.rel[recs[c].rel_off + tid] : -1;
        // ancestor values (the parent's hand-off) and own forward result, at once
        double* const p[2] = {a.down + (a.cbv_off[s] + tid) * NR, a.ypiv + (d.col0 + tid) * NR};
        double v[2][NR];
        slot_take_block(p, (tid < r ? 1u : 0u) | (tid < w ? 2u : 0u), v, err);
#pragma unroll
        for (int q = 0; q < NR; ++q) {
            if (tid < r) xs[q * FMAX + xa + tid] = v[0][q];
            t[q] = (tid < w) ? v[1][q] * dinv : 0.0;
        }
        if constexpr (PAIRS) {
            // a block's partner row is in the same front: its forward value through xs[0, w), free until the back-substitution
            if (tid < w) {
#pragma unroll
                for (int q = 0; q < NR; ++q) xs[q * FMAX + tid] = v[1][q];
            }
            team_sync<NW>(team);
            const int i = d.col0 + tid;
            const bool first = tid < w && dsub[i] != 0.0, second = tid < w && tid > 0 && dsub[i - 1] != 0.0;
            if (first || second) {
                const int i0 = first ? i : i - 1, k0 = first ? tid : tid - 1;
                const double akm1k = dsub[i0], akm1 = a.dvec[i0] / akm1k, ak = a.dvec[i0 + 1] / akm1k;
                const double denom = akm1 * ak - 1.0;
#pragma unroll
                for (int q = 0; q < NR; ++q) {
                    const double bkm1 = xs[q * FMAX + k0] / akm1k, bk = xs[q * FMAX + k0 + 1] / akm1k;
                    t[q] = first ? (ak * bkm1 - bk) / denom : (akm1 * bk - bkm1) / denom;
                }
            }
        }
    }
    cp_async_wait_all();
    team_sync<NW>(team);
    {   // t_j -= sum_{i >= w} L(i,j) x_i : no recurrence
        double acc[NR];
#pragma unroll
        for (int q = 0; q < NR; ++q) acc[q] = 0.0;
        if (tid < w) {
#pragma unroll 8
            for (int i = 0; i < r; ++i) {
#pragma unroll
                for (int q = 0; q < NR; ++q) acc[q] = fma(P[(w + i) * w + tid], xs[q * FMAX + xa + i], acc[q]);
            }
        }
#pragma unroll
        for (int q = 0; q < NR; ++q) t[q] -= acc[q];
    }
    // back-substitution with L11': x_k final -> t_j -= L(k,j) x_k for j < k
    if (NW == 1) {
        for (int k0 = w - 1; k0 >= 1; k0 -= 8) {
            double l[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int k = k0 - u;
                if (k >= 1) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) t[q] = fma(-l[u], __shfl_sync(0xffffffffu, t[q], k), t[q]);
                }
            }
        }
    } else if (NW == 2) {
        // blocked by warp (front_bwd_team): warp 1 finishes columns 32.. and publishes them in xs[32..w); warp 0 applies them
        if (w > 32) {
            if (tid >= 32) {
                for (int k0 = w - 1; k0 >= 33; k0 -= 8) {
                    double l[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 33 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const int k = k0 - u;
                        if (k >= 33) {
#pragma unroll
                            for (int q = 0; q < NR; ++q) t[q] = fma(-l[u], __shfl_sync(0xffffffffu, t[q], k - 32), t[q]);
                        }
                    }
                }
                if (tid < w) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) xs[q * FMAX + tid] = t[q];
                }
            }
            team_sync<NW>(team);
            if (tid < 32) {
                double acc[NR];
#pragma unroll
                for (int q = 0; q < NR; ++q) acc[q] = 0.0;
#pragma unroll 8
                for (int k = 32; k < w; ++k) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) acc[q] = fma(P[k * w + tid], xs[q * FMAX + k], acc[q]);
                }
#pragma unroll
                for (int q = 0; q < NR; ++q) t[q] -= acc[q];
            }
        }
        if (tid < 32) {
            for (int k0 = min(w, 32) - 1; k0 >= 1; k0 -= 8) {
                double l[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int k = k0 - u;
                    if (k >= 1) {
#pragma unroll
                        for (int q = 0; q < NR; ++q) t[q] = fma(-l[u], __shfl_sync(0xffffffffu, t[q], k), t[q]);
                    }
                }
            }
        }
    } else {
        // four-warp team, last block first (front_bwd_team)
        const int wp = tid >> 5;
        for (int kb = ((w - 1) >> 5) * 32; kb >= 0; kb -= 32) {
            const int ke = min(w, kb + 32);
            if (wp == kb >> 5) {
                for (int k0 = ke - 1; k0 >= kb + 1; k0 -= 8) {
                    double l[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const int k = k0 - u; l[u] = (k >= kb + 1 && tid < k) ? P[k * w + tid] : 0.0; }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const int k = k0 - u;
                        if (k >= kb + 1) {
#pragma unroll
                            for (int q = 0; q < NR; ++q) t[q] = fma(-l[u], __shfl_sync(0xffffffffu, t[q], k - kb), t[q]);
                        }
                    }
                }
                if (kb > 0 && tid < w) {
#pragma unroll
                    for (int q = 0; q < NR; ++q) xs[q * FMAX + tid] = t[q];
                }
            }
            if (kb > 0) {
                team_sync<NW>(team);
                if (wp < (kb >> 5)) {
                    double acc[NR];
#pragma unroll
                    for (int q = 0; q < NR; ++q) acc[q] = 0.0;
#pragma unroll 8
                    for (int k = kb; k < ke; ++k) {
#pragma unroll
                        for (int q = 0; q < NR; ++q) acc[q] = fma(P[k * w + tid], xs[q * FMAX + k], acc[q]);
                    }
#pragma unroll
                    for (int q = 0; q < NR; ++q) t[q] -= acc[q];
                }
            }
        }
    }
    if constexpr (!DEP) {
        if (tid < w) {
#pragma unroll
            for (int q = 0; q < NR; ++q) a.xp[(d.col0 + tid) * NR + q] = t[q];
        }
        team_sync<NW>(team);
    } else {
        if (tid < w) {
#pragma unroll
            for (int q = 0; q < NR; ++q) {
                xs[q * FMAX + tid] = t[q];
                if (q < ncol) a.x[q * ldx + pj] = t[q];
            }
        }
        team_sync<NW>(team);
        // hand-off to the children: slot i of child c takes the front's value at row rel_c[i]
        auto put_down = [&](int64_t cbv_off, int row) {
            double v[NR];
#pragma unroll
            for (int q = 0; q < NR; ++q) v[q] = xs[q * FMAX + row];
            slot_put_block(a.down + (cbv_off + tid) * NR, v);
        };
#pragma unroll
        for (int c = 0; c < MAXC; ++c) if (tg[c] >= 0) put_down(recs[c].cbv_off, tg[c]);
        for (int c0 = MAXC; c0 < d.nchild; c0 += MAXC) {          // (fronts with more than MAXC children)
            const int nc = min(MAXC, d.nchild - c0);
            team_sync<NW>(team);
            if (tid < nc) recs[tid] = childrec[d.child_off + c0 + tid];
            team_sync<NW>(team);
            for (int c = 0; c < nc; ++c)
                if (tid < recs[c].rc) put_down(recs[c].cbv_off, a.rel[recs[c].rel_off + tid]);
        }
    }
}

// NTEAM teams per CTA.  Measured on OPF-10k (tools/sweep_headline.sh): sweeping the fused bottom subtrees with 8 one-warp teams per
// CTA instead of 4 is SLOWER (fewer resident CTAs, wider barriers), while smaller subtrees (fuse_max_fronts 16 -> 8) are
// faster -- so the fused launches keep TeamsPerCta teams.
constexpr int SOLVE_FUSED_TEAMS = 4;
// One sweep of a level-launch solve: a CTA walks its stages (forward: ascending, backward: descending), its NTEAM teams sharing each
// stage's fronts.  NR = 1 is the one-column solve on xp / cbv; NR > 1 (b2_solve's level-launch block solve) holds NR interleaved columns
// of xp and cbv, with front_bwd_block as the backward front.  The kernels below keep their names as thin wrappers.
template <int NW, int NTEAM, int NR>
__device__ __forceinline__ void fwd_warp_sweep(const SolveArgs& a, const ChildRec* childrec, const WarpSched& ws) {
    extern __shared__ __align__(16) double smd[];
    double (*sm)[SolveSmem<NW, NR>::doubles] = (double (*)[SolveSmem<NW, NR>::doubles])smd;
    const int team = threadIdx.x / (32 * NW), tid = threadIdx.x % (32 * NW);
    pdl_trigger();
    const int s0 = ws.cta_ptr[blockIdx.x], s1 = ws.cta_ptr[blockIdx.x + 1];
    for (int st = s0; st < s1; ++st) {
        const int off = ws.stage_off[st], cnt = ws.stage_cnt[st];
        for (int q = team; q < cnt; q += NTEAM) front_fwd_team<NW, false, NR>(a, childrec, ws.list[off + q], sm[team], tid, team);
        if (s1 - s0 > 1) __syncthreads();
    }
    pdl_wait();                                         // (idle teams too: this grid's completion must imply its predecessor's)
}

template <int NW, int NTEAM, int NR>
__device__ __forceinline__ void bwd_warp_sweep(const SolveArgs& a, const WarpSched& ws) {
    extern __shared__ __align__(16) double smd[];
    double (*sm)[SolveSmem<NW, NR>::doubles] = (double (*)[SolveSmem<NW, NR>::doubles])smd;
    const int team = threadIdx.x / (32 * NW), tid = threadIdx.x % (32 * NW);
    pdl_trigger();
    const int s0 = ws.cta_ptr[blockIdx.x], s1 = ws.cta_ptr[blockIdx.x + 1];
    for (int st = s1 - 1; st >= s0; --st) {
        const int off = ws.stage_off[st], cnt = ws.stage_cnt[st];
        for (int q = team; q < cnt; q += NTEAM) {
            if constexpr (NR == 1) front_bwd_team<NW>(a, ws.list[off + q], sm[team], tid, team);
            else front_bwd_block<NW, false, NR, false>(a, ws.list[off + q], sm[team], tid, team, nullptr, nullptr, nullptr, 0, 0);
        }
        if (s1 - s0 > 1) __syncthreads();
    }
    pdl_wait();
}

template <int NW, int NTEAM = TeamsPerCta<NW>::value>
__global__ void __launch_bounds__(NTEAM * NW * 32) k_fwd_warp2(SolveArgs a, const ChildRec* childrec, WarpSched ws) {
    fwd_warp_sweep<NW, NTEAM, 1>(a, childrec, ws);
}
template <int NW, int NTEAM = TeamsPerCta<NW>::value>
__global__ void __launch_bounds__(NTEAM * NW * 32) k_bwd_warp2(SolveArgs a, WarpSched ws) {
    bwd_warp_sweep<NW, NTEAM, 1>(a, ws);
}
template <int NW, int NTEAM, int NR>
__global__ void __launch_bounds__(NTEAM * NW * 32) k_fwd_warp2_block(SolveArgs a, const ChildRec* childrec, WarpSched ws) {
    fwd_warp_sweep<NW, NTEAM, NR>(a, childrec, ws);
}
template <int NW, int NTEAM, int NR>
__global__ void __launch_bounds__(NTEAM * NW * 32) k_bwd_warp2_block(SolveArgs a, WarpSched ws) {
    bwd_warp_sweep<NW, NTEAM, NR>(a, ws);
}


// ------------------------------------------------------------------------------------------------ single-launch schedule
// The whole (team-class) elimination tree in ONE launch per sweep: CTAs are issued in topological order, a front waits on
// its children's completion flags (acquire loads on global memory, bounded spin) instead of on a kernel boundary.  A CTA
// of 128 threads runs a GROUP of tasks: four one-warp teams (fronts of order <= 32) or one two-warp team (order <= 64); with PAIRS
// also one four-warp team (order 65..96).
struct DepSched {
    const int32_t* grp_type;   // 1 or 2 (warps per team); PAIRS also 4 (one front of order 65..96)
    const int32_t* grp_ptr;    // [ngroup+1] into tasks
    const int32_t* tasks;      // supernode ids in topological ticket order (dep_ticket_order in sparse_ldl.cu)
    int ngroup;
};

// Forward progress: a CTA only ever waits for groups that come EARLIER in the topological order.  Groups are therefore claimed
// through an atomic ticket instead of blockIdx.x: whichever CTA the hardware starts first takes the earliest unclaimed group, so a
// running CTA never waits for work that no running (or finished) CTA owns -- independent of the block dispatch order, which the
// programming model does not specify (the bounded spin of the flag polls stays as a second line of defence).
__device__ __forceinline__ int claim_group(int* ticket, int ngroup) {
    __shared__ int g_sh;
    if (threadIdx.x == 0) {
        const int t = atomicAdd(ticket, 1);
        if (t == ngroup - 1) atomicExch(ticket, 0);     // last claim of this launch: re-arm the counter for the next one
        g_sh = t;
    }
    __syncthreads();
    return g_sh;
}

// A group's team and the thread's index in it: type 1 is four one-warp teams, type 2 one two-warp team, type 4 (PAIRS only) one
// four-warp team.
template <bool PAIRS>
__device__ __forceinline__ void group_team(int type, int& team, int& tid) {
    team = (type == 1) ? (threadIdx.x >> 5) : (!PAIRS || type == 2) ? (threadIdx.x >> 6) : 0;
    tid = (type == 1) ? (threadIdx.x & 31) : (!PAIRS || type == 2) ? (threadIdx.x & 63) : threadIdx.x;
}

// PAIRS (b2_options.sparse_pivoting = B2_SPARSE_PIVOT_PAIRS): front_factor_team's pivot loop with candidate 2 x 2 pivots, and type-4
// groups, one front of order 65..96 as a four-warp team (the pair ordering makes fronts larger: DESIGN.md section 3).  maxf4 and pa
// are unused without PAIRS.  The static instance folds every PAIRS test away and compiles to the same machine code as a body written
// for it alone (tools/sass_diff.py compares the builds).
template <bool PAIRS>
__device__ __forceinline__ void factor_dep_body(const FactorArgs& a, const ChildRec* childrec, const DepSched& ds, int maxf1, int maxf2,
                                                int maxf4, int* done, int* err, int* ticket, const PairArgs& pa) {
    extern __shared__ __align__(16) double sm[];
    const int g = claim_group(ticket, ds.ngroup);
    const int type = ds.grp_type[g], t0 = ds.grp_ptr[g], n = ds.grp_ptr[g + 1] - t0;
    int npert = 0, nneg = 0;                            // (declared in this order, the static kernel's code is unchanged)
    if (type == 1) {
        const int team = threadIdx.x >> 5, tid = threadIdx.x & 31;
        if (team < n) front_factor_team<1, true, PAIRS>(a, childrec, ds.tasks[t0 + team], sm + (size_t)team * TeamSmem<1>::doubles(maxf1),
                                                        tid, team, maxf1, nneg, npert, nullptr, done, err, pa);
        if (tid == 0) flush_counters(a.counters, nneg, npert);
    } else if (!PAIRS || type == 2) {
        const int team = threadIdx.x >> 6, tid = threadIdx.x & 63;
        if (team < n) front_factor_team<2, true, PAIRS>(a, childrec, ds.tasks[t0 + team], sm, tid, team, maxf2, nneg, npert, nullptr, done, err, pa);
        if (tid == 0 && team < n) flush_counters(a.counters, nneg, npert);
    } else if constexpr (PAIRS) {
        front_factor_team<4, true, true>(a, childrec, ds.tasks[t0], sm, threadIdx.x, 0, maxf4, nneg, npert, nullptr, done, err, pa);
        if (threadIdx.x == 0) flush_counters(a.counters, nneg, npert);
    }
}

__global__ void __launch_bounds__(128) k_factor_dep(FactorArgs a, const ChildRec* childrec, DepSched ds, int maxf1, int maxf2,
                                                    int* done, int* err, int* ticket) {
    factor_dep_body<false>(a, childrec, ds, maxf1, maxf2, 0, done, err, ticket, PairArgs());
}

__global__ void __launch_bounds__(128) k_factor_dep_pairs(FactorArgs a, const ChildRec* childrec, DepSched ds, int maxf1, int maxf2,
                                                          int maxf4, int* done, int* err, int* ticket, PairArgs pa) {
    factor_dep_body<true>(a, childrec, ds, maxf1, maxf2, maxf4, done, err, ticket, pa);
}

// ------------------------------------------------------------------------------------------------ single-launch solve
// Forward sweep, D^-1 and backward sweep of the whole (team-class, unsharded) tree in ONE launch.  The tasks are the groups of
// k_factor_dep (DepSched: fronts in ticket order, four fronts of order <= 32 as one-warp teams or one front of order <= 64 as a
// two-warp team per group):
//   ticket [0, ngroup)          forward sweep of group t: a front takes its children's contribution vectors from their `up` slots
//   ticket [ngroup, 2 ngroup)   backward sweep of the groups in reverse order: a front takes its ancestors' values from its `down`
//                               slots (its parent's hand-off) and its own forward result from its `ypiv` slots
// A persistent grid claims the tickets through an atomic counter, one task at a time.  A front waits only on fronts of smaller
// tickets or of its own group (another team: no CTA-wide barrier inside a task), and a CTA claims a ticket only while it runs, so
// forward progress does not depend on how many CTAs are resident or in which order they are dispatched.
// Fronts of order <= 32 run as one-warp teams here and as two-warp teams in the level-launch solve above the fused subtrees; for
// w <= f <= 32 the two-warp code runs warp 0 alone through the same loops, so the result is bit-identical to the level solve.
// Hand-offs are per front (measured: that beats running fused bottom subtrees stage by stage inside one CTA, whose stages each
// cost a front's full latency and which need more than two waves of the resident CTAs on OPF-10k).
//
// Every hand-off is a slot that holds the value itself (slot_take / slot_put): a consumer polls the data, so a tree hop costs one
// L2 round trip and no release fence.  Why each value read across CTAs inside the launch is safe:
//   * an `up`, `down` or `ypiv` slot has exactly one writer and one reader per launch, and 8-byte aligned accesses are
//     single-copy atomic: a reader that sees anything but SLOT_EMPTY sees the whole value, and nothing else it reads depends on
//     the writer's other stores (each value a front needs from another CTA travels in its own slot);
//   * the reader re-arms the slot after it has the value, and the next launch is ordered behind that store by the kernel boundary;
//   * everything else a task reads (descriptors, panels, D, indices, the right-hand side x) was written by earlier launches;
//   * the caller's x[perm[j]] is read by front s's forward task and written by its backward task, which takes that forward
//     task's result (ypiv) first: the write data-depends on the read having completed.
// Re-arming needs no other graph node.  There are exactly ntask + gridDim claims (each CTA ends with one failing claim); a CTA
// then fences its stores and counts itself out, and the last CTA out -- every task of the launch has finished -- resets both
// counters (ctl = {ticket, CTAs out}).  If a wait timed out anywhere (or in the factorisation), that CTA writes NaN into x so
// that Richardson refinement rejects the step, and fills every slot with SLOT_EMPTY again: a slot whose consumer gave up may
// hold a value the next launch must not see.
// (six CTAs per SM: what the 35 KB of shared memory allows; the bound also keeps ptxas from spilling)
//
// The ticket claim and the count-out / time-out path are shared with k_solve_dep_block; each kernel writes its own claim loop around
// them, because one loop body inlined into all of them compiles the block kernels to different machine code (tools/sass_diff.py).
__device__ __forceinline__ int claim_task(int* ctl) {
    __shared__ int tk_sh;
    if (threadIdx.x == 0) tk_sh = atomicAdd(ctl, 1);
    __syncthreads();
    return tk_sh;
}

// after the last claim: count the CTA out, re-arm the counters once every CTA is out, and on a time-out anywhere write NaN into the
// ncol columns of x (ld n) and SLOT_EMPTY into every slot
__device__ __forceinline__ void solve_dep_finish(double* x, int n, int ncol, int* err, int* ctl, double* slots, int64_t nslot) {
    __shared__ int bad_sh;
    if (threadIdx.x == 0) {
        bad_sh = 0;
        __threadfence();                                // this CTA's stores (the barrier above orders the whole CTA's) before it counts out
        if (atomicAdd(ctl + 1, 1) == (int)gridDim.x - 1) {
            atomicExch(ctl, 0);
            atomicExch(ctl + 1, 0);
            __threadfence();
            bad_sh = *(volatile int*)err;
        }
    }
    __syncthreads();
    if (bad_sh) {
        for (int q = 0; q < ncol; ++q)
            for (int i = threadIdx.x; i < n; i += blockDim.x) x[(int64_t)q * n + i] = __longlong_as_double((long long)CANON_NAN);
        for (int64_t i = threadIdx.x; i < nslot; i += blockDim.x) st_relaxed_b64(slots + i, SLOT_EMPTY);
    }
}

// PAIRS: D has 2 x 2 blocks (dsub, front_bwd_team<.., PAIRS>), and a type-4 group is one front of order 65..96 on a four-warp slice
// (SolveSmem<4>::doubles_panel).  The static kernel compiles to the same machine code as a body written for it alone.
template <bool PAIRS>
__device__ __forceinline__ void solve_dep_body(const SolveArgs& a, const ChildRec* childrec, const DepSched& ds, int* err, int* ctl, int n,
                                               double* slots, int64_t nslot, const double* dsub) {
    extern __shared__ __align__(16) double smd[];       // max(4 one-warp slices, 1 two-warp slice, PAIRS: 1 four-warp slice)
    double (*sm1)[SolveSmem<1>::doubles] = (double (*)[SolveSmem<1>::doubles])smd;
    const int ntask = 2 * ds.ngroup;
    for (;;) {
        const int t = claim_task(ctl);
        if (t >= ntask) break;
        const bool fwd = t < ds.ngroup;
        const int g = fwd ? t : ntask - 1 - t;
        const int type = ds.grp_type[g], t0 = ds.grp_ptr[g], cnt = ds.grp_ptr[g + 1] - t0;
        int team, tid;
        group_team<PAIRS>(type, team, tid);
        if (team < cnt) {
            const int s = ds.tasks[t0 + team];
            if (fwd) {
                if (type == 1) front_fwd_team<1, true>(a, childrec, s, sm1[team], tid, team, err);
                else if (!PAIRS || type == 2) front_fwd_team<2, true>(a, childrec, s, smd, tid, team, err);
                else front_fwd_team<4, true>(a, childrec, s, smd, tid, 0, err);
            } else {
                if (type == 1) front_bwd_team<1, true, PAIRS>(a, s, sm1[team], tid, team, childrec, err, dsub);
                else if (!PAIRS || type == 2) front_bwd_team<2, true, PAIRS>(a, s, smd, tid, team, childrec, err, dsub);
                else front_bwd_team<4, true, PAIRS>(a, s, smd, tid, 0, childrec, err, dsub);
            }
        }
        __syncthreads();                                // (tk_sh is rewritten by the next claim)
    }
    solve_dep_finish(a.x, n, 1, err, ctl, slots, nslot);
}

__global__ void __launch_bounds__(128, 6) k_solve_dep(SolveArgs a, const ChildRec* childrec, DepSched ds, int* err, int* ctl, int n,
                                                   double* slots, int64_t nslot) {
    solve_dep_body<false>(a, childrec, ds, err, ctl, n, slots, nslot, nullptr);
}

__global__ void __launch_bounds__(128, 6) k_solve_dep_pairs(SolveArgs a, const ChildRec* childrec, DepSched ds, int* err, int* ctl,
                                                         int n, double* slots, int64_t nslot, const double* dsub) {
    solve_dep_body<true>(a, childrec, ds, err, ctl, n, slots, nslot, dsub);
}

// k_solve_dep (PAIRS: k_solve_dep_pairs) for NR right-hand sides in one walk of the tree: the same tasks, tickets, count-out and
// time-out path; every front stages its panel, descriptors, child records and relative indices once for all NR columns, and each
// hand-off is a block slot of NR words (slot_take_block).  Column q is x + q * n; columns ncol .. NR-1 are padding, computed on zeros
// and never read from or written to x.  Each column goes through the operations of the one-column kernel in the same order, so
// column q of the result is bit-identical to a one-column solve of column q.  `slots` are the block slots (up | down | ypiv, NR words
// per index); the {ticket, CTAs out} counters are k_solve_dep's.
// (PAIRS: a minimum of one CTA per SM lifts ptxas's 128-register target, under which the four-warp class spilled 48 bytes at NR = 4;
// the static instantiations compile exactly as without the minimum)
template <int NR, bool PAIRS>
__global__ void __launch_bounds__(128, PAIRS ? 1 : 0) k_solve_dep_block(SolveArgs a, const ChildRec* childrec, DepSched ds, int* err, int* ctl, int n,
                                                         int ncol, double* slots, int64_t nslot, const double* dsub) {
    extern __shared__ __align__(16) double smd[];       // max(4 one-warp slices, 1 two-warp slice, PAIRS: 1 four-warp slice)
    double (*sm1)[SolveSmem<1, NR>::doubles] = (double (*)[SolveSmem<1, NR>::doubles])smd;
    const int ntask = 2 * ds.ngroup;
    for (;;) {
        const int t = claim_task(ctl);
        if (t >= ntask) break;
        const bool fwd = t < ds.ngroup;
        const int g = fwd ? t : ntask - 1 - t;
        const int type = ds.grp_type[g], t0 = ds.grp_ptr[g], cnt = ds.grp_ptr[g + 1] - t0;
        int team, tid;
        group_team<false>(type, team, tid);
        if constexpr (PAIRS) {                          // (type 4 after the others: group_team<true> compiles this kernel differently)
            if (type == 4) { team = 0; tid = threadIdx.x; }
        }
        if (team < cnt) {
            const int s = ds.tasks[t0 + team];
            if (fwd) {
                if (type == 1) front_fwd_team<1, true, NR>(a, childrec, s, sm1[team], tid, team, err, ncol, n);
                else if constexpr (PAIRS) {
                    if (type == 4) front_fwd_team<4, true, NR>(a, childrec, s, smd, tid, 0, err, ncol, n);
                    else front_fwd_team<2, true, NR>(a, childrec, s, smd, tid, team, err, ncol, n);
                } else front_fwd_team<2, true, NR>(a, childrec, s, smd, tid, team, err, ncol, n);
            } else {
                if (type == 1) front_bwd_block<1, PAIRS, NR>(a, s, sm1[team], tid, team, childrec, err, dsub, ncol, n);
                else if constexpr (PAIRS) {
                    if (type == 4) front_bwd_block<4, PAIRS, NR>(a, s, smd, tid, 0, childrec, err, dsub, ncol, n);
                    else front_bwd_block<2, PAIRS, NR>(a, s, smd, tid, team, childrec, err, dsub, ncol, n);
                } else front_bwd_block<2, PAIRS, NR>(a, s, smd, tid, team, childrec, err, dsub, ncol, n);
            }
        }
        __syncthreads();                                // (tk_sh is rewritten by the next claim)
    }
    solve_dep_finish(a.x, n, ncol, err, ctl, slots, nslot);
}

}  // namespace b2
