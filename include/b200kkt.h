/*
 * b200kkt.h -- C ABI of the H100-native KKT hot path (assembly -> LDL^T + inertia -> solve).
 *
 * This is the drop-in boundary a MadNLP.jl maintainer binds with `ccall` (see INTEGRATION.md
 * and madnlp.jl_b200/julia/B200KKT.jl).  Plain pointers and sizes only; no exceptions cross
 * the boundary: every entry point returns a status code (B2_OK == 0) and b2_last_error()
 * gives the message.  All matrix values are fp64; all sparse indices are 0-based int32
 * (the reference uses 1-based Int32: src/KKT/Sparse/augmented.jl:20, condensed.jl:11,17);
 * COO->CSC maps are int64 like the reference's Vector{Int} (src/matrixtools.jl:91).
 *
 * Pointer suffix convention:  *_h = host memory,  *_d = device memory (cuda:current).
 * `stream` arguments are a cudaStream_t passed as void* (NULL = legacy default stream).
 *
 * Reference interface each group replaces (paths relative to MadNLP.jl @ v0.10.1):
 *   b2_*  sparse solver  : AbstractLinearSolver surface, src/LinearSolvers/linearsolvers.jl:13-95,
 *                          as implemented by CUDSSSolver lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cudss.jl:88-214
 *                          and Ma97Solver lib/MadNLPHSL/src/ma97.jl:29-115.
 *   b2d_* dense solver   : LapackCUDASolver/LapackCPUSolver, src/LinearSolvers/lapack.jl:164-172,
 *                          lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cusolver.jl:150-187.
 *   b2_coo_to_csc, b2_transfer*          : src/matrixtools.jl:55-95, lib/MadNLPGPU/src/KKT/gpu_sparse.jl:260-302,
 *                                          kernels_sparse.jl:161-167.
 *   b2_condensed_*                       : src/KKT/Sparse/condensed.jl:201-366, gpu_sparse.jl:308-340.
 *   b2d_condensed_assemble               : src/KKT/Dense/condensed.jl:120-186, kernels_dense.jl:81-119.
 *   b2d_aug_assemble, b2d_copy_diag      : src/KKT/Dense/augmented.jl:116-161, kernels_dense.jl:39-75.
 *   b2_set_aug_diagonal_unreduced,
 *   b2_unreduced_solve_pre / _post       : src/IPM/kernels.jl:29-34, src/IPM/factorization.jl:29-39.
 *   b2_set_aug_diagonal .. b2_kkt_mul_*  : src/IPM/kernels.jl:4-27,161-204, src/IPM/factorization.jl:41-46,
 *                                          143-167,190-237,303-324, src/KKT/KKTsystem.jl:222-226.
 */
#ifndef B200KKT_H
#define B200KKT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK                 0
#define B2_ERR_INVALID        1   /* bad argument */
#define B2_ERR_CUDA           2   /* CUDA runtime error (message in b2_last_error) */
#define B2_ERR_SYMBOLIC       3   /* analysis failed         (SymbolicException,      linearsolvers.jl:133) */
#define B2_ERR_FACTORIZATION  4   /* numeric failure         (FactorizationException, linearsolvers.jl:134) */
#define B2_ERR_SOLVE          5   /* solve before factorize  (SolveException,         linearsolvers.jl:135) */
#define B2_ERR_NO_DEVICE      6   /* no CUDA device: the product path has no CPU fallback */
#define B2_ERR_UNSUPPORTED    7   /* the driver refuses a feature the entry needs (e.g. CUDA graph conditional nodes) */

#define B2_ORDER_METIS_ND 0   /* nested dissection (METIS_NodeND, statically linked)        */
#define B2_ORDER_MINDEG   1   /* built-in minimum-degree                                    */
#define B2_ORDER_NATURAL  2   /* identity                                                   */
#define B2_ORDER_USER     3   /* caller-supplied permutation (cf. cudss_perm, cudss.jl:7)   */

const char* b2_last_error(void);
int b2_version(void);
/* number of visible CUDA devices; B2_ERR_NO_DEVICE if none */
int b2_device_count(int* count);

/* ------------------------------------------------------------------ options */
typedef struct b2_options {
    int32_t ordering;        /* B2_ORDER_*                                              */
    int32_t nemin;           /* supernode amalgamation: always merge while width <= nemin */
    double  relax_zeros;     /* additionally merge when explicit-zero fraction below this */
    double  pivot_eps;       /* |d| < pivot_eps -> static perturbation, counted as "zero"  */
    int32_t use_cuda_graph;  /* 1: capture factor/solve launch sequences into CUDA graphs  */
    int32_t small_front_max; /* fronts with order <= this run in the fused shared-memory kernel */
    int32_t n_parts;         /* multi-GPU: number of ranks sharing the elimination tree (1 = off) */
    int32_t part_rank;       /* multi-GPU: this rank                                        */
    int32_t kkt_n_primal;    /* > 0: the matrix is an augmented KKT system [[H, J'],[J, -D]] whose first kkt_n_primal
                                rows are primal; the ordering then eliminates every dual row only after one of its
                                primal neighbours, so that a zero (2,2) block never yields a structurally zero pivot */
    int32_t fuse_max_fronts; /* bottom elimination subtrees with at most this many (warp-class) fronts run inside ONE
                                CTA of a single launch (0 = plain level-by-level schedule)                      */
    int32_t dep_schedule;    /* bit 0 (default 1): for a single-part solver whose fronts are all team-class (order <= 64),
                                the factorisation and b2_solve each run as ONE launch whose CTAs wait on completion
                                flags instead of on kernel boundaries (b2_solve: one launch per right-hand side, with
                                the same arithmetic as the level-launch solve).  0: level-by-level launches.  Other
                                bits are ignored (earlier flag-driven sweep variants)                            */
    int32_t chain_merge_f;   /* > 0: a supernode with exactly ONE child absorbs it whatever the explicit zeros cost, as long as the
                                merged front stays team-class (order <= min(chain_merge_f, 64)): on latency-bound trees every
                                level of the critical path costs microseconds of hand-off besides its pivots, the zeros nothing.
                                Default 0 = off (measured slower on the OPF trees: the single-child chains sit at the bottom, where the
                                tree is throughput-bound and bigger leaves hurt); kept as an option for trees with long chains on top */
    int32_t kkt_n_dual;      /* with kkt_n_primal > 0: rows [kkt_n_primal, kkt_n_primal + kkt_n_dual) are constraint duals and every
                                later row is a bound dual of the unreduced KKT system (src/KKT/Sparse/unreduced.jl): a row with exactly
                                one off-diagonal entry, in a primal column.  The ordering places each bound row immediately before
                                its primal neighbour, so that it is eliminated first and adds its barrier term to that variable's
                                pivot.  0 (default): every non-primal row is a constraint dual.  Ignored with B2_ORDER_USER. */
    int32_t dense_pivoting;  /* dense solver (b2d_*) only, B2_DENSE_PIVOT_*: STATIC (default) eliminates in natural order with
                                |d| < pivot_eps -> +-pivot_eps; BUNCH_KAUFMAN uses LAPACK dsytrf('L')'s pivot sequence (1x1 and
                                2x2 pivots, symmetric interchanges) and exact inertia (MadNLP's lapack_algorithm = BUNCHKAUFMAN).
                                The sparse solver (b2_create*) rejects any value but STATIC.  BUNCH_KAUFMAN needs
                                N <= 128 * (number of SMs of the device), 16,896 on an H100 SXM: its solve is one launch
                                with one resident CTA per 128 rows; b2d_create rejects a larger N (B2_ERR_INVALID).      */
    int32_t sparse_pivoting; /* sparse solver (b2_*) only, B2_SPARSE_PIVOT_*: STATIC (default) pivots 1x1 with |d| < pivot_eps ->
                                +-pivot_eps.  PAIRS: the analysis places every constraint dual it can match with a distinct primal
                                neighbour immediately after that neighbour, in one supernode, and the factorisation takes the pair as
                                one 2x2 pivot block when |a_kk| < alpha |a_k+1,k| (alpha = (1+sqrt(17))/8) and the block is indefinite,
                                else as two 1x1 pivots (DESIGN.md section 3).  No rows move at run time.  b2_create accepts PAIRS only
                                with kkt_n_primal > 0, n_parts == 1, dep_schedule bit 0 set and every front of order <= 96 after the
                                analysis (fronts of order 65..96 run as four-warp teams) (B2_ERR_INVALID otherwise, before any device work; b2_create_symbolic_only skips the front-order
                                condition so that tooling can inspect the tree).  The dense solver (b2d_create) rejects any value but
                                STATIC.                                                                                    */
    int32_t dense_algorithm; /* dense solver (b2d_*) only, B2_DENSE_ALG_*: LDLT (default) factors A = L D L' with the pivoting chosen
                                by dense_pivoting; LU mirrors the lower triangle into the full matrix and factors it with partial
                                pivoting, LAPACK dgetrf's pivot sequence (MadNLP's lapack_algorithm = LU).  LU reports no inertia
                                (b2d_inertia* return B2_ERR_INVALID), needs dense_pivoting = STATIC and, like BUNCH_KAUFMAN,
                                N <= 128 * (number of SMs of the device); b2d_create rejects anything else (B2_ERR_INVALID).
                                The sparse solver (b2_create*) rejects any value but LDLT.                                  */
} b2_options;

#define B2_DENSE_PIVOT_STATIC        0
#define B2_DENSE_PIVOT_BUNCH_KAUFMAN 1
#define B2_DENSE_ALG_LDLT            0
#define B2_DENSE_ALG_LU              1
#define B2_SPARSE_PIVOT_STATIC       0
#define B2_SPARSE_PIVOT_PAIRS        1

/* pivot kinds reported by b2_get_pivot_blocks */
#define B2_PIVOT_1X1            0
#define B2_PIVOT_1X1_PERTURBED  1
#define B2_PIVOT_2X2_FIRST      2
#define B2_PIVOT_2X2_SECOND     3

int b2_options_default(b2_options* opt);

/* ------------------------------------------------------------------ sparse LDL^T */
typedef struct b2_solver b2_solver;

typedef struct b2_stats {
    int64_t n, nnz_a, nnz_l, flops;        /* nnz(L) incl. diagonal and explicit zeros; flops of one factorisation */
    int64_t n_supernodes, n_levels;
    int64_t max_front, n_small_fronts, n_big_fronts;
    int64_t factor_bytes, workspace_bytes; /* device memory held */
    int64_t sep_rows;                      /* multi-GPU: order of the shared (replicated) top tree */
    int64_t n_factor_launches, n_solve_launches;
    int64_t n_perturbed;                   /* pivots perturbed in the last factorisation */
} b2_stats;

/* Analysis (ordering + symbolic factorisation); `nzval_d` is KEPT BY REFERENCE and re-read by
 * every b2_factorize -- the reference's aliasing contract (cudss.jl:154-158, ma97.jl:72-88).
 * colptr_h[n+1], rowval_h[nnz]: lower-triangular CSC pattern on the host, 0-based.
 * user_perm_h: n entries (perm[new]=old) when ordering == B2_ORDER_USER, else NULL. */
int b2_create(int32_t n, int64_t nnz, const int32_t* colptr_h, const int32_t* rowval_h,
              const double* nzval_d, const b2_options* opt, const int32_t* user_perm_h,
              b2_solver** out);
/* analysis only (no device state): for tooling/tests on machines without a GPU; every numeric entry point
 * returns B2_ERR_INVALID on such a handle -- it is NOT a compute fallback. */
int b2_create_symbolic_only(int32_t n, int64_t nnz, const int32_t* colptr_h, const int32_t* rowval_h,
                            const b2_options* opt, const int32_t* user_perm_h, b2_solver** out);
int b2_destroy(b2_solver* s);
/* re-point the aliased value buffer (same pattern) */
int b2_set_values_ptr(b2_solver* s, const double* nzval_d);
/* numeric factorisation of the CURRENT values; asynchronous on `stream` */
int b2_factorize(b2_solver* s, void* stream);
/* (num_pos, num_zero, num_neg) in the reference's code order (src/IPM/solver.jl:626);
 * synchronises `stream`.  Perturbed pivots are reported as zeros (cf. mumps.jl:248-250). */
int b2_inertia(b2_solver* s, int64_t* num_pos, int64_t* num_zero, int64_t* num_neg, void* stream);
/* the same read split in two so that a caller can queue more work behind the factorisation before it blocks:
 * b2_inertia_enqueue() queues the 32-byte D2H copy on `stream`; after the caller has synchronised that stream,
 * b2_inertia_fetch() returns the counts without touching the device.  (b2_inertia == enqueue + synchronise + fetch.) */
int b2_inertia_enqueue(b2_solver* s, void* stream);
int b2_inertia_fetch(b2_solver* s, int64_t* num_pos, int64_t* num_zero, int64_t* num_neg);
/* in-place x <- K^{-1} x, nrhs columns of length n (ld = n); asynchronous on `stream` */
int b2_solve(b2_solver* s, double* x_d, int32_t nrhs, void* stream);
/* raise robustness after a failed refinement (improve!, linearsolvers.jl / ma97.jl:103-111);
 * *changed = 1 if something changed and a re-factorisation is worthwhile */
int b2_improve(b2_solver* s, int32_t* changed);
int b2_get_stats(b2_solver* s, b2_stats* st);
/* copy out the fill-reducing permutation (perm[new]=old), n entries, host */
int b2_get_perm(b2_solver* s, int32_t* perm_h);

/* Multi-GPU (subtree-to-rank) support.  With opt.n_parts = P > 1 every rank analyses the same
 * pattern; rank r factors the subtrees it owns plus (replicated) the shared top tree.  The only
 * exchange is the sum of the subtree roots' update (Schur-complement) blocks, which the host
 * reduces with NCCL:   b2_factorize_local -> allreduce(b2_exchange_buffer) -> b2_factorize_top.
 * b2_solve_* mirror this for the triangular solves (the exchange buffer then holds vectors). */
int b2_exchange_buffer(b2_solver* s, double** buf_d, int64_t* n_factor_doubles, int64_t* n_solve_doubles);
int b2_exchange_vector(b2_solver* s, double** buf_d, int64_t* n_doubles);   /* forward-solve contributions */
/* inertia split for the multi-GPU reduction: counts of the owned subtrees and of the replicated top tree */
int b2_inertia_parts(b2_solver* s, int64_t* local_neg, int64_t* local_zero, int64_t* top_neg, int64_t* top_zero, void* stream);
int b2_factorize_local(b2_solver* s, void* stream);
int b2_factorize_top(b2_solver* s, void* stream);
int b2_solve_fwd_local(b2_solver* s, double* x_d, void* stream);
int b2_solve_top(b2_solver* s, double* x_d, void* stream);      /* after allreduce of the exchange buffer */
int b2_solve_bwd_local(b2_solver* s, double* x_d, void* stream); /* leaves x complete only on owned + top rows */
int b2_owned_mask(b2_solver* s, uint8_t* owned_h);               /* n entries: 1 if this rank finalises x[i] */

/* Debug/test export of the symbolic structure (host arrays, caller-allocated; pass NULL to query sizes):
 * used by tests/ to replay the multifrontal arithmetic in numpy on machines without a GPU. */
typedef struct b2_symbolic_sizes {
    int64_t n, n_supernodes, n_rows, n_children, n_rel, n_amap, n_levels, lval_size, cb_size;
} b2_symbolic_sizes;
int b2_symbolic_query(b2_solver* s, b2_symbolic_sizes* sz);
int b2_symbolic_export(b2_solver* s, int32_t* perm, int32_t* sn_first, int32_t* sn_parent, int32_t* sn_level,
                       int64_t* rows_ptr, int32_t* rows, int64_t* lp_off, int64_t* cb_off,
                       int64_t* rel_ptr, int32_t* rel, int64_t* amap_ptr, int64_t* amap_src, int64_t* amap_dst);
int b2_symbolic_owner(b2_solver* s, int32_t* owner);   /* n_supernodes entries: rank, or -1 for the shared top tree */
/* layout of the multi-GPU exchange: contribution-vector offsets (n_supernodes+1) and the sizes (in doubles) of the
 * leading regions of the update-block / contribution-vector workspaces that are all-reduced */
int b2_symbolic_exchange(b2_solver* s, int64_t* cbv_off, int64_t* exch_cb, int64_t* exch_cbv);
/* test/debug: copy the numeric factor (lval_size doubles, panel layout of b2_symbolic_export) and D (n doubles, permuted
 * order) to the host; synchronises the device. */
int b2_debug_get_factor(b2_solver* s, double* lval_h, double* dvec_h);
/* analysis export of opt.sparse_pivoting = B2_SPARSE_PIVOT_PAIRS: pair_start_h[j] = 1 when permuted column j starts a candidate pair
 * (j, j+1) -- a primal followed by its matched constraint dual, both in one supernode -- else 0; n entries.  All zero for STATIC. */
int b2_symbolic_pairs(b2_solver* s, uint8_t* pair_start_h);
/* test/debug: the pivots of the last factorisation of a PAIRS handle in elimination (permuted) order, n entries each on the host:
 * kind_h B2_PIVOT_*; d_h D's diagonal (a perturbed pivot as +-pivot_eps); d_off_h D's subdiagonal (b at the first index of a 2x2
 * block, else 0).  Synchronises the device; B2_ERR_INVALID on a STATIC handle. */
int b2_get_pivot_blocks(b2_solver* s, int8_t* kind_h, double* d_h, double* d_off_h);
/* test/debug: re-factor one warp-class front `reps` times with clock64() stamps at its 8 phase boundaries */
int b2_debug_profile_front(b2_solver* s, int32_t sn, int32_t reps, int64_t* stamps_h);
/* Debug: per-front device timeline of the team-class factor kernels.  With B2_SPARSE_TRACE=1 in the environment at b2_create every
 * front of order <= 64 stamps %globaltimer (ns) when its team starts, when its children have been assembled and when it has
 * finished: stamps_h[3 * sn + {0,1,2}].  Also returns the supernode parents and (w, f) of every front.  *count = number of
 * supernodes; data is copied when capacity >= *count (stamps are zero when tracing is off). */
int b2_debug_trace(b2_solver* s, uint64_t* stamps_h, int32_t* parent_h, int32_t* w_h, int32_t* f_h, int64_t capacity, int64_t* count);
/* Debug: per-front device timeline of the single-launch solve, under the same B2_SPARSE_TRACE=1 switch.  Each front stamps
 * %globaltimer (ns) for its forward and its backward task: when the task is claimed, when its inputs have arrived (children's
 * contributions / ancestor values and own forward result) and when it has handed its outputs on: stamps_h[6 * sn + {0,1,2}]
 * forward, {3,4,5} backward, as left by the last solve.  *count = number of uint64 values (0 when tracing is off); stamps are
 * copied when capacity >= *count. */
int b2_debug_trace_solve(b2_solver* s, uint64_t* stamps_h, int64_t capacity, int64_t* count);
/* Debug (also on a symbolic-only handle): the ticket order of the single-launch factorisation and solve (dep_schedule bit 0, used
 * when every front has order <= 64, or <= 96 with sparse_pivoting = PAIRS) over this rank's supernodes: depth from the root descending, then level, then id.  *count =
 * number of supernodes in it; order_h is filled when capacity >= *count (may be NULL). */
int b2_debug_dep_order(b2_solver* s, int32_t* order_h, int64_t capacity, int64_t* count);

/* ------------------------------------------------------------------ dense LDL^T */
typedef struct b2d_solver b2d_solver;
/* A_d: N x N column-major (ld = lda) on the device, lower triangle read, KEPT BY REFERENCE
 * (lapack.jl:40); the factor is written to an internal buffer (lapack_common.jl:28). */
int b2d_create(int32_t N, int32_t lda, const double* A_d, const b2_options* opt, b2d_solver** out);
int b2d_destroy(b2d_solver* s);
/* Debug: device timeline of the dense look-ahead factorisation.  With B2_DENSE_TRACE=1 in the environment at b2d_create, every kernel
 * of b2d_factorize stamps %globaltimer (ns) at its first entry and last exit; slot = 8 * block column + kind (0 diagonal block, 1 near
 * trsm, 2 near syrk, 3 panel trsm, 4 block-column update, 5 trailing update), two uint64 per slot.  *count = number of
 * uint64 values (0 when tracing is off); stamps are copied when capacity >= *count. */
int b2d_debug_trace(b2d_solver* s, uint64_t* stamps_h, int64_t capacity, int64_t* count);
int b2d_factorize(b2d_solver* s, void* stream);
/* the three inertia entries return B2_ERR_INVALID on an LU handle (opt.dense_algorithm = B2_DENSE_ALG_LU): LU reports no inertia */
int b2d_inertia(b2d_solver* s, int64_t* num_pos, int64_t* num_zero, int64_t* num_neg, void* stream);
int b2d_inertia_enqueue(b2d_solver* s, void* stream);
int b2d_inertia_fetch(b2d_solver* s, int64_t* num_pos, int64_t* num_zero, int64_t* num_neg);
int b2d_solve(b2d_solver* s, double* x_d, int32_t nrhs, void* stream);
/* Test/debug export of a Bunch-Kaufman factor (opt.dense_pivoting = B2_DENSE_PIVOT_BUNCH_KAUFMAN) in LAPACK's convention, N entries
 * each on the host: ipiv_h 1-based (a 1x1 pivot interchanged row k with ipiv[k]; -kp on both rows of a 2x2 block), d_h D's diagonal,
 * e_h D's subdiagonal (0 for a 1x1 pivot, d21 at the first index of a 2x2 block).  A zero column is reported with its perturbed
 * pivot +-pivot_eps.  Synchronises the device; B2_ERR_INVALID on a static-pivoting handle. */
int b2d_get_pivots(b2d_solver* s, int32_t* ipiv_h, double* d_h, double* e_h);
/* Export of an LU factor (opt.dense_algorithm = B2_DENSE_ALG_LU) as LAPACK dgetrf leaves it, on the host: ipiv_h (N entries,
 * 1-based: row k was interchanged with row ipiv[k]), *info_h (the first exactly-zero pivot of U, 1-based, else 0) and lu_h (N x N
 * column-major, unit-lower L below the diagonal, U on and above it).  Any pointer may be NULL.  Synchronises the device;
 * B2_ERR_SOLVE if a device-wide wait of the factorisation or of a solve timed out, B2_ERR_INVALID on an LDLT handle. */
int b2d_get_lu(b2d_solver* s, int32_t* ipiv_h, int32_t* info_h, double* lu_h);

/* ------------------------------------------------------------------ assembly: COO -> CSC */
/* Host, one-time: CSC pattern of a COO matrix with duplicate merging and the COO->CSC map
 * (src/matrixtools.jl:55-95).  colptr_h[n+1]; rowval_h capacity nnz_coo; map_h[nnz_coo]. */
int b2_coo_to_csc(int32_t m, int32_t n, int64_t nnz_coo, const int32_t* I_h, const int32_t* J_h,
                  int32_t* colptr_h, int32_t* rowval_h, int64_t* map_h, int64_t* nnz_csc);

/* The same construction with device sorts (lib/MadNLPGPU/src/KKT/gpu_sparse.jl:260-302): I_d, J_d, and all outputs are DEVICE arrays
 * (rowval_d capacity nnz_coo); identical output to b2_coo_to_csc.  Synchronises `stream` once to return *nnz_csc. */
int b2_coo_to_csc_device(int32_t m, int32_t n, int64_t nnz_coo, const int32_t* I_d, const int32_t* J_d,
                         int32_t* colptr_d, int32_t* rowval_d, int64_t* map_d, int64_t* nnz_csc, void* stream);

/* Device plan for  dst .= 0; dst[map[k]] += V[k]  (src/matrixtools.jl:79-88) as a race-free,
 * deterministic segmented gather: one thread per destination slot summing its sources in COO
 * order -- bit-identical to the reference's sequential CPU loop. */
typedef struct b2_transfer_plan b2_transfer_plan;
int b2_transfer_plan_create(int64_t nnz_coo, int64_t nnz_csc, const int64_t* map_h, b2_transfer_plan** out);
int b2_transfer_plan_destroy(b2_transfer_plan* p);
int b2_transfer(b2_transfer_plan* p, double* dst_nz_d, const double* V_d, void* stream);

/* ------------------------------------------------------------------ assembly: sparse condensed */
typedef struct b2_condensed_plan b2_condensed_plan;
/* Symbolic (host, one-time): pattern of tril(H) U diag U tril(Jt*Jt') and the dptr/hptr/jptr maps
 * (src/KKT/Sparse/condensed.jl:201-301).  H: n x n lower CSC; Jt: n x m CSC. */
int b2_condensed_symbolic(int32_t n, int32_t m,
                          const int32_t* H_colptr_h, const int32_t* H_rowval_h,
                          const int32_t* Jt_colptr_h, const int32_t* Jt_rowval_h,
                          b2_condensed_plan** out, int64_t* nnz_aug);
/* the same construction with device sorts (condensed.jl:251 on the GPU, lib/MadNLPGPU/src/KKT/gpu_sparse.jl:100-130): patterns are
 * DEVICE arrays; the resulting plan is identical to b2_condensed_symbolic's.  Synchronises `stream`. */
int b2_condensed_symbolic_device(int32_t n, int32_t m,
                                 const int32_t* H_colptr_d, const int32_t* H_rowval_d,
                                 const int32_t* Jt_colptr_d, const int32_t* Jt_rowval_d,
                                 b2_condensed_plan** out, int64_t* nnz_aug, void* stream);
int b2_condensed_pattern(b2_condensed_plan* p, int32_t* colptr_h, int32_t* rowval_h);
int b2_condensed_plan_sizes(b2_condensed_plan* p, int64_t* n_dptr, int64_t* n_hptr, int64_t* n_jptr);
int b2_condensed_plan_destroy(b2_condensed_plan* p);
/* Numeric (device, every iteration), two launches instead of the reference's fill! + 3 kernels
 * (src/KKT/Sparse/condensed.jl:328-366, gpu_sparse.jl:308-340):
 *   diag_buffer = Ss ./ (1 - Sd .* Ss)   with Ss = pr_diag[n:n+m], Sd = du_diag
 *   nz[i] = sum H.nz[..] + pr_diag[..] + sum diag_buffer[c]*Jt.nz[k]*Jt.nz[l]
 * summed per slot in the reference's order (hess, diag, triples) without FMA contraction. */
int b2_condensed_assemble(b2_condensed_plan* p, double* aug_nz_d, const double* pr_diag_d,
                          const double* du_diag_d, const double* H_nz_d, const double* Jt_nz_d,
                          double* diag_buffer_d, void* stream);

/* ------------------------------------------------------------------ assembly: dense condensed */
/* src/KKT/Dense/condensed.jl:157-186.  hess n x n (ld n), jac m x n (ld m), aug N x N (ld N), N = n + n_eq.
 * Only the LOWER triangle of aug is written (what dsytrf('L') and b2d_* read), plus the equality rows. */
int b2d_condensed_assemble(int32_t n, int32_t m, int32_t ns, int32_t n_eq,
                           const int64_t* ind_ineq_d, const int64_t* ind_eq_d,
                           const double* hess_d, const double* jac_d,
                           const double* pr_diag_d, const double* du_diag_d,
                           double* diag_buffer_d, double* aug_d, void* stream);

/* ------------------------------------------------------------------ assembly: dense augmented */
/* src/KKT/Dense/augmented.jl:116-156.  hess n x n (ld n; strict lower triangle read), jac m x n (ld m),
 * aug N x N (ld N), N = n + ns + m, ind_ineq 0-based (ns entries).  Writes EVERY element of the lower triangle of aug
 * (structural zeros included) and nothing above the diagonal. */
int b2d_aug_assemble(int32_t n, int32_t m, int32_t ns, const int64_t* ind_ineq_d,
                     const double* hess_d, const double* jac_d, const double* pr_diag_d,
                     const double* du_diag_d, const double* diag_hess_d, double* aug_d, void* stream);
/* compress_hessian!(::DenseKKTSystem) = diag!(diag_hess, hess)  (augmented.jl:158-161): d[i] = A[i, i], i < n */
int b2d_copy_diag(int32_t n, int32_t lda, const double* A_d, double* d_d, void* stream);

/* The same assembly with the J' D J contraction on the Hopper tensor cores: fp64 is cut into 8 signed 7-bit digits per entry
 * (Ozaki scheme) and the 36 digit-pair products run as exact int8 GEMMs on wgmma.mma_async (s8) with TMA-staged operands
 * (csrc/ozaki_kernels.cuh).  Entry by entry, with a = sqrt(D) J_I and e_m the frexp exponent of max_i |a_im|:
 *   |W^ - W|_mn <= 2^-51 ns 2^(e_m + e_n) + 2^-52 (|W| + |H_mn| + |pr_m|)
 * from the truncation of each entry below 2^-56 of its column's maximum, the digit pairs s + t >= 8 that are never multiplied
 * (2^-53.2 per term) and the fp64 Horner sum; results under- and overflow as the fp64 contraction's do, and a column holding
 * a NaN or an Inf gives NaN in its row and column (tests/test_gpu_dense_assembly_entrywise.py).  The plan owns the digit planes (8 * n_pad * ns_pad bytes), exponents, tile list and tensor maps.
 * ns <= 16384.  b2d_ozaki_plan_status reports whether a (bounded) pipeline wait ever timed out. */
typedef struct b2d_ozaki_plan b2d_ozaki_plan;
int b2d_ozaki_plan_create(int32_t n, int32_t ns, b2d_ozaki_plan** out);
int b2d_ozaki_plan_destroy(b2d_ozaki_plan* p);
int b2d_condensed_assemble_ozaki(b2d_ozaki_plan* p, int32_t n, int32_t m, int32_t ns, int32_t n_eq,
                                 const int64_t* ind_ineq_d, const int64_t* ind_eq_d,
                                 const double* hess_d, const double* jac_d,
                                 const double* pr_diag_d, const double* du_diag_d,
                                 double* diag_buffer_d, double* aug_d, void* stream);
int b2d_ozaki_plan_status(b2d_ozaki_plan* p, int32_t* timed_out, void* stream);

/* dense mat-vecs on column-major device matrices for the DenseCondensedKKTSystem wrappers (jtprod!/mul!/solve_kkt!,
 * src/IPM/factorization.jl:190-229,326-344; the reference calls cuBLAS gemv/symv, lib/MadNLPGPU/.../cuda.jl:54-84):
 *   gemv_n: y = alpha*A*x + beta*y (A rows x cols, ld = lda)   gemv_t: y = alpha*A'*x + beta*y
 *   symv_lower: y = alpha*sym(A)*x + beta*y reading only the lower triangle (the reference's _symv!('L', ...)) */
int b2d_gemv_n(int32_t rows, int32_t cols, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);
int b2d_gemv_t(int32_t rows, int32_t cols, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);
int b2d_symv_lower(int32_t n, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);

/* solve_kkt!(::DenseCondensedKKTSystem, w) (src/IPM/factorization.jl:190-229) and mul!(w, ::AbstractDenseKKTSystem, x, alpha, beta)
 * (:303-324) around b2d_solve.  `b2d_kkt` holds ind_ineq (host, 0-based, ns entries), the derived ind_eq and their inverse map on
 * the device.  jac: m x n column-major (ld m); hess: n x n (lower triangle read, ld n); pd_buffer: n + n_eq; buffer: m;
 * w, x: UnreducedKKTVector buffers [x (n) s (ns) | y (m) | zl | zu].
 *   pre : reduce_rhs!; buffer = 0; buffer[ind_ineq] = D .* (wz + ws ./ Ss); xx = jac' * buffer + wx; xy = wy
 *   (caller: b2d_solve(pd_buffer))
 *   post: wx = xx; dual(w) = jac * wx; wy = xy; wz .*= D; dual(w) .-= buffer; ws = (ws + wz) ./ Ss; finish_aug_solve! */
typedef struct b2_bounds b2_bounds;   /* created by b2_bounds_create, below */
typedef struct b2d_kkt b2d_kkt;
int b2d_kkt_create(int32_t n, int32_t m, int32_t ns, const int64_t* ind_ineq_h, b2d_kkt** out);
int b2d_kkt_destroy(b2d_kkt* k);
int b2d_kkt_solve_pre(b2d_kkt* k, b2_bounds* b, const double* jac_d, const double* pr_diag_d, const double* diag_buffer_d,
                      const double* l_diag_d, const double* u_diag_d, double* buffer_d, double* pd_buffer_d, double* w_d, void* stream);
int b2d_kkt_solve_post(b2d_kkt* k, b2_bounds* b, const double* jac_d, const double* pr_diag_d, const double* diag_buffer_d,
                       const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                       const double* buffer_d, const double* pd_buffer_d, double* w_d, void* stream);
int b2d_kkt_mul(b2d_kkt* k, b2_bounds* b, const double* hess_d, const double* jac_d, const double* reg_d, const double* du_diag_d,
                const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                double alpha, double beta, const double* x_d, double* w_d, void* stream);

/* ------------------------------------------------------------------ IPM vector kernels */
/* Index sets ind_lb / ind_ub over the primal vector (x,s) (src/Callbacks/nlpmodels.jl:369-406), uploaded once
 * together with their inverse maps so that every kernel below is a single race-free pass over n_tot. */
typedef struct b2_bounds b2_bounds;
int b2_bounds_create(int64_t n_tot, int64_t nlb, int64_t nub, const int64_t* ind_lb_h, const int64_t* ind_ub_h,
                     b2_bounds** out);
int b2_bounds_destroy(b2_bounds* b);

/* pr_diag = reg; pr_diag[ind_lb] -= l_lower./l_diag; pr_diag[ind_ub] -= u_lower./u_diag  (IPM/kernels.jl:22-27) */
int b2_set_aug_diagonal(b2_bounds* b, const double* reg_d, const double* l_lower_d, const double* l_diag_d,
                        const double* u_lower_d, const double* u_diag_d, double* pr_diag_d, void* stream);
/* SparseUnreducedKKTSystem (src/KKT/Sparse/unreduced.jl).  _set_aug_diagonal!(::AbstractUnreducedKKTSystem) (IPM/kernels.jl:29-34)
 * as one launch:  pr_diag = reg (n_tot);  l_lower_aug = sqrt(l_lower) (nlb);  u_lower_aug = sqrt(u_lower) (nub), correctly rounded */
int b2_set_aug_diagonal_unreduced(int64_t n_tot, int64_t nlb, int64_t nub, const double* reg_d, const double* l_lower_d,
                                  const double* u_lower_d, double* pr_diag_d, double* l_lower_aug_d, double* u_lower_aug_d,
                                  void* stream);
/* solve_kkt!(::SparseUnreducedKKTSystem) (IPM/factorization.jl:29-39) around b2_solve on the FULL vector
 * w = [x (n_tot) | y (m) | zl (nlb) | zu (nub)]:
 *   pre : wzl = iszero(l_lower_aug) ? wzl : wzl / l_lower_aug ; the same for wzu   (-0.0 counts as zero)
 *   post: wzl = wzl * (-l_lower_aug) ; wzu = wzu * u_lower_aug */
int b2_unreduced_solve_pre(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* l_lower_aug_d,
                           const double* u_lower_aug_d, double* w_d, void* stream);
int b2_unreduced_solve_post(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* l_lower_aug_d,
                            const double* u_lower_aug_d, double* w_d, void* stream);
/* ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl): the augmented system under the congruence by the scaling factor
 * s = sqrt((x - xl)(xu - x)) over the bounds a variable has.  Here l_diag = x - xl and u_diag = xu - x, both positive (the opposite
 * sign of the reduced systems').  One launch each, one thread per variable (b2_bounds' inverse maps), no atomics; every formula is
 * evaluated with rounding intrinsics in the reference's order, so the results are bit-identical to its broadcasts.
 *   b2_scaled_set_aug_diagonal   _set_aug_diagonal! (IPM/kernels.jl:47-68): s = (1 * sqrt(l_diag)) * sqrt(u_diag) (factors of the
 *                                bounds present), pr_diag = (xlzu + xuzl) + reg * (s * s) with xlzu = u_lower * l_diag, xuzl = l_lower *
 *                                u_diag (0 for a missing multiplier, times the other bound's distance when there is one); scaling = s
 *   b2_scaled_transfer           build_kkt! (scaled_augmented.jl:209-236) on aug_com: transfer! through the plan of the K2 COO layout
 *                                with each source scaled before the slot's sum (pr_diag and du_diag sources by 1, Hessian sources
 *                                (v s_i) s_j, Jacobian and slack sources v s_j).  colptr / rowval: aug_com's pattern on the device, n columns
 *   b2_scaled_solve_pre / _post  solve_kkt! (IPM/factorization.jl:48-74) around b2_solve on primal_dual(w):
 *                                pre xp = xp s + (r3 + r4); post xp = xp s, wzl = (wzl - l_lower xp) / l_diag,
 *                                wzu = (-wzu + u_lower xp) / u_diag
 *   b2_scaled_kktmul             mul!'s diagonal and bound part (IPM/factorization.jl:239-251), after the three SpMVs of b2_kktmul's
 *                                callers: the bound rows take + xzl l_diag and - xzu u_diag
 *   b2_scaled_regularize_diagonal regularize_diagonal! (scaled_augmented.jl:238-242): reg += dw; pr_diag += dw (s s); du_diag -= dc */
int b2_scaled_set_aug_diagonal(b2_bounds* b, const double* reg_d, const double* l_lower_d, const double* l_diag_d,
                               const double* u_lower_d, const double* u_diag_d, double* pr_diag_d, double* scaling_d, void* stream);
int b2_scaled_transfer(b2_transfer_plan* p, int64_t n, int64_t n_tot, const int32_t* colptr_d, const int32_t* rowval_d,
                       const double* scaling_d, double* dst_nz_d, const double* V_d, void* stream);
int b2_scaled_solve_pre(b2_bounds* b, int64_t m, const double* l_diag_d, const double* u_diag_d, const double* scaling_d, double* w_d,
                        void* stream);
int b2_scaled_solve_post(b2_bounds* b, int64_t m, const double* l_lower_d, const double* u_lower_d, const double* l_diag_d,
                         const double* u_diag_d, const double* scaling_d, double* w_d, void* stream);
int b2_scaled_kktmul(b2_bounds* b, int64_t m, const double* reg_d, const double* du_diag_d, const double* l_lower_d,
                     const double* u_lower_d, const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                     const double* x_d, double* w_d, void* stream);
int b2_scaled_regularize_diagonal(int64_t n_tot, int64_t m, double dw, double dc, const double* scaling_d, double* reg_d,
                                  double* pr_diag_d, double* du_diag_d, void* stream);
/* reg += dw; pr_diag += dw; du_diag -= dc   (KKTsystem.jl:222-226) */
int b2_regularize_diagonal(int64_t n_tot, int64_t m, double dw, double dc, double* reg_d, double* pr_diag_d,
                           double* du_diag_d, void* stream);
/* reduce_rhs! / finish_aug_solve!  (IPM/kernels.jl:182-204) on an UnreducedKKTVector buffer
 * w = [xp(n_tot) | y(m) | zl(nlb) | zu(nub)]  (KKT/rhs.jl:101-117) */
int b2_reduce_rhs(b2_bounds* b, int64_t m, const double* l_diag_d, const double* u_diag_d, double* w_d, void* stream);
int b2_finish_aug_solve(b2_bounds* b, int64_t m, const double* l_lower_d, const double* u_lower_d,
                        const double* l_diag_d, const double* u_diag_d, double* w_d, void* stream);

/* CSC sparse mat-vec helpers:  y = alpha*A*x + beta*y  /  y = alpha*A'*x + beta*y  and the symmetric-lower
 * product y = alpha*(L + L' - diag(L))*x + beta*y; gather (row-parallel) forms built once per pattern --
 * replaces the cuSPARSE SpMV calls of lib/MadNLPGPU/src/KKT/gpu_sparse.jl:14-65. */
typedef struct b2_spmv_plan b2_spmv_plan;
int b2_spmv_plan_create(int32_t nrow, int32_t ncol, const int32_t* colptr_h, const int32_t* rowval_h, b2_spmv_plan** out);
int b2_spmv_plan_destroy(b2_spmv_plan* p);
int b2_spmv_n(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);
int b2_spmv_t(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);
int b2_spmv_symlower(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream);

/* _kktmul!  (IPM/kernels.jl:161-180) on UnreducedKKTVector buffers w, x */
int b2_kktmul(b2_bounds* b, int64_t m, const double* reg_d, const double* du_diag_d,
              const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
              double alpha, double beta, const double* x_d, double* w_d, void* stream);

/* solve_kkt!(::SparseCondensedKKTSystem) pre/post stages around b2_solve (IPM/factorization.jl:143-167), n = nvar, m = ncon,
 * pre in two launches, post in one:
 *   pre : reduce_rhs!; buffer = D.*(wz + ws./Ss); wx += Jt*buffer
 *   post: buffer2 = Jt'*wx; wz = -buffer + D.*buffer2; ws = (ws+wz)./Ss; finish_aug_solve! */
int b2_condensed_solve_pre(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m,
                           const double* jt_nz_d, const double* pr_diag_d, const double* diag_buffer_d,
                           const double* l_diag_d, const double* u_diag_d, double* buffer_d, double* w_d, void* stream);
int b2_condensed_solve_post(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m,
                            const double* jt_nz_d, const double* pr_diag_d, const double* diag_buffer_d,
                            const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                            const double* buffer_d, double* w_d, void* stream);
/* One Richardson step (src/LinearSolvers/backsolve.jl:45-52) of the condensed system in five launches:
 *   b2_condensed_refine_pre        (= b2_condensed_solve_pre; also norms_d[0] = norms_d[1] = 0)
 *   b2_solve on w[0:n)
 *   b2_condensed_solve_post_update (= b2_condensed_solve_post; also x += w and norms_d[1] = ||x||_inf)
 *   b2_condensed_kkt_mul_norm_y    with alpha = -1, beta = 1, y = b: w = b - K x, norms_d[0] = ||w||_inf
 * bit-identical to solve_pre -> b2_solve -> solve_post -> b2_richardson_update -> b2_condensed_kkt_mul_norm */
int b2_condensed_refine_pre(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m,
                            const double* jt_nz_d, const double* pr_diag_d, const double* diag_buffer_d,
                            const double* l_diag_d, const double* u_diag_d, double* buffer_d, double* w_d, double* norms_d, void* stream);
int b2_condensed_solve_post_update(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m,
                                   const double* jt_nz_d, const double* pr_diag_d, const double* diag_buffer_d,
                                   const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                   const double* buffer_d, double* w_d, double* x_d, double* norms_d, void* stream);
/* mul!(w, ::SparseCondensedKKTSystem, x, alpha, beta)  (IPM/factorization.jl:303-324) incl. _kktmul! */
int b2_condensed_kkt_mul(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                         const double* hess_nz_d, const double* jt_nz_d,
                         const double* reg_d, const double* du_diag_d, const double* l_lower_d, const double* u_lower_d,
                         const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                         const double* x_d, double* w_d, void* stream);
/* the same product that also accumulates ||w||_inf of its result into *norm_inf_d (device; the caller zeroes it -- 
 * b2_richardson_update does); the residual norm of a Richardson step then costs no extra pass */
int b2_condensed_kkt_mul_norm(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                         const double* hess_nz_d, const double* jt_nz_d,
                         const double* reg_d, const double* du_diag_d, const double* l_lower_d, const double* u_lower_d,
                         const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                         const double* x_d, double* w_d, double* norm_inf_d, void* stream);
/* the same with the beta term read from y (a vector other than w): w = alpha*K*x + beta*y ; ||w||_inf into *norm_inf_d */
int b2_condensed_kkt_mul_norm_y(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                           const double* hess_nz_d, const double* jt_nz_d,
                           const double* reg_d, const double* du_diag_d, const double* l_lower_d, const double* u_lower_d,
                           const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                           const double* x_d, const double* y_d, double* w_d, double* norm_inf_d, void* stream);

/* infinity norm of a device vector into a device scalar (no host sync) */
/* start of solve_refine! (src/LinearSolvers/backsolve.jl:36-44) in one pass: *norm_b_d = ||b||_inf ; x = 0 ; w = b */
int b2_richardson_begin(int64_t n, const double* b_d, double* w_d, double* x_d, double* norm_b_d, void* stream);
/* vector part of one Richardson step (src/LinearSolvers/backsolve.jl:45-48) in one pass: x += w ; w = b ;
 * norms_d[0] = 0 (accumulator for b2_condensed_kkt_mul_norm) ; norms_d[1] = ||x||_inf */
int b2_richardson_update(int64_t n, const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream);
int b2_norm_inf(int64_t n, const double* x_d, double* out_d, void* stream);
/* y += a*x ; y = x ; x = v */
int b2_axpy(int64_t n, double a, const double* x_d, double* y_d, void* stream);
int b2_copy(int64_t n, const double* x_d, double* y_d, void* stream);
/* count <= 16 independent copies dst[k][0:n[k]) = src[k][0:n[k]) in one launch (host arrays of device pointers): how the
 * outputs of the model callbacks (eval_jac_wrapper!/eval_lag_hess_wrapper!, src/IPM/callbacks.jl) and the iterate's
 * diagonals reach the KKT buffers when they are produced elsewhere on the device */
int b2_copy_many(int32_t count, const double* const* src_d, double* const* dst_d, const int64_t* n, void* stream);
int b2_fill(int64_t n, double v, double* x_d, void* stream);

/* ------------------------------------------------------------------ IPM reductions (SURVEY 8f rows 2, 4)
 * The scalars the filter line-search reads every iteration, one single-pass kernel each; same names and argument meaning
 * as src/IPM/kernels.jl (x, xl, xu, f, zl, zu, jacl, dx: length n_tot with +-Inf for absent bounds; zl/zu FULL length,
 * the *_r views of the reference are taken through ind_lb / ind_ub of `b`; dzl/dzu, l: compressed lengths nlb/nub, m).
 * The result is ONE device double at out_d (fetch several with one D2H copy).  Deterministic (fixed reduction tree),
 * NaN-propagating min/max like Julia.  A b2_bounds object serialises its reductions: use it from one stream at a time. */
int b2_get_alpha_max(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d, double tau,
                     double* out_d, void* stream);                                   /* kernels.jl:356-371 */
int b2_get_alpha_z(b2_bounds* b, const double* zl_d, const double* zu_d, const double* dzl_d, const double* dzu_d, double tau,
                   double* out_d, void* stream);                                     /* :373-388 */
int b2_get_varphi(b2_bounds* b, double obj_val, const double* x_d, const double* xl_d, const double* xu_d, double mu, double* out_d,
                  void* stream);                                                     /* :263-283 */
int b2_get_varphi_d(b2_bounds* b, const double* f_d, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d,
                    double mu, double* out_d, void* stream);                         /* :341-354 */
int b2_get_inf_du(b2_bounds* b, const double* f_d, const double* zl_d, const double* zu_d, const double* jacl_d, double sd,
                  double* out_d, void* stream);                                      /* :285-291 */
int b2_get_inf_compl(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d, const double* zu_d,
                     double mu, double sc, double* out_d, void* stream);             /* :293-303 */
int b2_get_average_complementarity(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                                   const double* zu_d, double* out_d, void* stream); /* :305-314 */
int b2_get_min_complementarity(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                               const double* zu_d, double* out_d, void* stream);     /* :322-333 */
int b2_get_rel_search_norm(b2_bounds* b, int64_t n, const double* x_d, const double* dx_d, double* out_d, void* stream);   /* :675-681 */
int b2_get_sd(b2_bounds* b, int64_t m, const double* l_d, const double* zl_d, const double* zu_d, double s_max, double* out_d,
              void* stream);                                                         /* :684-689 */
int b2_get_sc(b2_bounds* b, const double* zl_d, const double* zu_d, double s_max, double* out_d, void* stream);            /* :690-695 */
/* set_aug_rhs! (:113-130): p = [ -f + zl - zu - jacl | -c | (xl_r - x_lr) zl_r + mu | (xu_r - x_ur) zu_r - mu ] */
int b2_set_aug_rhs(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* f_d,
                   const double* zl_d, const double* zu_d, const double* jacl_d, const double* c_d, double mu, double* p_d, void* stream);

/* ------------------------------------------------------------------ inertia-free regularisation (inertia_correction_method = InertiaFree)
 * src/IPM/solver.jl:672-737, 785-788; src/IPM/kernels.jl:233-248; src/IPM/factorization.jl:326-350.  One elementwise launch each;
 * outputs are bit-identical to the reference's broadcasts (left-to-right, no contraction; +-0, +-Inf and NaN as in IEEE). */
/* set_g_ifr!: g = f - mu ./ (x - xl) + mu ./ (xu - x) + jacl over n entries (n_tot; an infinite bound contributes mu / Inf = 0) */
int b2_set_g_ifr(int64_t n, const double* f_d, const double* x_d, const double* xl_d, const double* xu_d, const double* jacl_d, double mu,
                 double* g_d, void* stream);
/* set_aug_rhs_ifr!: p0 = [0 (n_tot) | -c (m) | 0 (nlb) | 0 (nub)] */
int b2_set_aug_rhs_ifr(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* c_d, double* p0_d, void* stream);
/* mul_hess_blk! after the Hessian product: wx[0:n_h) holds Symmetric(H, :L) t[0:n_h) (b2_spmv_symlower on hess_com, or b2d_symv_lower on
 * the dense hess); this pass sets wx[n_h:n_tot) = 0, then wx .+= t .* pr_diag and, with unreduced = 1, wx[ind_lb] .-= t[ind_lb] .*
 * (l_lower ./ l_diag) followed by the same for ub (n_tot, ind_lb, ind_ub from `b`).  With result_d = NULL that is all (n_d, g_d and tol
 * are ignored).  With result_d (B2_CURV_RESULT_LEN device doubles) the same launch also forms wx't, wx'n, g'n and t't as fixed-order
 * block partials and writes them, lhs = wx't + max(wx'n - g'n, 0) - tol t't (NaN-propagating max) and pass = (lhs >= 0) as 1.0 / 0.0.
 * Deterministic, never synchronises, graph-capturable.  The partials live in `b`: one test at a time per b2_bounds object. */
#define B2_CURV_WXT  0
#define B2_CURV_WXN  1
#define B2_CURV_GN   2
#define B2_CURV_TT   3
#define B2_CURV_LHS  4
#define B2_CURV_PASS 5
#define B2_CURV_RESULT_LEN 6
int b2_mul_hess_blk_tail(b2_bounds* b, int64_t n_h, int32_t unreduced, const double* pr_diag_d, const double* l_lower_d,
                         const double* l_diag_d, const double* u_lower_d, const double* u_diag_d, const double* t_d, double* wx_d,
                         const double* n_d, const double* g_d, double tol, double* result_d, void* stream);

/* ------------------------------------------------------------------ feasibility restoration (robust!, src/IPM/solver.jl:413-540)
 * The restorer's state (src/IPM/types.jl:1-32) and the solver vectors as device arrays: x, xl, xu, zl, zu, f, jacl, x_ref, D_R, f_R and
 * dx of length n_tot (zl / zu FULL length, +-Inf for an absent bound; the _r views go through ind_lb / ind_ub of `b`); c, y, pp, nn,
 * zp, zn and their steps of length m; dzl / dzu compressed (nlb / nub).  Elementwise kernels: one launch each, outputs bit-identical to
 * the reference's broadcasts (left-to-right, no contraction, x^2 = x*x, Julia's NaN-propagating min / max).  Reductions: as the IPM
 * reductions above (one device double at out_d, deterministic, min / max exact, sums up to association); the m-length segments
 * follow the n_tot or bound segments.  Nothing synchronises; everything can be captured in a CUDA graph.  The reference's _RR / _R
 * suffixes are spelled _rr / _r here (every exported symbol is lowercase). */
/* initialize_robust_restorer! after its two norms (src/IPM/restoration.jl:45-67; the host forms mu_R = max(mu, ||c||_inf)):
 * x_ref = x; D_R = min(1, 1 ./ |x_ref|); f_R = 0; nn by populate_RR_nn! (kernels.jl:825-829) with mu_R; pp = c + nn; zp = mu_R ./ pp;
 * zn = mu_R ./ nn; y = 0; zl_r = min(rho, zl_r); zu_r = min(rho, zu_r) */
int b2_rr_init(b2_bounds* b, int64_t m, const double* x_d, const double* c_d, double mu_R, double rho, double* x_ref_d, double* D_R_d,
               double* f_R_d, double* pp_d, double* nn_d, double* zp_d, double* zn_d, double* y_d, double* zl_d, double* zu_d, void* stream);
/* set_aug_RR! (kernels.jl:72-84) before the KKT type's own _set_aug_diagonal!: reg = del_w + zeta D_R^2 (n_tot);
 * du_diag = -del_c - pp ./ zp - nn ./ zn (m); l_lower = zl_r, l_diag = xl_r - x_lr (nlb); u_lower = zu_r, u_diag = x_ur - xu_r (nub).
 * del_w / del_c: default_primal_regularization / default_dual_regularization */
int b2_set_aug_rr(b2_bounds* b, int64_t m, double del_w, double del_c, double zeta, const double* D_R_d, const double* pp_d,
                  const double* nn_d, const double* zp_d, const double* zn_d, const double* x_d, const double* xl_d, const double* xu_d,
                  const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d, double* u_lower_d,
                  double* l_diag_d, double* u_diag_d, void* stream);
/* set_aug_RR!(::ScaledSparseKKTSystem) (:89-104): b2_set_aug_rr with l_diag = x_lr - xl_r and u_diag = xu_r - x_ur (K2.5's signs) */
int b2_set_aug_rr_scaled(b2_bounds* b, int64_t m, double del_w, double del_c, double zeta, const double* D_R_d, const double* pp_d,
                         const double* nn_d, const double* zp_d, const double* zn_d, const double* x_d, const double* xl_d, const double* xu_d,
                         const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d, double* u_lower_d,
                         double* l_diag_d, double* u_diag_d, void* stream);
/* set_aug_rhs_RR! (:133-158): p = [ -f_R + zl - zu - jacl | -c + pp - nn + (mu_R - (rho - y) pp) ./ zp - (mu_R - (rho + y) nn) ./ zn |
 *                                  (xl_r - x_lr) zl_r + mu_R | (xu_r - x_ur) zu_r - mu_R ] */
int b2_set_aug_rhs_rr(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                      const double* zu_d, const double* jacl_d, const double* f_R_d, const double* c_d, const double* y_d, const double* pp_d,
                      const double* nn_d, const double* zp_d, const double* zn_d, double mu_R, double rho, double* p_d, void* stream);
/* finish_aug_solve_RR! (:251-257) with l = y, dl = dual(d): dzp = rho - l - dl - zp; dzn = rho + l + dl - zn;
 * dpp = -pp + mu_R ./ zp - (pp ./ zp) dzp; dnn = -nn + mu_R ./ zn - (nn ./ zn) dzn */
int b2_finish_aug_solve_rr(int64_t m, const double* l_d, const double* dl_d, const double* pp_d, const double* nn_d, const double* zp_d,
                           const double* zn_d, double mu_R, double rho, double* dpp_d, double* dnn_d, double* dzp_d, double* dzn_d,
                           void* stream);
/* set_f_RR! (:106-110): f_R = zeta D_R^2 (x - x_ref) over n entries */
int b2_set_f_rr(int64_t n, double zeta, const double* D_R_d, const double* x_d, const double* x_ref_d, double* f_R_d, void* stream);
/* reset_bound_dual! (:775-800).  One-vector form (zp with pp, zn with nn): z = max(min(z, (ks mu) ./ x), (mu / ks) ./ x) over n.
 * Two-vector form on the bounded entries: zl_r with x_lr - xl_r and zu_r with xu_r - x_ur, one launch; the other entries of zl / zu
 * are left as they are (the reference maps them too: a zero multiplier against an infinite bound stays zero) */
int b2_reset_bound_dual(int64_t n, double* z_d, const double* x_d, double mu, double kappa_sigma, void* stream);
int b2_reset_bound_dual_lu(b2_bounds* b, double* zl_d, double* zu_d, const double* x_d, const double* xl_d, const double* xu_d, double mu,
                           double kappa_sigma, void* stream);
/* adjust_boundary! (:656-673): with c1 = eps mu, c2 = eps^(3/4): xl_r = x_lr - xl_r < c1 ? xl_r - c2 max(1, |x_lr|) : xl_r, and
 * xu_r = xu_r - x_ur < c1 ? xu_r + c2 max(1, |x_ur|) : xu_r */
int b2_adjust_boundary(b2_bounds* b, const double* x_d, double* xl_d, double* xu_d, double mu, void* stream);
/* the restoration line search's reductions (kernels.jl:390-636) and get_theta (:409, ||c||_1 over m; ||c||_inf is b2_norm_inf) */
int b2_get_theta(b2_bounds* b, int64_t m, const double* c_d, double* out_d, void* stream);
int b2_get_theta_r(b2_bounds* b, int64_t m, const double* c_d, const double* pp_d, const double* nn_d, double* out_d, void* stream);  /* :411-421 */
int b2_get_inf_pr_r(b2_bounds* b, int64_t m, const double* c_d, const double* pp_d, const double* nn_d, double* out_d, void* stream); /* :423-433 */
int b2_get_obj_val_r(b2_bounds* b, int64_t m, const double* pp_d, const double* nn_d, const double* D_R_d, const double* x_d,
                     const double* x_ref_d, double rho, double zeta, double* out_d, void* stream);                         /* :390-407 */
int b2_get_inf_du_r(b2_bounds* b, int64_t m, const double* f_R_d, const double* l_d, const double* zl_d, const double* zu_d,
                    const double* jacl_d, const double* zp_d, const double* zn_d, double rho, double sd, double* out_d, void* stream); /* :435-454 */
int b2_get_inf_compl_r(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                       const double* zu_d, const double* pp_d, const double* zp_d, const double* nn_d, const double* zn_d, double mu_R,
                       double sc, double* out_d, void* stream);                                                          /* :456-484 */
int b2_get_alpha_max_r(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d,
                       const double* pp_d, const double* dpp_d, const double* nn_d, const double* dnn_d, double tau_R, double* out_d,
                       void* stream);                                                                                    /* :486-515 */
int b2_get_alpha_z_r(b2_bounds* b, int64_t m, const double* zl_d, const double* zu_d, const double* dzl_d, const double* dzu_d,
                     const double* zp_d, const double* dzp_d, const double* zn_d, const double* dzn_d, double tau_R, double* out_d,
                     void* stream);                                                                                      /* :517-542 */
int b2_get_varphi_r(b2_bounds* b, int64_t m, double obj_val, const double* x_d, const double* xl_d, const double* xu_d, const double* pp_d,
                    const double* nn_d, double mu_R, double* out_d, void* stream);                                       /* :544-570 */
int b2_get_varphi_d_r(b2_bounds* b, int64_t m, const double* f_R_d, const double* x_d, const double* xl_d, const double* xu_d,
                      const double* dx_d, const double* pp_d, const double* nn_d, const double* dpp_d, const double* dnn_d, double mu_R,
                      double rho, double* out_d, void* stream);                                                          /* :612-636 */

/* ------------------------------------------------------------------ the other solve sites of the IPM (src/IPM/solver.jl)
 * The least-squares dual initialisation (initialize_dual(solver, DualInitializeLeastSquares), :86-97), robust!'s return to the regular
 * phase (:518-530), the second-order correction (second_order_correction, :547-608) and the soft restoration (restore!, :300-411).
 * Vectors as in the IPM reductions above: x, xl, xu, f, zl, zu, jacl, dx, wx, x_trial of length n_tot (zl / zu FULL length, +-Inf for
 * an absent bound; the _r views go through ind_lb / ind_ub of `b`); c, c_trial, y, dy of length m; dzl / dzu compressed (nlb / nub);
 * p: an UnreducedKKTVector buffer [x (n_tot) | y (m) | zl (nlb) | zu (nub)].  Elementwise outputs are bit-identical to the reference's
 * broadcasts (left-to-right, no contraction, unary minus a sign flip, Julia's min).  axpy! on a Julia vector goes to BLAS, which may
 * fuse the multiply and the add; these kernels form y + (a x) with two roundings and can differ from a fused BLAS by one rounding.
 * Reductions are deterministic (one device double, or the result array below).  Nothing synchronises; everything can be captured in
 * a CUDA graph; the step lengths are read from device scalars, never by the host. */
/* set_aug_diagonal!(kkt, solver) (src/IPM/kernels.jl:4-20) before the KKT type's own _set_aug_diagonal! (b2_set_aug_diagonal or
 * b2_set_aug_diagonal_unreduced): reg = del_w (n_tot); du_diag = -del_c (m); l_lower = zl_r, l_diag = xl_r - x_lr (nlb);
 * u_lower = zu_r, u_diag = x_ur - xu_r (nub).  del_w / del_c: default_primal_regularization / default_dual_regularization */
int b2_set_aug_diagonal_iterate(b2_bounds* b, int64_t m, double del_w, double del_c, const double* x_d, const double* xl_d, const double* xu_d,
                                const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d,
                                double* u_lower_d, double* l_diag_d, double* u_diag_d, void* stream);
/* set_aug_diagonal!(::ScaledSparseKKTSystem, solver) (:36-45) before b2_scaled_set_aug_diagonal: b2_set_aug_diagonal_iterate with
 * l_diag = x_lr - xl_r and u_diag = xu_r - x_ur (K2.5's signs) */
int b2_set_aug_diagonal_iterate_scaled(b2_bounds* b, int64_t m, double del_w, double del_c, const double* x_d, const double* xl_d,
                                       const double* xu_d, const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d,
                                       double* l_lower_d, double* u_lower_d, double* l_diag_d, double* u_diag_d, void* stream);
/* set_aug_rhs!(solver, kkt, w, mu) (:113-130) then dual_inf_perturbation!(px, ind_llb, ind_uub, mu, kappa_d) (:818-823) in one launch,
 * bit-identical to b2_set_aug_rhs followed by the perturbation: p = [-f + zl - zu - jacl | -w | (xl_r - x_lr) zl_r + mu | (xu_r - x_ur) zu_r
 * - mu], then px[ind_llb] -= mu kappa_d, px[ind_uub] += mu kappa_d (mu kappa_d formed once).  w = c when c_trial_d is NULL, else
 * w = c_trial + alpha c (the second-order correction's first right-hand side, copyto!(wy, c_trial); axpy!(alpha, c, wy), formed on the
 * fly).  ind_llb / ind_uub as for b2_set_centering_aug_rhs: ascending device index arrays */
int b2_set_aug_rhs_perturbed(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* f_d,
                             const double* zl_d, const double* zu_d, const double* jacl_d, const double* c_d, const double* c_trial_d,
                             double alpha, double mu, double kappa_d, int64_t nllb, const int64_t* ind_llb_d, int64_t nuub,
                             const int64_t* ind_uub_d, double* p_d, void* stream);
/* set_initial_rhs! (:220-230): p = [(-f + zl) - zu | 0 | 0 | 0] */
int b2_set_initial_rhs(b2_bounds* b, int64_t m, const double* f_d, const double* zl_d, const double* zu_d, double* p_d, void* stream);
/* The y rule of initialize_dual (solver.jl:92-96) and of robust!'s exit (:526-530), decided on the device in two launches:
 * result_d[B2_DUAL_INIT_NORM] = ||dy||_inf (NaN-propagating, as b2_norm_inf), result_d[B2_DUAL_INIT_COPY] = 1.0 when
 * solved && !(norm > constr_mult_init_max), else 0.0; then y = dy where that is 1.0, else y = +0.0.  A NaN norm compares false and
 * dy is copied, as in Julia.  robust!'s exit passes solved = 1: it does not check its solve.  Uses the reduction scratch of `b`. */
#define B2_DUAL_INIT_NORM       0
#define B2_DUAL_INIT_COPY       1
#define B2_DUAL_INIT_RESULT_LEN 2
int b2_dual_init_select(b2_bounds* b, int64_t m, const double* dy_d, int32_t solved, double constr_mult_init_max, double* y_d,
                        double* result_d, void* stream);
/* get_F (:572-610) into one device double: F1 + F2 + F3 + F4 in that order, with F1 = sum |c|, F2 = sum |f - zl + zu + jacl| (n_tot),
 * F3 = sum over ind_lb of (x_lr >= xl_r && zl_r >= 0 ? |(x_lr - xl_r) zl_r - mu| : Inf), and F4 = sum over ind_ub of
 * (xu_r >= x_ur && zu_r >= 0 ? |(xu_r - xu_r) zu_r - mu| : Inf).  F4 keeps the reference's (xu_r - xu_r) (:606) where xu_r - x_ur is
 * meant: that factor is 0 for a finite bound (NaN at an infinite one), so a feasible upper-bounded entry contributes |mu| whatever its
 * complementarity.  Each sum is deterministic and differs from the scalar loop only by association. */
int b2_get_pd_error(b2_bounds* b, int64_t m, const double* c_d, const double* f_d, const double* zl_d, const double* zu_d,
                    const double* jacl_d, const double* x_d, const double* xl_d, const double* xu_d, double mu, double* out_d, void* stream);
/* restore!'s step (solver.jl:324-339) in one launch: alpha = min(*alpha_max_d, *alpha_z_d) (Julia's min; the two scalars that
 * b2_get_alpha_max and b2_get_alpha_z wrote) is written to *alpha_d, then x += alpha dx (n_tot), y += alpha dy (m),
 * zl_r += alpha dzl (nlb), zu_r += alpha dzu (nub).  alpha_d must not alias either input scalar. */
int b2_restore_update(b2_bounds* b, int64_t m, const double* alpha_max_d, const double* alpha_z_d, double* alpha_d, const double* dx_d,
                      const double* dy_d, const double* dzl_d, const double* dzu_d, double* x_d, double* y_d, double* zl_d, double* zu_d,
                      void* stream);
/* x_trial = x + alpha wx over n entries with alpha = *alpha_d (the second-order correction's trial point after b2_get_alpha_max,
 * solver.jl:567-575; the line search's trial point, line_search.jl:39-40) */
int b2_soc_trial(int64_t n, const double* alpha_d, const double* x_d, const double* wx_d, double* x_trial_d, void* stream);

/* ------------------------------------------------------------------ adaptive barrier (barrier = QualityFunctionUpdate, src/IPM/barrier.jl:150-302)
 * The device half of get_adaptive_mu(solver, ::QualityFunctionUpdate): the new mu is computed on the device, and the free / monotone mode
 * switch and the filter stay with the caller (barrier.jl:121-148).  Vectors as in the IPM reductions above (x, xl, xu, zl, zu: n_tot, zl / zu
 * full length, +-Inf for an absent bound); aff_d, cen_d, p_d: UnreducedKKTVector buffers [x (n_tot) | y (m) | zl (nlb) | zu (nub)].
 * The per-iteration scalars live in a small device array scal_d, so that a captured graph stays valid when they change: */
#define B2_QF_TAU         0   /* tau (written by the caller) */
#define B2_QF_NRM_PRIMAL  1   /* norm(primal(p)) of the affine right-hand side (b2_primal_dual_norm2) */
#define B2_QF_NRM_DUAL    2   /* norm(dual(p)) */
#define B2_QF_MU_AVG      3   /* get_average_complementarity (b2_get_average_complementarity) */
#define B2_QF_SCAL_LEN    4
/* result_d of b2_qf_search: sigma_opt, the new mu, the number of evaluations of the quality function, the golden-section iterations run, 1.0
 * when the sigma_tol exit was taken (else 0.0), then one (sigma, phi, alpha_pr, alpha_du) row per evaluation in evaluation order */
#define B2_QF_SIGMA       0
#define B2_QF_MU          1
#define B2_QF_N_EVAL      2
#define B2_QF_N_GS_ITER   3
#define B2_QF_TOL_EXIT    4
#define B2_QF_TRACE       8
#define B2_QF_MAX_GS_ITER 64
#define B2_QF_RESULT_LEN(max_gs_iter) (B2_QF_TRACE + 4 * (6 + (max_gs_iter)))
/* out_d[0] = ||p[0:n_tot)||_2, out_d[1] = ||p[n_tot:n_tot+m)||_2 in one deterministic launch (the two norms of barrier.jl:270-271;
 * pass out_d = scal_d + B2_QF_NRM_PRIMAL) */
int b2_primal_dual_norm2(b2_bounds* b, int64_t m, const double* p_d, double* out_d, void* stream);
/* set_centering_aug_rhs! (barrier.jl:248-258) then dual_inf_perturbation! (kernels.jl:818-823) in one launch, with mu = *mu_d (device):
 * p = [0 | 0 | mu | -mu]; px[ind_llb] -= mu kappa_d; px[ind_uub] += mu kappa_d.  ind_llb / ind_uub (src/Callbacks/nlpmodels.jl:391-392):
 * device index arrays, ascending (findall order), over the model variables that have only a lower / only an upper bound */
int b2_set_centering_aug_rhs(b2_bounds* b, int64_t m, int64_t nllb, const int64_t* ind_llb_d, int64_t nuub, const int64_t* ind_uub_d,
                             const double* mu_d, double kappa_d, double* p_d, void* stream);
/* The quality-function search of get_adaptive_mu (barrier.jl:276-301, with _evaluate_quality_function :152-201 and _run_golden_search!
 * :205-246) for the affine and centering steps aff_d, cen_d: phi at sigma = 1 and 1 - 1e-4, the interval, the golden-section search,
 * clamp(sigma_opt mu, mu_min, mu_max).  A fixed sequence of 2 (2 + max_gs_iter) launches that never synchronises (graph-capturable); the
 * launches after the sigma_tol exit return at once.  Each evaluation forms aff + sigma cen on the fly: one pass for alpha_pr and alpha_du,
 * one for the complementarity sums; the last CTA of the second finishes phi and moves the search on.  Kept as the reference has them: the
 * infeasibility norms enter swapped (phi = (1 - alpha_du)^2 ||dual(p)||^2 / n_tot + (1 - alpha_pr)^2 ||primal(p)||^2 / m + compl), and the
 * else branch of the search sets phi_mid2 = phi_mid1 after phi_mid1 has been recomputed.  Requires nlb + nub > 0 (the reference returns
 * mu_min before any of this) and 0 <= max_gs_iter <= B2_QF_MAX_GS_ITER; result_d holds B2_QF_RESULT_LEN(max_gs_iter) doubles.
 * One search at a time per b2_bounds object, from the stream its other reductions use (they share one scratch). */
int b2_qf_search(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d, const double* zu_d,
                 const double* aff_d, const double* cen_d, const double* scal_d, double sigma_min, double sigma_max, double mu_min,
                 double mu_max, double sigma_tol, int32_t max_gs_iter, double* result_d, void* stream);

/* ------------------------------------------------------------------ compact L-BFGS (SparseKKTSystem, hessian_approximation = CompactLBFGS)
 * src/quasi_newton.jl:212-437 and src/IPM/factorization.jl:76-139, 253-276.  B_k = sigma I - U U' + V V' on the n model variables
 * (no slacks); S, Y are n x max_history, the memory p <= max_history.  max_history is limited to 32, so that
 * T = P + E'C^{-1}E (2 max_history square) fits in one CTA's shared memory.  Every state value (counters, sigma, pairs, small
 * matrices) is device memory: no entry point below synchronises except b2_lbfgs_state and the debug getters, and all can be
 * captured in a CUDA graph.  Reductions are deterministic (fixed order).  Use a handle from one stream at a time.
 * init_strategy: 1..4 = SCALAR1..SCALAR4 (src/enums.jl).  Bk_d is kkt.hess: the n diagonal values of B_k. */
typedef struct b2_lbfgs b2_lbfgs;
int b2_lbfgs_create(int64_t n, int32_t max_history, int32_t init_strategy, double init_value, double sigma_min, double sigma_max,
                    b2_lbfgs** out);
int b2_lbfgs_destroy(b2_lbfgs* h);
/* p = current_mem, skipped = skipped_iter, sigma; synchronises `stream` (tests and tools) */
int b2_lbfgs_state(b2_lbfgs* h, int64_t* p, int64_t* skipped, double* sigma, void* stream);
/* init!: Bk .= 2 rho0 init_value (Gilbert-Lemarechal rule with norm_g0 = g0'g0); 2 launches */
int b2_lbfgs_init(b2_lbfgs* h, double* Bk_d, const double* g0_d, double f0, void* stream);
/* update!: skip (Bk untouched) when |s| < 100 eps, |y| < 100 eps or s'y < sqrt(eps)|s||y|, reset on the second skip since the
 * last reset; otherwise store the pair (dropping the oldest when full), Bk .= sigma and recompute U, V.  2 launches */
int b2_lbfgs_update(b2_lbfgs* h, double* Bk_d, const double* sk_d, const double* yk_d, void* stream);
/* once per factorisation of C (the augmented matrix with Bk on its diagonal): H_d (N x 2 max_history, ld N = n_tot + m) = E, then
 * b2_solve(s, H_d, 2 max_history), then T = P + E'H and its Bunch-Kaufman factorisation (dsytf2 'L').  Columns of E beyond the
 * current p are zero, so their H columns are exactly zero and T carries unit pivots there. */
/* n_tot_plus_m must equal the solver's order (B2_ERR_INVALID otherwise). */
int b2_lbfgs_smw_prepare(b2_lbfgs* h, b2_solver* s, int64_t n_tot_plus_m, double* H_d, void* stream);
/* after b2_solve of w (primal_dual, N entries): w -= H T^{-1} E'w; an exact no-op when p = 0.  2 launches.
 * H and T belong to the state at the last b2_lbfgs_smw_prepare: a b2_lbfgs_update in between invalidates them until the next
 * prepare (MadNLP's order is update!, then the factorisation, then the solves, src/IPM/solver.jl). */
int b2_lbfgs_smw_apply(b2_lbfgs* h, int64_t n_tot_plus_m, const double* H_d, double* w_d, void* stream);
/* mul!: w[0:n) += alpha (-U U'x + V V'x); issued between the Jacobian products and b2_kktmul.  2 launches */
int b2_lbfgs_kkt_mul_lowrank(b2_lbfgs* h, double alpha, const double* x_d, double* w_d, void* stream);
/* Debug/test: copy one state buffer to the host and return the ring slot of the oldest pair; synchronises.  Sizes (doubles):
 * S, Y, U, V: n x max_history (S, Y in ring-slot order); SS, L, J, DL: max_history^2 (ld max_history); D: max_history;
 * T, TF: (2 max_history)^2.  b2_lbfgs_debug_ipiv copies the 2 max_history pivots of TF (LAPACK convention, 1-based). */
#define B2_LBFGS_BUF_S  0
#define B2_LBFGS_BUF_Y  1
#define B2_LBFGS_BUF_U  2
#define B2_LBFGS_BUF_V  3
#define B2_LBFGS_BUF_SS 4
#define B2_LBFGS_BUF_L  5
#define B2_LBFGS_BUF_D  6
#define B2_LBFGS_BUF_J  7
#define B2_LBFGS_BUF_DL 8
#define B2_LBFGS_BUF_T  9
#define B2_LBFGS_BUF_TF 10
int b2_lbfgs_debug_get(b2_lbfgs* h, int32_t what, double* dst_h, int64_t* first, void* stream);
int b2_lbfgs_debug_ipiv(b2_lbfgs* h, int32_t* ipiv_h, void* stream);
/* Debug/test: the same Bunch-Kaufman kernels on a caller's N x N matrix (N <= 64, column-major, lower triangle; factor in place)
 * and the dsytrs 'L' solve of one right-hand side. */
int b2_debug_bk_factor(int32_t N, double* A_d, int32_t* ipiv_d, void* stream);
int b2_debug_bk_solve(int32_t N, const double* F_d, const int32_t* ipiv_d, double* b_d, void* stream);

/* ------------------------------------------------------------------ dense quasi-Newton (DenseKKTSystem / DenseCondensedKKTSystem,
 * hessian_approximation = BFGS or DampedBFGS; src/quasi_newton.jl:71-201, 425-437).  Bk_d is the KKT system's `hess`: n x n,
 * column-major, leading dimension n; only its lower triangle is read or written.  Every state value (is_instantiated, the last
 * decision, the scalars, bsk = B s and r) is device memory: no entry point below synchronises except b2d_qn_state and the debug
 * getter, each issues a fixed launch sequence, and all can be captured in a CUDA graph.  Reductions are deterministic (fixed
 * order).  Use a handle from one stream at a time.  n <= 2^31 - 1; element offsets are 64-bit. */
#define B2_QN_BFGS        1
#define B2_QN_DAMPED_BFGS 2
typedef struct b2d_qn b2d_qn;
int b2d_qn_create(int64_t n, int32_t kind, b2d_qn** out);
int b2d_qn_destroy(b2d_qn* h);
/* init!: Bk[i, i] = 2 rho0 (Gilbert-Lemarechal rule with norm_g0 = g0'g0; f0 = +-0 takes the 1 / norm_g0 branch); the rest of Bk
 * and is_instantiated are left alone.  2 launches */
int b2d_qn_init(b2d_qn* h, double* Bk_d, const double* g0_d, double f0, void* stream);
/* update!: BFGS skips (Bk bit-unchanged) when y's < 1e-8; DampedBFGS never skips.  The first accepted call sets the diagonal to
 * y's / s's.  Then bsk = B s (b2d_symv_lower), alpha1 = 1 / s'bsk and, in one pass over the lower triangle, per element
 * a = a + b_i ((-alpha1) b_j); a = a + v_i (alpha2 v_j) (no contraction), with v = y, alpha2 = 1 / y's (BFGS) or
 * v = r = (0 + theta y) + (1 - theta) bsk, alpha2 = 1 / r's (DampedBFGS).  6 launches */
int b2d_qn_update(b2d_qn* h, double* Bk_d, const double* sk_d, const double* yk_d, void* stream);
/* the fused rank-2 pass of b2d_qn_update alone, with the decision, scalars and vectors of the last update (benchmarks); yk_d is
 * read by BFGS only */
int b2d_qn_rank2(b2d_qn* h, double* Bk_d, const double* yk_d, void* stream);
/* is_instantiated, the last decision, and scalars[6] = {y's, s's, s'Bs, theta, alpha1, alpha2} of the last update (on a skipped
 * BFGS call, the values the update would have used); synchronises `stream` */
int b2d_qn_state(b2d_qn* h, int32_t* instantiated, int32_t* accepted, double* scalars, void* stream);
/* Debug/test: host copies of bsk and r (n doubles each; r is written by DampedBFGS only); synchronises */
int b2d_qn_debug_vectors(b2d_qn* h, double* bsk_h, double* rk_h, void* stream);

/* ---- KrylovIterator: restarted GMRES preconditioned on the RIGHT by the KKT solve (x = M^-1 u, the preconditioned vectors kept).
 * The caller runs solve_kkt! and mul! of its KKT type between these entries; one Arnoldi step k is
 *     b2_krylov_scale(k, w)           v_k = w / s, z_k = v_k       (s = beta at k = 0, h_{k,k-1} after)
 *     solve_kkt!(z_k) ; mul!(w, K, z_k, 1, 0)
 *     b2_krylov_orthogonalize(k, w)   k + 2 modified Gram-Schmidt passes: h_{0..k,k}, h_{k+1,k}, the Givens update of g, the record
 * and a cycle is b2_krylov_begin, steps k = 0, 1, ..., then b2_krylov_close followed by w -= K x and ||w||_inf into
 * state[B2_KRYLOV_REC + B2_KRYLOV_REC_NORM_W] (b2_norm_inf, or a fused mul-norm).  The handle owns V ((restart + 1) x n) and Z
 * (restart x n), contiguous with stride n, and the state below (device memory; doubles at these offsets).  No entry allocates or
 * synchronises; reductions have a fixed order, so a captured sequence replays bit-identically.  One handle serves one stream at a
 * time.  n >= 1, 1 <= restart <= 16. */
#define B2_KRYLOV_MAX_RESTART 16
#define B2_KRYLOV_H           0       /* 17 x 16 column-major: H, rotated into R in place */
#define B2_KRYLOV_CS          272     /* 16: cosines of the rotations */
#define B2_KRYLOV_SN          288     /* 16: sines */
#define B2_KRYLOV_G           304     /* 17: the rotated beta e_1 */
#define B2_KRYLOV_Y           321     /* 16: y of the last close */
#define B2_KRYLOV_SCALE       337     /* the divisor of the next scale pass */
#define B2_KRYLOV_REC         344     /* the record the host reads: */
#define B2_KRYLOV_REC_EST     0       /*   |g_{k+1}| of the last step */
#define B2_KRYLOV_REC_H       1       /*   h_{k+1,k} of the last step */
#define B2_KRYLOV_REC_NORM_W  2       /*   ||b - K x||_inf after a close (accumulated by the caller's norm) */
#define B2_KRYLOV_REC_NORM_X  3       /*   ||x||_inf after a close */
#define B2_KRYLOV_REC_NORM_B  4       /*   ||b||_inf (first begin) */
#define B2_KRYLOV_REC_NORM_B2 5       /*   ||b||_2 (first begin) */
#define B2_KRYLOV_REC_LEN     8
#define B2_KRYLOV_STATE_LEN   352
typedef struct b2_krylov b2_krylov;
int b2_krylov_create(int64_t n, int32_t restart, b2_krylov** out);
int b2_krylov_destroy(b2_krylov* h);
/* device pointers of V, Z and the state */
int b2_krylov_buffers(b2_krylov* h, double** V_d, double** Z_d, double** state_d);
/* start of a cycle.  first != 0: x = 0, w = b, the record zeroed, ||b||_inf and ||b||_2 into it.  Then beta = ||w||_2 and g = beta e_1
 * (w holds r = b - K x; b and x are not read when first = 0).  2 launches (first) or 1 */
int b2_krylov_begin(b2_krylov* h, int32_t first, const double* b_d, double* x_d, double* w_d, void* stream);
/* v_k = z_k = w / s, 0 <= k < restart.  1 launch */
int b2_krylov_scale(b2_krylov* h, int32_t k, const double* w_d, void* stream);
/* w = K z_k on entry; MGS of w against v_0..v_k, h_{k+1,k} = ||w||_2, the Givens update and the record; w leaves as the unscaled
 * v_{k+1}.  k + 2 launches */
int b2_krylov_orthogonalize(b2_krylov* h, int32_t k, double* w_d, void* stream);
/* close over m = k + 1 columns (1 <= m <= restart): y = R^-1 g (one warp), x += Z y, w = b, record NORM_W = 0 and
 * NORM_X = ||x||_inf.  3 launches (a memset, the y solve and the pass) */
int b2_krylov_close(b2_krylov* h, int32_t m, const double* b_d, double* x_d, double* w_d, void* stream);

/* ---- Richardson refinement as ONE CUDA graph (solve_refine!, src/LinearSolvers/backsolve.jl:27-76, for the first trial of
 * inertia_correction!): the loop body runs under a conditional WHILE node and a one-thread test kernel decides on the device
 * whether it runs again, so the host waits once per solve instead of once per refinement step.  The graph is
 *     b2_richardson_begin (||b||, x = 0, w = b) ; WHILE { caller's step ; test }
 * Building it:  b2_refine_loop_begin(h, ...)  -- captures the part before the WHILE node and starts capturing its body on `stream`
 *               the caller issues one refinement step on `stream` (x += M^-1 w ; w = b - K x ; norms_d[0] = ||w||, norms_d[1] = ||x||)
 *               b2_refine_loop_end(h, ...)    -- issues the test, ends the capture, instantiates
 * then b2_refine_loop_launch(h, stream) replays it.  The last test writes the solve's record to pinned host memory, its sequence
 * number last; b2_refine_loop_wait returns as soon as that record is there (before the graph's completion reaches the host, and
 * also after any D2H copy queued on the stream before the launch), and b2_refine_loop_record reads it.  The test applies solve_refine!'s stopping rule in the same IEEE operations,
 *     ratio = ||w|| / (min(||x||, 1e6 ||b||) + ||b||) ; ir += 1 ; stop when ir >= max_iter or ratio < tol
 * (||b|| == 0: one step, ir = 0, ratio = 0), and also stops after the first step when the factorisation's inertia, read from the
 * solver's device counters (b2_inertia_source), fails the KKT type's is_inertia_correct: num_zero == 0 and, where given (>= 0),
 * num_pos == expect_pos and num_neg == expect_neg.  B2_ERR_UNSUPPORTED from begin / end: the driver refuses conditional graph
 * nodes (the caller refines on the host); the stream is left out of capture. */
typedef struct b2_inertia_source {
    const int32_t* counters_d;    /* the solver's device pivot counters, written by its factorisation */
    int64_t n;                    /* order of the factored matrix: num_pos = n - num_neg - num_zero */
    int32_t neg[2], zero[2];      /* num_neg = the sum of counters_d[neg[k]] over the k with neg[k] >= 0; num_zero likewise */
    int32_t fail;                 /* counters_d[fail] != 0: a device-wide wait timed out, the factorisation is not valid */
    int32_t reserved;
} b2_inertia_source;
int b2_inertia_source_get(b2_solver* s, b2_inertia_source* out);       /* single-part solvers only */
typedef struct b2_refine_record {
    double ratio;                 /* residual ratio of the last step (0 when ||b|| == 0) */
    double norm_w, norm_x, norm_b;
    int64_t ir;                   /* steps counted by the stopping rule (solve_refine!'s cnt.ir) */
    int64_t steps;                /* steps run */
    int64_t num_pos, num_zero, num_neg;
    int32_t inertia_ok;           /* the inertia test of the first step */
    int32_t fail;                 /* counters_d[fail] of the first step */
    int64_t seq;                  /* solves this handle has finished, written last */
} b2_refine_record;
typedef struct b2_refine_loop b2_refine_loop;
int b2_refine_loop_create(b2_refine_loop** out);
int b2_refine_loop_destroy(b2_refine_loop* h);
/* any graph the handle held is dropped; b, w, x, norms_d (3 doubles: ||w||, ||x||, ||b||) are baked into the graph */
int b2_refine_loop_begin(b2_refine_loop* h, int64_t n, const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream);
int b2_refine_loop_end(b2_refine_loop* h, const b2_inertia_source* src, int64_t expect_pos, int64_t expect_neg, int32_t max_iter,
                       double tol, void* stream);
int b2_refine_loop_launch(b2_refine_loop* h, void* stream);
/* wait for the record of the last launch: polls it and the stream; an error of the stream is returned, not waited for */
int b2_refine_loop_wait(b2_refine_loop* h);
int b2_refine_loop_record(b2_refine_loop* h, b2_refine_record* out);

/* ---- The trials of inertia_correction! after a wrong first inertia (src/IPM/solver.jl:611-670) as ONE CUDA graph:
 *     WHILE { schedule ; regularise ; caller's build_kkt + factorize ; trial test ;
 *             IF { b2_richardson_begin ; WHILE { caller's refinement step ; the test of b2_refine_loop } } ; close }
 * so the host waits once for all the regularised trials of a step instead of once per trial and per refinement step.  The
 * schedule kernel reproduces the host's del_w sequence operation for operation:
 *     first trial:  del_w = first_hessian_perturbation if del_w_last == 0, else max(min_hessian_perturbation, perturb_dec_fact * del_w_last)
 *     later trials: del_w *= (del_w_last == 0 ? perturb_inc_fact_first : perturb_inc_fact); stop as failed when del_w > max_hessian_perturbation
 *     del_c = the launch's del_c when dual_always or the previous inertia has num_zero != 0, else 0
 * (max is Python's: the first argument unless the second is greater) and regularises by (del_w - del_w_prev, del_c - del_c_prev)
 * with the arithmetic of b2_regularize_diagonal.  The trial test applies the KKT type's inertia rule (as b2_refine_loop_end) to the
 * solver's device counters; only a right inertia runs the refinement.  The close accepts when ratio < acceptable_tol (0 when
 * ||b|| == 0), goes round again after a wrong inertia, and hands over to the host when the inertia is right but the refinement is
 * not acceptable (the improve! retry changes the factorisation's pivot threshold, which this graph bakes in) or when the
 * factorisation reports a timed-out wait (the host's inertia read reports it).
 * Building it:  b2_inertia_loop_begin   -- starts capturing the WHILE body on `stream` (schedule and regularise are issued)
 *               the caller issues its build_kkt and factorisation on `stream`
 *               b2_inertia_loop_refine  -- the trial test, the IF node, b2_richardson_begin; starts capturing the refinement body
 *               the caller issues one refinement step (as for b2_refine_loop_begin)
 *               b2_inertia_loop_end     -- the refinement test, the close; instantiates (and ends any capture left open)
 * B2_ERR_UNSUPPORTED from these: the driver refuses (nested) conditional graph nodes, and the caller keeps the host loop.  The
 * record is written to pinned host memory by the close, its sequence number last, as b2_refine_loop's. */
typedef struct b2_inertia_options {
    double first_hessian_perturbation, min_hessian_perturbation, max_hessian_perturbation;
    double perturb_inc_fact_first, perturb_inc_fact, perturb_dec_fact;
} b2_inertia_options;
#define B2_TRIALS_ACCEPTED 1      /* a trial with the right inertia whose refinement is acceptable */
#define B2_TRIALS_FAILED   2      /* del_w went past max_hessian_perturbation */
#define B2_TRIALS_HANDOVER 3      /* the last trial's inertia is right and its refinement not acceptable: improve! is the host's */
#define B2_TRIALS_FAULT    4      /* the last factorisation's counters report a timed-out wait (not a valid inertia) */
typedef struct b2_inertia_record {
    int32_t status;               /* B2_TRIALS_* */
    int32_t inertia_ok;           /* the inertia test of the last trial */
    int64_t trials;               /* regularised trials run (factorisations); the del_w of each: b2_inertia_loop_record */
    double del_w, del_w_prev, del_c_prev;   /* the schedule's state after the last trial */
    int64_t num_pos, num_zero, num_neg;     /* inertia of the last factorisation */
    int64_t ir;                   /* of the last solve (status ACCEPTED or HANDOVER) */
    double ratio;
    int64_t ir_total;             /* ir summed over the solves that ended a trial: the host's cnt.backsolves adds it */
    int64_t seq;                  /* launches this handle has finished, written last */
} b2_inertia_record;
/* trials a step can take before del_w > max_hessian_perturbation: from min(min_, first_hessian_perturbation), by the smaller of
 * the two increase factors.  B2_ERR_UNSUPPORTED when the schedule is unbounded (a factor <= 1, a start <= 0, an infinite or NaN
 * bound) or bounded above 2^20 trials.  Host only. */
int b2_inertia_trial_bound(const b2_inertia_options* opt, int64_t* out);
typedef struct b2_inertia_loop b2_inertia_loop;
/* the del_w list is sized by b2_inertia_trial_bound (its errors are returned) */
int b2_inertia_loop_create(const b2_inertia_options* opt, b2_inertia_loop** out);
int b2_inertia_loop_destroy(b2_inertia_loop* h);
/* any graph the handle held is dropped; reg, pr_diag (n_tot), du_diag (m) are baked in */
int b2_inertia_loop_begin(b2_inertia_loop* h, int64_t n_tot, int64_t m, double* reg_d, double* pr_diag_d, double* du_diag_d,
                          int32_t dual_always, void* stream);
/* b2_inertia_loop_begin for ScaledSparseKKTSystem: the regularisation is b2_scaled_regularize_diagonal's, pr_diag += dw (s s) with
 * scaling_d the system's scaling factor (n_tot) */
int b2_inertia_loop_begin_scaled(b2_inertia_loop* h, int64_t n_tot, int64_t m, double* reg_d, double* pr_diag_d, double* du_diag_d,
                                 const double* scaling_d, int32_t dual_always, void* stream);
/* expect_pos / expect_neg as for b2_refine_loop_end; b, w, x (n) and norms_d (3 doubles) as for b2_refine_loop_begin */
int b2_inertia_loop_refine(b2_inertia_loop* h, const b2_inertia_source* src, int64_t expect_pos, int64_t expect_neg, int64_t n,
                           const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream);
int b2_inertia_loop_end(b2_inertia_loop* h, int32_t max_iter, double tol, double acceptable_tol, void* stream);
/* one step's trials: del_w_last as the host holds it, del_c = jacobian_regularization_value * mu^jacobian_regularization_exponent,
 * num_zero of the first trial's inertia (the dual rule of the first regularised trial).  The previous launch must have been waited for */
int b2_inertia_loop_launch(b2_inertia_loop* h, double del_w_last, double del_c, int64_t num_zero, void* stream);
/* wait for the record of the last launch: polls it and the stream; an error of the stream is returned, not waited for */
int b2_inertia_loop_wait(b2_inertia_loop* h);
/* the record and the first min(trials, cap) entries of the del_w list */
int b2_inertia_loop_record(b2_inertia_loop* h, b2_inertia_record* out, double* del_w_out, int64_t cap);


#ifdef __cplusplus
}
#endif
#endif /* B200KKT_H */
