// b2_bounds: the index sets of the bounded primal variables (ind_lb / ind_ub of MadNLP, src/nlpmodels.jl:369-406) on the
// device, their inverse maps, and the scratch of the deterministic reductions (grid_reduce.cuh) of ipm_reductions.cu, barrier.cu
// and inertia_free.cu.  Those kernels share the one scratch pair: an object is used from one stream at a time.
#pragma once
#include "common.cuh"
#include "grid_reduce.cuh"

struct b2_bounds {
    int64_t n_tot = 0, nlb = 0, nub = 0;
    b2::DevBuf<int64_t> ind_lb, ind_ub;
    b2::DevBuf<int32_t> lbpos, ubpos;      // [n_tot] position in ind_lb / ind_ub or -1
    b2::DevBuf<double> red_part;           // [8 * B2_RED_BLOCKS] per-CTA partial results, up to 8 values per reduction
    b2::DevBuf<unsigned> red_ticket;       // [1] arrival counter (reset by the last CTA)
    b2::DevBuf<double> qf_state;           // [B2_QF_STATE_DOUBLES] the quality-function search between its launches
};

constexpr int B2_QF_STATE_DOUBLES = 64;
