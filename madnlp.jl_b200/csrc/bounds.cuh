// b2_bounds: the index sets of the bounded primal variables (ind_lb / ind_ub of MadNLP, src/nlpmodels.jl:369-406) on the
// device, their inverse maps, and the scratch of the deterministic reductions (ipm_reductions.cu).
#pragma once
#include "common.cuh"

constexpr int B2_RED_BLOCKS = 512;         // fixed grid of the reductions: partial results are combined in index order

struct b2_bounds {
    int64_t n_tot = 0, nlb = 0, nub = 0;
    b2::DevBuf<int64_t> ind_lb, ind_ub;
    b2::DevBuf<int32_t> lbpos, ubpos;      // [n_tot] position in ind_lb / ind_ub or -1
    b2::DevBuf<double> red_part;           // [B2_RED_BLOCKS] per-CTA partial results
    b2::DevBuf<unsigned> red_ticket;       // [1] arrival counter (reset by the last CTA)
    b2::DevBuf<double> curv_part;          // [4 * B2_RED_BLOCKS] partials of the curvature test (inertia_free.cu)
    b2::DevBuf<unsigned> curv_ticket;      // [1] its arrival counter
    b2::DevBuf<double> qf_part;            // [8 * B2_RED_BLOCKS] partials of the adaptive-barrier passes (barrier.cu)
    b2::DevBuf<unsigned> qf_ticket;        // [1] their arrival counter
    b2::DevBuf<double> qf_state;           // [B2_QF_STATE_DOUBLES] the quality-function search between its launches
};

constexpr int B2_QF_STATE_DOUBLES = 64;
