// Symbolic analysis for the supernodal multifrontal LDL^T (host side, one-time per pattern).
// Replaces what the reference delegates to cuDSS "analysis" (lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cudss.jl:148)
// or ma97_analyse (lib/MadNLPHSL/src/ma97.jl:45-46): fill-reducing ordering, elimination tree,
// supernode amalgamation, front row structures, assembly maps and the level schedule.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace b2 {

struct AnalysisOptions {
    int ordering = 0;          // B2_ORDER_*
    int nemin = 16;
    double relax_zeros = 0.25;
    int n_parts = 1;           // multi-GPU partition count
    int kkt_n_primal = 0;      // augmented-KKT hint: dual rows are ordered after one primal neighbour
    int kkt_n_dual = 0;        // > 0: rows from kkt_n_primal + kkt_n_dual on are bound duals, ordered just before their neighbour
    int chain_merge_f = 0;     // > 0: single-child chains are merged while the front order stays <= this (latency, not flops)
    bool pairs = false;        // B2_SPARSE_PIVOT_PAIRS: every matchable constraint dual right after a distinct primal neighbour, in one supernode
};

// One front per supernode.  Pivot columns [first, first+w) in the PERMUTED numbering; the front has
// order f = w + r with row list rows[rows_ptr .. rows_ptr+f) (first w entries = the pivot columns).
struct Symbolic {
    int32_t n = 0;
    int64_t nnz_a = 0;
    std::vector<int32_t> perm;        // perm[new] = old
    std::vector<int32_t> iperm;       // iperm[old] = new
    int32_t nsuper = 0;
    std::vector<int32_t> sn_first;    // [nsuper+1]
    std::vector<int32_t> sn_parent;   // [nsuper], -1 for roots
    std::vector<int32_t> sn_level;    // [nsuper], leaves = 0
    std::vector<int64_t> rows_ptr;    // [nsuper+1]
    std::vector<int32_t> rows;
    std::vector<int64_t> lp_off;      // [nsuper+1] panel offsets in the factor array (f*w doubles each, ld=f)
    std::vector<int64_t> cb_off;      // [nsuper+1] update-block offsets in the workspace (r*r doubles, ld=r)
    std::vector<int32_t> child_ptr;   // [nsuper+1]
    std::vector<int32_t> child_idx;   // children, ascending supernode id (fixes the extend-add order)
    std::vector<int64_t> rel_ptr;     // [nsuper+1]  (r entries per supernode)
    std::vector<int32_t> rel;         // position of each below-row inside the PARENT's front row list
    std::vector<int64_t> amap_ptr;    // [nsuper+1]
    std::vector<int64_t> amap_src;    // index into the caller's CSC value array
    std::vector<int64_t> amap_dst;    // absolute offset into the factor array (panel entry)
    int32_t nlevels = 0;
    std::vector<int32_t> level_ptr;   // [nlevels+1]
    std::vector<int32_t> level_sn;    // supernodes grouped by level
    // multi-GPU partition: owner[s] in [0,n_parts) for subtree supernodes, -1 for the shared top tree
    std::vector<int32_t> owner;
    int64_t nnz_l = 0;
    int64_t flops = 0;
    int32_t max_front = 0;
    int64_t top_rows = 0;             // sum of w over the shared top tree
    int64_t exch_cb = 0;              // doubles at the start of the update-block workspace that cross rank->top
    std::vector<uint8_t> pair_start;  // [n] (AnalysisOptions::pairs) 1 where permuted column j starts a candidate 2x2 pivot (j, j+1)
};

// Checks the row classes of an unreduced KKT pattern: kkt_n_dual >= 0, kkt_n_primal + kkt_n_dual <= n, kkt_n_primal > 0 when
// kkt_n_dual > 0, and every bound row (index >= kkt_n_primal + kkt_n_dual) has exactly one off-diagonal entry, in a primal column.
// Returns "" when the options are valid, else what is wrong.
std::string check_kkt_rows(int32_t n, const int32_t* colptr, const int32_t* rowval, int kkt_n_primal, int kkt_n_dual);

// colptr/rowval: lower-triangular CSC (0-based).  Throws std::runtime_error on failure.
void analyse(int32_t n, const int32_t* colptr, const int32_t* rowval, const AnalysisOptions& opt,
             const int32_t* user_perm, Symbolic& S);

}  // namespace b2
