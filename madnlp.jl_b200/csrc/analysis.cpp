// Symbolic analysis for the supernodal multifrontal LDL^T (host, one-time per sparsity pattern).
// See analysis.hpp.  Pipeline:
//   ordering (METIS nested dissection | built-in minimum degree | natural | user)
//   -> elimination tree + postorder -> column counts -> maximal supernodes
//   -> relaxed amalgamation on the supernode tree (any child may merge into its parent; the final
//      permutation is re-derived so that merged groups are contiguous)
//   -> front row structures, child->parent relative indices, A->front scatter map, level schedule,
//      subtree-to-rank partition for multi-GPU.
#include "analysis.hpp"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <climits>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <queue>
#include <set>
#include <stdexcept>

extern "C" {
// METIS 5 (libmetis_static.a shipped with the CUDA toolkit is built with 64-bit idx_t).
int METIS_NodeND(int64_t* nvtxs, int64_t* xadj, int64_t* adjncy, int64_t* vwgt, int64_t* options,
                 int64_t* perm, int64_t* iperm);
int METIS_SetDefaultOptions(int64_t* options);
}

namespace b2 {

namespace {

void build_adjacency(int32_t n, const int32_t* colptr, const int32_t* rowval,
                     std::vector<int64_t>& xadj, std::vector<int64_t>& adj) {
    std::vector<int64_t> deg(n, 0);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t i = rowval[p];
            if (i == j) continue;
            if (i < 0 || i >= n) throw std::runtime_error("row index out of range");
            deg[i]++; deg[j]++;
        }
    xadj.assign(n + 1, 0);
    for (int32_t i = 0; i < n; ++i) xadj[i + 1] = xadj[i] + deg[i];
    adj.assign(xadj[n], 0);
    std::vector<int64_t> pos(xadj.begin(), xadj.end() - 1);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t i = rowval[p];
            if (i == j) continue;
            adj[pos[i]++] = j;
            adj[pos[j]++] = i;
        }
    // remove duplicate edges (the reference's CSC has none, but be safe)
    std::vector<int64_t> nx(n + 1, 0), na;
    na.reserve(adj.size());
    for (int32_t i = 0; i < n; ++i) {
        std::sort(adj.begin() + xadj[i], adj.begin() + xadj[i + 1]);
        int64_t last = -1;
        for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p)
            if (adj[p] != last) { na.push_back(adj[p]); last = adj[p]; }
        nx[i + 1] = (int64_t)na.size();
    }
    xadj.swap(nx);
    adj.swap(na);
}

void order_metis(int32_t n, std::vector<int64_t>& xadj, std::vector<int64_t>& adj, std::vector<int32_t>& perm) {
    std::vector<int64_t> p(n), ip(n);
    int64_t nn = n;
    int64_t options[40];
    METIS_SetDefaultOptions(options);
    int rc = METIS_NodeND(&nn, xadj.data(), adj.data(), nullptr, options, p.data(), ip.data());
    if (rc != 1) throw std::runtime_error("METIS_NodeND failed");
    perm.resize(n);
    for (int32_t i = 0; i < n; ++i) perm[i] = (int32_t)p[i];
}

// Built-in minimum-degree ordering on the quotient graph (element absorption, approximate external
// degree as in AMD; no supervariables).  Fallback when METIS is not wanted.
void order_mindeg(int32_t n, const std::vector<int64_t>& xadj, const std::vector<int64_t>& adj,
                  std::vector<int32_t>& perm) {
    std::vector<std::vector<int32_t>> vadj(n), velem(n), evars;
    for (int32_t i = 0; i < n; ++i) vadj[i].assign(adj.begin() + xadj[i], adj.begin() + xadj[i + 1]);
    std::vector<int64_t> deg(n);
    std::vector<char> dead_e;
    std::vector<char> elim(n, 0);
    std::set<std::pair<int64_t, int32_t>> pq;
    for (int32_t i = 0; i < n; ++i) { deg[i] = (int64_t)vadj[i].size(); pq.insert({deg[i], i}); }
    std::vector<int32_t> mark(n, -1);
    perm.clear(); perm.reserve(n);
    std::vector<int32_t> Lp;
    for (int32_t step = 0; step < n; ++step) {
        auto it = pq.begin();
        int32_t v = it->second;
        pq.erase(it);
        elim[v] = 1;
        perm.push_back(v);
        Lp.clear();
        mark[v] = step;
        for (int32_t u : vadj[v]) if (!elim[u] && mark[u] != step) { mark[u] = step; Lp.push_back(u); }
        for (int32_t e : velem[v]) {
            if (dead_e[e]) continue;
            for (int32_t u : evars[e]) if (!elim[u] && mark[u] != step) { mark[u] = step; Lp.push_back(u); }
            dead_e[e] = 1;
            std::vector<int32_t>().swap(evars[e]);
        }
        int32_t enew = (int32_t)evars.size();
        evars.push_back(Lp);
        dead_e.push_back(0);
        std::vector<int32_t>().swap(vadj[v]);
        std::vector<int32_t>().swap(velem[v]);
        for (int32_t u : Lp) {
            // variable neighbours now covered by the new element are dropped
            auto& a = vadj[u];
            size_t k = 0;
            for (size_t q = 0; q < a.size(); ++q) if (mark[a[q]] != step) a[k++] = a[q];
            a.resize(k);
            auto& el = velem[u];
            k = 0;
            for (size_t q = 0; q < el.size(); ++q) if (!dead_e[el[q]]) el[k++] = el[q];
            el.resize(k);
            el.push_back(enew);
            int64_t d = (int64_t)a.size();
            for (int32_t e : el) d += (int64_t)evars[e].size() - 1;
            if (d > n - step - 1) d = n - step - 1;
            pq.erase({deg[u], u});
            deg[u] = d;
            pq.insert({d, u});
        }
    }
}

// strict-lower pattern of the permuted matrix, stored by row (CSR): for row i, the columns k < i.
void permuted_lower_rows(int32_t n, const int32_t* colptr, const int32_t* rowval, const std::vector<int32_t>& iperm,
                         std::vector<int64_t>& rptr, std::vector<int32_t>& rcol) {
    rptr.assign(n + 1, 0);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t a = iperm[rowval[p]], b = iperm[j];
            if (a == b) continue;
            rptr[std::max(a, b) + 1]++;
        }
    for (int32_t i = 0; i < n; ++i) rptr[i + 1] += rptr[i];
    rcol.assign(rptr[n], 0);
    std::vector<int64_t> pos(rptr.begin(), rptr.end() - 1);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            int32_t a = iperm[rowval[p]], b = iperm[j];
            if (a == b) continue;
            rcol[pos[std::max(a, b)]++] = std::min(a, b);
        }
}

void etree(int32_t n, const std::vector<int64_t>& rptr, const std::vector<int32_t>& rcol, std::vector<int32_t>& parent) {
    parent.assign(n, -1);
    std::vector<int32_t> anc(n, -1);
    for (int32_t i = 0; i < n; ++i)
        for (int64_t p = rptr[i]; p < rptr[i + 1]; ++p) {
            int32_t j = rcol[p];
            while (j != -1 && j < i) {
                int32_t nx = anc[j];
                anc[j] = i;
                if (nx == -1) parent[j] = i;
                j = nx;
            }
        }
}

// postorder of a forest; children visited in ascending order.  post[k] = node visited k-th.
void postorder(int32_t n, const std::vector<int32_t>& parent, std::vector<int32_t>& post) {
    std::vector<int32_t> head(n, -1), next(n, -1);
    for (int32_t j = n - 1; j >= 0; --j)
        if (parent[j] != -1) { next[j] = head[parent[j]]; head[parent[j]] = j; }
    post.clear(); post.reserve(n);
    std::vector<int32_t> stack;
    for (int32_t r = 0; r < n; ++r) {
        if (parent[r] != -1) continue;
        stack.push_back(r);
        while (!stack.empty()) {
            int32_t v = stack.back();
            int32_t c = head[v];
            if (c != -1) { head[v] = next[c]; stack.push_back(c); }
            else { post.push_back(v); stack.pop_back(); }
        }
    }
}

void colcounts(int32_t n, const std::vector<int64_t>& rptr, const std::vector<int32_t>& rcol,
               const std::vector<int32_t>& parent, std::vector<int64_t>& cc) {
    cc.assign(n, 1);
    std::vector<int32_t> mark(n, -1);
    for (int32_t i = 0; i < n; ++i) {
        mark[i] = i;
        for (int64_t p = rptr[i]; p < rptr[i + 1]; ++p)
            for (int32_t j = rcol[p]; mark[j] != i; j = parent[j]) { cc[j]++; mark[j] = i; }
    }
}

inline int64_t trap_nnz(int64_t w, int64_t f) { return w * f - w * (w - 1) / 2; }

// off-diagonal neighbours of the rows [nc, n): cnt[b - nc] = how many (each stored entry counted once, upper or lower),
// nb[b - nc] = the last one seen
void bound_neighbours(int32_t n, const int32_t* colptr, const int32_t* rowval, int32_t nc, std::vector<int32_t>& nb,
                      std::vector<int32_t>& cnt) {
    nb.assign(n - nc, -1);
    cnt.assign(n - nc, 0);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
            const int32_t i = rowval[p];
            if (i == j) continue;
            if (i >= nc) { nb[i - nc] = j; cnt[i - nc]++; }
            if (j >= nc) { nb[j - nc] = i; cnt[j - nc]++; }
        }
}

// B2_ANALYSIS_TIMING=1: print the wall time of each phase of analyse() to stderr
struct PhaseTimer {
    bool on;
    std::chrono::steady_clock::time_point t0;
    PhaseTimer() : on(getenv("B2_ANALYSIS_TIMING") != nullptr), t0(std::chrono::steady_clock::now()) {}
    void lap(const char* what) {
        if (!on) return;
        const auto t1 = std::chrono::steady_clock::now();
        fprintf(stderr, "[b2 analyse] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
        t0 = t1;
    }
};
}  // namespace

std::string check_kkt_rows(int32_t n, const int32_t* colptr, const int32_t* rowval, int kkt_n_primal, int kkt_n_dual) {
    if (kkt_n_dual == 0) return "";
    if (kkt_n_dual < 0) return "kkt_n_dual < 0";
    if ((int64_t)kkt_n_primal + kkt_n_dual > n) return "kkt_n_primal + kkt_n_dual > n";
    if (kkt_n_primal <= 0) return "kkt_n_dual > 0 needs kkt_n_primal > 0";
    const int32_t nc = kkt_n_primal + kkt_n_dual;
    for (int32_t j = 0; j < n; ++j)
        for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p)
            if (rowval[p] < 0 || rowval[p] >= n) return "row index out of range";
    std::vector<int32_t> nb, cnt;
    bound_neighbours(n, colptr, rowval, nc, nb, cnt);
    for (int32_t b = nc; b < n; ++b) {
        if (cnt[b - nc] != 1)
            return "bound row " + std::to_string(b) + " has " + std::to_string(cnt[b - nc]) + " off-diagonal entries (needs exactly 1)";
        if (nb[b - nc] >= kkt_n_primal)
            return "bound row " + std::to_string(b) + " is coupled to row " + std::to_string(nb[b - nc]) + ", which is not primal";
    }
    return "";
}

void analyse(int32_t n, const int32_t* colptr, const int32_t* rowval, const AnalysisOptions& opt,
             const int32_t* user_perm, Symbolic& S) {
    if (n <= 0) throw std::runtime_error("n must be positive");
    S = Symbolic();
    S.n = n;
    S.nnz_a = colptr[n];
    const int64_t nnz = colptr[n];
    PhaseTimer timer;

    // ---- 1. ordering.  With bound-dual rows (kkt_n_dual > 0) the fill-reducing ordering runs on the leading nc rows only: the
    //          bound rows are inserted at 1c as leaves, so the other rows get the order the reduced system's matrix would get.
    const bool bound_rows = opt.kkt_n_dual > 0 && opt.ordering != 3;
    const int32_t nc = bound_rows ? opt.kkt_n_primal + opt.kkt_n_dual : n;
    if (bound_rows && (opt.kkt_n_primal <= 0 || nc > n)) throw std::runtime_error("invalid kkt_n_primal / kkt_n_dual");
    std::vector<int32_t> perm0;
    if (opt.ordering == 3) {
        if (!user_perm) throw std::runtime_error("user ordering requested but no permutation given");
        perm0.assign(user_perm, user_perm + n);
        std::vector<char> seen(n, 0);
        for (int32_t i = 0; i < n; ++i) {
            if (perm0[i] < 0 || perm0[i] >= n || seen[perm0[i]]) throw std::runtime_error("user_perm is not a permutation");
            seen[perm0[i]] = 1;
        }
    } else if (opt.ordering == 2 || nc < 3) {
        perm0.resize(nc);
        std::iota(perm0.begin(), perm0.end(), 0);
    } else {
        std::vector<int64_t> xadj, adj;
        if (nc == n) build_adjacency(n, colptr, rowval, xadj, adj);
        else {
            std::vector<int32_t> cp(nc + 1, 0), rv;
            rv.reserve(colptr[nc]);
            for (int32_t j = 0; j < nc; ++j) {
                for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) if (rowval[p] < nc) rv.push_back(rowval[p]);
                cp[j + 1] = (int32_t)rv.size();
            }
            build_adjacency(nc, cp.data(), rv.data(), xadj, adj);
        }
        if (opt.ordering == 1 || adj.empty()) order_mindeg(nc, xadj, adj, perm0);
        else order_metis(nc, xadj, adj, perm0);
    }
    std::vector<int32_t> iperm(n);
    for (int32_t i = 0; i < nc; ++i) iperm[perm0[i]] = i;

    timer.lap("ordering");
    // ---- 1b. augmented-KKT constraint.  With static (1 x 1) pivoting a dual row of [[H, J'], [J, -D]] (D possibly zero) gets a
    //          usable pivot only from primal neighbours eliminated BEFORE it, and two duals must not rely on the same single
    //          neighbour u: after u their Schur block is the rank-one -(a_i a_j)/d_u and the second pivot cancels exactly.
    //          So every dual is MATCHED with a distinct primal neighbour that precedes it (in effect a 2 x 2 pivot {u, v} spread
    //          over two consecutive 1 x 1 steps): duals are visited in elimination order; a dual keeps its place if an unused
    //          neighbour already precedes it, otherwise it is moved to just after its earliest unused neighbour (or, if every
    //          neighbour is taken, after its last neighbour).  Quasi-definite / condensed matrices do not need this (kkt_n_primal = 0).
    //          Only the constraint duals [kkt_n_primal, nc) take part; bound rows are placed at 1c.
    std::vector<std::pair<int32_t, int32_t>> pairs;            // PAIRS: (primal, its matched dual), original numbering
    if (opt.kkt_n_primal > 0 && opt.kkt_n_primal < nc && opt.ordering != 3) {
        const int32_t np_ = opt.kkt_n_primal;
        const int32_t nd_ = nc - np_;
        // primal neighbours of every dual (lower CSC: entry (i, j), i >= np_ > j, sits in column j)
        std::vector<int64_t> dptr(nd_ + 1, 0);
        for (int32_t j = 0; j < np_; ++j)
            for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) if (rowval[p] >= np_ && rowval[p] < nc) dptr[rowval[p] - np_ + 1]++;
        for (int32_t v = 0; v < nd_; ++v) dptr[v + 1] += dptr[v];
        std::vector<int32_t> dnb(dptr[nd_]);
        {
            std::vector<int64_t> fill(dptr.begin(), dptr.end() - 1);
            for (int32_t j = 0; j < np_; ++j)
                for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p)
                    if (rowval[p] >= np_ && rowval[p] < nc) dnb[fill[rowval[p] - np_]++] = j;
        }
        for (int32_t v = 0; v < nd_; ++v)                     // neighbours in elimination order
            std::sort(dnb.begin() + dptr[v], dnb.begin() + dptr[v + 1], [&](int32_t a, int32_t b) { return iperm[a] < iperm[b]; });
        std::vector<int32_t> duals(nd_);
        std::iota(duals.begin(), duals.end(), np_);
        std::sort(duals.begin(), duals.end(), [&](int32_t a, int32_t b) { return iperm[a] < iperm[b]; });
        std::vector<char> used(np_, 0);
        std::vector<int32_t> jdeg(opt.pairs ? np_ : 0, 0);    // dual neighbours of each primal
        for (int64_t q = 0; q < (opt.pairs ? dptr[nd_] : 0); ++q) jdeg[dnb[q]]++;
        std::vector<std::pair<int64_t, int32_t>> key(nc);
        for (int32_t v = 0; v < nc; ++v) key[v] = {2 * (int64_t)iperm[v], iperm[v]};
        for (int32_t v : duals) {
            const int64_t a = dptr[v - np_], b = dptr[v - np_ + 1];
            if (a == b) continue;                              // isolated dual row: nothing can help it
            int32_t partner = -1;
            if (opt.pairs) {
                // PAIRS: EVERY dual that can be matched goes immediately after its partner (key second -1: ahead of an unmatched dual
                // placed after the same row), so that the two can form one 2 x 2 pivot.  Partner: the unused neighbour with the fewest
                // dual neighbours (a column with one constraint, such as a free LP column, has no other dual to pair with), ties to
                // the closest one that precedes the dual (it moves least), else to the earliest one after it.
                auto better = [&](int32_t x, int32_t y) {      // x preferred over the current choice y
                    if (y < 0) return true;
                    if (jdeg[x] != jdeg[y]) return jdeg[x] < jdeg[y];
                    const bool xb = iperm[x] < iperm[v], yb = iperm[y] < iperm[v];
                    if (xb != yb) return xb;
                    return xb ? iperm[x] > iperm[y] : iperm[x] < iperm[y];
                };
                for (int64_t q = a; q < b; ++q) if (!used[dnb[q]] && better(dnb[q], partner)) partner = dnb[q];
                if (partner >= 0) { used[partner] = 1; key[v] = {2 * (int64_t)iperm[partner] + 1, -1}; pairs.push_back({partner, v}); }
                else key[v] = {2 * (int64_t)std::max(iperm[dnb[b - 1]], iperm[v]) + 1, iperm[v]};
                continue;
            }
            for (int64_t q = a; q < b && iperm[dnb[q]] < iperm[v]; ++q) if (!used[dnb[q]]) { partner = dnb[q]; break; }
            if (partner >= 0) { used[partner] = 1; continue; } // an own preceding neighbour exists: the dual stays where it is
            for (int64_t q = a; q < b; ++q) if (!used[dnb[q]]) { partner = dnb[q]; break; }
            if (partner >= 0) { used[partner] = 1; key[v] = {2 * (int64_t)iperm[partner] + 1, iperm[v]}; }
            else key[v] = {2 * (int64_t)std::max(iperm[dnb[b - 1]], iperm[v]) + 1, iperm[v]};
        }
        std::vector<int32_t> ord(nc);
        std::iota(ord.begin(), ord.end(), 0);
        std::sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) { return key[a] < key[b]; });
        perm0 = ord;
        for (int32_t i = 0; i < nc; ++i) iperm[perm0[i]] = i;
    }
    // ---- 1c. bound-dual rows of the unreduced KKT system: row b = [l_diag, sqrt(z)] couples only to its variable u.  Eliminated
    //          first, its pivot l_diag (< 0) adds -z / l_diag to u's pivot: the reduced system's barrier term.  Eliminated after u, it
    //          would leave u the pivot H_uu + reg, which is 0 for an LP.  So each bound row goes immediately before u.
    std::vector<int32_t> bnb;                                  // neighbour of bound row nc + k
    if (nc < n) {
        std::vector<int32_t> cnt;
        bound_neighbours(n, colptr, rowval, nc, bnb, cnt);
        const int32_t np_ = opt.kkt_n_primal;
        std::vector<int32_t> bptr(np_ + 1, 0);
        for (int32_t k = 0; k < n - nc; ++k) {
            if (cnt[k] != 1 || bnb[k] < 0 || bnb[k] >= np_) throw std::runtime_error("bound row without exactly one primal neighbour");
            bptr[bnb[k] + 1]++;
        }
        for (int32_t u = 0; u < np_; ++u) bptr[u + 1] += bptr[u];
        std::vector<int32_t> brow(n - nc);
        {
            std::vector<int32_t> fill(bptr.begin(), bptr.end() - 1);
            for (int32_t k = 0; k < n - nc; ++k) brow[fill[bnb[k]]++] = nc + k;
        }
        std::vector<int32_t> ord;
        ord.reserve(n);
        for (int32_t v : perm0) {
            if (v < np_) ord.insert(ord.end(), brow.begin() + bptr[v], brow.begin() + bptr[v + 1]);
            ord.push_back(v);
        }
        perm0.swap(ord);
        for (int32_t i = 0; i < n; ++i) iperm[perm0[i]] = i;
    }

    timer.lap("kkt ordering constraint");
    // ---- 2. etree + postorder
    std::vector<int64_t> rptr;
    std::vector<int32_t> rcol, parent, post;
    permuted_lower_rows(n, colptr, rowval, iperm, rptr, rcol);
    etree(n, rptr, rcol, parent);
    postorder(n, parent, post);
    std::vector<int32_t> perm1(n);
    for (int32_t k = 0; k < n; ++k) perm1[k] = perm0[post[k]];
    for (int32_t i = 0; i < n; ++i) iperm[perm1[i]] = i;

    timer.lap("etree + postorder");
    // ---- 3. structures under perm1
    permuted_lower_rows(n, colptr, rowval, iperm, rptr, rcol);
    etree(n, rptr, rcol, parent);
    // a bound row is a leaf whose parent is its variable, so it still precedes the variable after the postorder, and amalgamation
    // (children's columns before the parent's) and the final DFS keep that
    for (size_t k = 0; k < bnb.size(); ++k)
        if (parent[iperm[nc + k]] != iperm[bnb[k]]) throw std::runtime_error("internal: a bound row's etree parent is not its variable");
    // a matched pair (u, v) with v right after u and a_vu != 0 has parent(u) = v, and u, the last child of v, stays right before v in
    // the postorder
    for (const auto& pr : pairs)
        if (iperm[pr.second] != iperm[pr.first] + 1 || parent[iperm[pr.first]] != iperm[pr.second])
            throw std::runtime_error("internal: a matched dual does not follow its primal partner as its etree parent");
    std::vector<int64_t> cc;
    colcounts(n, rptr, rcol, parent, cc);

    timer.lap("structures / colcounts");
    // ---- 4. maximal supernodes under perm1
    std::vector<int32_t> fs_first;  // first column of each fundamental/maximal supernode
    for (int32_t j = 0; j < n; ++j) {
        bool join = j > 0 && parent[j - 1] == j && cc[j] == cc[j - 1] - 1;
        if (!join) fs_first.push_back(j);
    }
    const int32_t nfs = (int32_t)fs_first.size();
    fs_first.push_back(n);
    std::vector<int32_t> col2fs(n);
    for (int32_t s = 0; s < nfs; ++s)
        for (int32_t j = fs_first[s]; j < fs_first[s + 1]; ++j) col2fs[j] = s;
    std::vector<int32_t> fpar(nfs, -1);
    for (int32_t s = 0; s < nfs; ++s) {
        int32_t last = fs_first[s + 1] - 1;
        if (parent[last] != -1) fpar[s] = col2fs[parent[last]];
    }

    timer.lap("supernodes");
    // ---- 5. relaxed amalgamation on the supernode tree
    struct Node {
        int64_t w, f, zeros;
        std::vector<std::pair<int32_t, int32_t>> ranges;  // column ranges in perm1 numbering, elimination order
        std::vector<int32_t> kids;
        bool merged = false;
    };
    std::vector<Node> nd(nfs);
    for (int32_t s = 0; s < nfs; ++s) {
        nd[s].w = fs_first[s + 1] - fs_first[s];
        nd[s].f = cc[fs_first[s]];
        nd[s].zeros = 0;
        nd[s].ranges.push_back({fs_first[s], fs_first[s + 1]});
    }
    for (int32_t s = 0; s < nfs; ++s) if (fpar[s] != -1) nd[fpar[s]].kids.push_back(s);
    const int64_t nemin = std::max(1, opt.nemin);
    const double zr = opt.relax_zeros;
    // merge c into p (c's columns first)
    auto merge = [&](int32_t p, int32_t c, int64_t w2, int64_t f2, int64_t z2) {
        std::vector<std::pair<int32_t, int32_t>> r = nd[c].ranges;
        r.insert(r.end(), nd[p].ranges.begin(), nd[p].ranges.end());
        nd[p].ranges.swap(r);
        nd[p].w = w2; nd[p].f = f2; nd[p].zeros = z2;
        auto& pk = nd[p].kids;
        pk.erase(std::find(pk.begin(), pk.end(), c));
        pk.insert(pk.end(), nd[c].kids.begin(), nd[c].kids.end());
        nd[c].kids.clear();
        nd[c].merged = true;
    };
    // PAIRS: a pair split between a child supernode (ending with the primal) and its parent (starting with the dual) is merged
    // whatever it costs, and FIRST, while the parent holds only its own columns: the child's last column then stays adjacent to the
    // parent's first through every later merge and the final DFS.
    std::vector<char> force(nfs, 0);
    for (const auto& pr : pairs) {
        const int32_t j = iperm[pr.first];
        if (col2fs[j] != col2fs[j + 1]) force[col2fs[j]] = 1;
    }
    for (int32_t p = 0; p < nfs; ++p) {  // ascending ids = children before parents
        if (!pairs.empty()) {
            const std::vector<int32_t> kids = nd[p].kids;
            for (int32_t c : kids) {
                if (!force[c]) continue;
                const int64_t w2 = nd[p].w + nd[c].w, f2 = nd[c].w + nd[p].f, nnz2 = trap_nnz(w2, f2);
                merge(p, c, w2, f2, nd[p].zeros + nd[c].zeros + nnz2 - trap_nnz(nd[p].w, nd[p].f) - trap_nnz(nd[c].w, nd[c].f));
            }
        }
        bool again = true;
        while (again) {
            again = false;
            // candidate children, largest front first
            std::vector<int32_t> kids = nd[p].kids;
            std::sort(kids.begin(), kids.end(), [&](int32_t a, int32_t b) { return nd[a].f > nd[b].f; });
            for (int32_t c : kids) {
                int64_t w2 = nd[p].w + nd[c].w;
                int64_t f2 = nd[c].w + nd[p].f;
                int64_t nnz2 = trap_nnz(w2, f2);
                int64_t z2 = nd[p].zeros + nd[c].zeros + nnz2 - trap_nnz(nd[p].w, nd[p].f) - trap_nnz(nd[c].w, nd[c].f);
                double z = (double)z2 / (double)nnz2;
                bool ok = (w2 <= 4) || (w2 <= nemin && z < 0.8) || (w2 <= 3 * nemin && z < zr) || (z < 0.25 * zr);
                // latency rule: an only child is absorbed while the merged front stays team-class -- one level less on the tree's
                // critical path (hand-off + staging per level on the device) for a few explicit zeros in a front of order <= 64
                if (!ok && opt.chain_merge_f > 0 && nd[p].kids.size() == 1 && f2 <= std::min(opt.chain_merge_f, 64)) ok = true;
                if (!ok) continue;
                merge(p, c, w2, f2, z2);
                again = true;
                break;
            }
        }
    }

    timer.lap("amalgamation");
    // ---- 6. final permutation: DFS of the merged tree (subtrees first, then the node's own columns)
    std::vector<int32_t> ord2; ord2.reserve(n);
    std::vector<int32_t> sn_first;  // in final numbering
    {
        std::vector<int32_t> roots;
        for (int32_t s = 0; s < nfs; ++s) if (!nd[s].merged && fpar[s] == -1) roots.push_back(s);
        // a merged child's parent pointer is irrelevant; an unmerged node whose fundamental parent was merged
        // has been re-attached as a kid of the absorbing node, so the roots are exactly the unmerged nodes
        // with no fundamental parent.
        std::vector<std::pair<int32_t, size_t>> st;
        for (int32_t r : roots) {
            st.push_back({r, 0});
            while (!st.empty()) {
                int32_t v = st.back().first;
                size_t& k = st.back().second;
                if (k < nd[v].kids.size()) { int32_t c = nd[v].kids[k++]; st.push_back({c, 0}); }
                else {
                    sn_first.push_back((int32_t)ord2.size());
                    for (auto& rg : nd[v].ranges) for (int32_t j = rg.first; j < rg.second; ++j) ord2.push_back(j);
                    st.pop_back();
                }
            }
        }
        if ((int32_t)ord2.size() != n) throw std::runtime_error("internal: amalgamation lost columns");
        sn_first.push_back(n);
    }
    nd.clear(); nd.shrink_to_fit();
    S.perm.resize(n); S.iperm.resize(n);
    for (int32_t k = 0; k < n; ++k) S.perm[k] = perm1[ord2[k]];
    for (int32_t k = 0; k < n; ++k) S.iperm[S.perm[k]] = k;
    const int32_t ns = (int32_t)sn_first.size() - 1;
    S.nsuper = ns;
    S.sn_first = sn_first;
    std::vector<int32_t> col2sn(n);
    for (int32_t s = 0; s < ns; ++s) for (int32_t j = sn_first[s]; j < sn_first[s + 1]; ++j) col2sn[j] = s;
    S.pair_start.assign(n, 0);
    for (const auto& pr : pairs) {
        const int32_t j = S.iperm[pr.first];
        if (S.iperm[pr.second] != j + 1 || col2sn[j] != col2sn[j + 1])
            throw std::runtime_error("internal: a matched pair is not adjacent inside one supernode");
        S.pair_start[j] = 1;
    }

    timer.lap("final permutation");
    // ---- 7. permuted lower CSC (by column) with source positions
    std::vector<int64_t> cptr(n + 1, 0);
    std::vector<int32_t> crow(nnz);
    std::vector<int64_t> csrc(nnz);
    {
        for (int32_t j = 0; j < n; ++j)
            for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
                int32_t a = S.iperm[rowval[p]], b = S.iperm[j];
                cptr[std::min(a, b) + 1]++;
            }
        for (int32_t j = 0; j < n; ++j) cptr[j + 1] += cptr[j];
        std::vector<int64_t> pos(cptr.begin(), cptr.end() - 1);
        for (int32_t j = 0; j < n; ++j)
            for (int32_t p = colptr[j]; p < colptr[j + 1]; ++p) {
                int32_t a = S.iperm[rowval[p]], b = S.iperm[j];
                int64_t q = pos[std::min(a, b)]++;
                crow[q] = std::max(a, b);
                csrc[q] = p;
            }
    }

    timer.lap("permuted CSC");
    // ---- 8. front row structures (children before parents by construction of the numbering)
    S.rows_ptr.assign(ns + 1, 0);
    S.sn_parent.assign(ns, -1);
    std::vector<std::vector<int32_t>> kids(ns);
    std::vector<std::vector<int32_t>> below(ns);
    {
        std::vector<int32_t> mark(n, -1);
        for (int32_t s = 0; s < ns; ++s) {
            const int32_t c0 = sn_first[s], c1 = sn_first[s + 1];
            auto& bl = below[s];
            for (int32_t c = c0; c < c1; ++c)
                for (int64_t q = cptr[c]; q < cptr[c + 1]; ++q) {
                    int32_t r = crow[q];
                    if (r >= c1 && mark[r] != s) { mark[r] = s; bl.push_back(r); }
                }
            for (int32_t ch : kids[s])
                for (int32_t r : below[ch]) {
                    if (r < c0) throw std::runtime_error("internal: child row precedes parent front");
                    if (r >= c1 && mark[r] != s) { mark[r] = s; bl.push_back(r); }
                }
            std::sort(bl.begin(), bl.end());
            if (!bl.empty()) {
                int32_t p = col2sn[bl[0]];
                S.sn_parent[s] = p;
                kids[p].push_back(s);
            }
            S.rows_ptr[s + 1] = S.rows_ptr[s] + (c1 - c0) + (int64_t)bl.size();
        }
    }
    S.rows.resize(S.rows_ptr[ns]);
    S.lp_off.assign(ns + 1, 0);
    S.max_front = 0;
    for (int32_t s = 0; s < ns; ++s) {
        int64_t o = S.rows_ptr[s];
        const int32_t c0 = sn_first[s], c1 = sn_first[s + 1];
        for (int32_t c = c0; c < c1; ++c) S.rows[o++] = c;
        for (int32_t r : below[s]) S.rows[o++] = r;
        int64_t w = c1 - c0, f = w + (int64_t)below[s].size();
        S.lp_off[s + 1] = S.lp_off[s] + f * w;
        S.nnz_l += trap_nnz(w, f);
        for (int64_t k = 0; k < w; ++k) S.flops += (f - k) * (f - k);
        S.max_front = std::max<int32_t>(S.max_front, (int32_t)f);
    }

    // children lists
    S.child_ptr.assign(ns + 1, 0);
    for (int32_t s = 0; s < ns; ++s) S.child_ptr[s + 1] = S.child_ptr[s] + (int32_t)kids[s].size();
    S.child_idx.resize(S.child_ptr[ns]);
    for (int32_t s = 0; s < ns; ++s) {
        std::sort(kids[s].begin(), kids[s].end());
        std::copy(kids[s].begin(), kids[s].end(), S.child_idx.begin() + S.child_ptr[s]);
    }

    timer.lap("front row structures");
    // ---- 9. relative indices child -> parent front
    S.rel_ptr.assign(ns + 1, 0);
    for (int32_t s = 0; s < ns; ++s) S.rel_ptr[s + 1] = S.rel_ptr[s] + (int64_t)below[s].size();
    S.rel.resize(S.rel_ptr[ns]);
    for (int32_t s = 0; s < ns; ++s) {
        int32_t p = S.sn_parent[s];
        if (p < 0) continue;
        const int32_t p0 = sn_first[p], pw = sn_first[p + 1] - p0;
        const auto& pb = below[p];
        size_t k = 0;
        int64_t o = S.rel_ptr[s];
        for (int32_t r : below[s]) {
            if (r < p0 + pw) S.rel[o++] = r - p0;
            else {
                while (k < pb.size() && pb[k] < r) ++k;
                if (k == pb.size() || pb[k] != r) throw std::runtime_error("internal: child row missing in parent front");
                S.rel[o++] = pw + (int32_t)k;
            }
        }
    }

    timer.lap("relative indices");
    // ---- 10. A -> panel scatter map, grouped by supernode
    S.amap_ptr.assign(ns + 1, 0);
    for (int32_t s = 0; s < ns; ++s) S.amap_ptr[s + 1] = S.amap_ptr[s] + (cptr[sn_first[s + 1]] - cptr[sn_first[s]]);
    S.amap_src.resize(nnz);
    S.amap_dst.resize(nnz);
    for (int32_t s = 0; s < ns; ++s) {
        const int32_t c0 = sn_first[s], c1 = sn_first[s + 1];
        const int64_t w = c1 - c0, f = w + (int64_t)below[s].size();
        const auto& bl = below[s];
        int64_t o = S.amap_ptr[s];
        for (int32_t c = c0; c < c1; ++c)
            for (int64_t q = cptr[c]; q < cptr[c + 1]; ++q) {
                int32_t r = crow[q];
                int64_t pos;
                if (r < c1) pos = r - c0;
                else {
                    auto it = std::lower_bound(bl.begin(), bl.end(), r);
                    pos = w + (it - bl.begin());
                }
                S.amap_src[o] = csrc[q];
                S.amap_dst[o] = S.lp_off[s] + pos + (int64_t)(c - c0) * f;
                ++o;
            }
    }

    timer.lap("scatter map");
    // ---- 11. levels
    S.sn_level.assign(ns, 0);
    for (int32_t s = 0; s < ns; ++s) {
        int32_t p = S.sn_parent[s];
        if (p >= 0) S.sn_level[p] = std::max(S.sn_level[p], S.sn_level[s] + 1);
    }
    S.nlevels = 0;
    for (int32_t s = 0; s < ns; ++s) S.nlevels = std::max(S.nlevels, S.sn_level[s] + 1);
    S.level_ptr.assign(S.nlevels + 1, 0);
    for (int32_t s = 0; s < ns; ++s) S.level_ptr[S.sn_level[s] + 1]++;
    for (int32_t l = 0; l < S.nlevels; ++l) S.level_ptr[l + 1] += S.level_ptr[l];
    S.level_sn.resize(ns);
    {
        std::vector<int32_t> pos(S.level_ptr.begin(), S.level_ptr.end() - 1);
        for (int32_t s = 0; s < ns; ++s) S.level_sn[pos[S.sn_level[s]]++] = s;
    }

    timer.lap("levels");
    // ---- 12. subtree-to-rank partition
    S.owner.assign(ns, 0);
    S.top_rows = 0;
    const int P = std::max(1, opt.n_parts);
    if (P > 1) {
        std::vector<int64_t> work(ns, 0);
        for (int32_t s = 0; s < ns; ++s) {
            int64_t w = sn_first[s + 1] - sn_first[s], f = w + (int64_t)below[s].size();
            for (int64_t k = 0; k < w; ++k) work[s] += (f - k) * (f - k);
            work[s] += 2000;  // fixed per-front latency weight
        }
        std::vector<int64_t> sub(work);
        for (int32_t s = 0; s < ns; ++s) if (S.sn_parent[s] >= 0) sub[S.sn_parent[s]] += sub[s];
        int64_t total = 0;
        for (int32_t s = 0; s < ns; ++s) if (S.sn_parent[s] < 0) total += sub[s];
        std::vector<char> is_top(ns, 0);
        auto cmp = [&](int32_t a, int32_t b) { return sub[a] < sub[b]; };
        std::priority_queue<int32_t, std::vector<int32_t>, decltype(cmp)> cand(cmp);
        for (int32_t s = 0; s < ns; ++s) if (S.sn_parent[s] < 0) cand.push(s);
        int64_t top_work = 0;
        std::vector<int32_t> best_assign;
        for (int iter = 0; iter < 100000; ++iter) {
            // LPT packing of the current candidates
            std::vector<int32_t> c;
            { auto q = cand; while (!q.empty()) { c.push_back(q.top()); q.pop(); } }
            std::vector<int64_t> load(P, 0);
            for (int32_t s : c) { int r = (int)(std::min_element(load.begin(), load.end()) - load.begin()); load[r] += sub[s]; }
            int64_t mx = *std::max_element(load.begin(), load.end());
            int64_t sumc = std::accumulate(load.begin(), load.end(), (int64_t)0);
            bool balanced = (double)mx <= 1.10 * (double)sumc / P + 1.0;
            if ((balanced && (int)c.size() >= P) || cand.empty()) break;
            int32_t h = cand.top();
            if (kids[h].empty()) break;  // cannot split a leaf
            if (top_work + work[h] > total / 4 && (int)c.size() >= P) break;  // do not let the replicated part dominate
            cand.pop();
            is_top[h] = 1; top_work += work[h];
            for (int32_t k : kids[h]) cand.push(k);
        }
        std::vector<int32_t> c;
        while (!cand.empty()) { c.push_back(cand.top()); cand.pop(); }
        std::vector<int64_t> load(P, 0);
        std::vector<int32_t> root_owner(ns, -2);
        for (int32_t s : c) { int r = (int)(std::min_element(load.begin(), load.end()) - load.begin()); load[r] += sub[s]; root_owner[s] = r; }
        for (int32_t s = ns - 1; s >= 0; --s) {  // parents before children
            if (is_top[s]) { S.owner[s] = -1; S.top_rows += sn_first[s + 1] - sn_first[s]; }
            else if (root_owner[s] >= 0) S.owner[s] = root_owner[s];
            else S.owner[s] = S.owner[S.sn_parent[s]];
        }
    }

    timer.lap("partition");
    // ---- 13. update-block offsets: blocks crossing from an owned subtree into the shared top tree first
    S.cb_off.assign(ns + 1, 0);
    {
        int64_t off = 0;
        std::vector<int64_t> o(ns, 0);
        for (int pass = 0; pass < 2; ++pass) {
            for (int32_t s = 0; s < ns; ++s) {
                int32_t p = S.sn_parent[s];
                bool boundary = (P > 1) && S.owner[s] >= 0 && p >= 0 && S.owner[p] == -1;
                if ((pass == 0) != boundary) continue;
                int64_t r = (int64_t)below[s].size();
                o[s] = off;
                off += (r * r + 1) & ~(int64_t)1;      // even number of doubles: 16-byte aligned blocks (cp.async.cg)
            }
            if (pass == 0) S.exch_cb = off;
        }
        // cb_off is indexed by supernode, not cumulative: store start offsets; cb_off[ns] = total
        for (int32_t s = 0; s < ns; ++s) S.cb_off[s] = o[s];
        S.cb_off[ns] = off;
    }
}

}  // namespace b2
