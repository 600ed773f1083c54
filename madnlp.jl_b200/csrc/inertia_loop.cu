// The trials of inertia_correction! after a wrong first inertia as ONE CUDA graph (IPMLinearAlgebra._inertia_correction,
// madnlp.jl_b200/ipm.py):
//     WHILE { schedule ; regularise ; the caller's build_kkt + factorize ; trial test ;
//             IF { b2_richardson_begin ; WHILE { the caller's refinement step ; k_refine_test } } ; close }
// Three nested conditional nodes (CUDA >= 12.4), all handles created on the top graph.  The schedule, the regularisation, the
// inertia test and the acceptance rule are the host loop's, operation for operation, so every trial is bit-identical to it; the
// host waits once per step for all the trials instead of once per trial and once per refinement step.
#include <atomic>
#include <cmath>
#include <cstring>

#include "common.cuh"

using namespace b2;

namespace {

// the schedule's state on the device.  Each launch stages it whole: the launch parameters, zeros, and the inertia of the first trial
struct TrialState {
    double del_w_last;            // the host's del_w_last (constant over a step)
    double del_c;                 // jacobian_regularization_value * mu^jacobian_regularization_exponent
    double dw, dc;                // the regularisation of the trial in progress
    int32_t fault;                // the last factorisation's counters report a timed-out wait
    int32_t reserved;
    b2_inertia_record rec;        // the record in progress (rec.seq: the number this launch writes)
};

}  // namespace

struct b2_inertia_loop {
    b2_inertia_options opt{};
    int64_t cap = 0;                               // entries of the del_w list (b2_inertia_trial_bound)
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraph_t body = nullptr;                    // the outer WHILE's body
    cudaGraphNode_t if_node = nullptr;             // the IF node in it, which the close follows
    cudaGraphConditionalHandle c_loop = 0, c_if = 0, c_refine = 0;
    int stage = 0;                                 // 1: body being captured, 2: refinement body being captured, 3: built
    b2_inertia_source src{};
    int64_t expect_pos = -1, expect_neg = -1;
    const double* norms = nullptr;
    DevBuf<TrialState> state;
    DevBuf<double> del_w;                          // the del_w of each trial
    DevBuf<b2_refine_record> rrec, rout;           // k_refine_test's record in progress and its last record (device)
    TrialState* stage_h = nullptr;                 // pinned: what a launch copies into `state`
    b2_inertia_record* rec_h = nullptr;            // pinned, written by the close
    double* del_w_h = nullptr;                     // pinned, written by the close
    cudaStream_t stream = nullptr;                 // of the last launch
    int64_t launched = 0;
    void drop() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        exec = nullptr; graph = nullptr; body = nullptr; if_node = nullptr; stage = 0;
    }
    ~b2_inertia_loop() {
        drop();
        if (stage_h) cudaFreeHost(stage_h);
        if (rec_h) cudaFreeHost(rec_h);
        if (del_w_h) cudaFreeHost(del_w_h);
    }
};

namespace {

// Python's max(a, b): a unless b is greater
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }

// the del_w of the next trial (IPMLinearAlgebra._trials_from)
__device__ __forceinline__ double next_del_w(const TrialState& t, const b2_inertia_options& o) {
    if (t.rec.trials == 0)
        return t.del_w_last == 0.0 ? o.first_hessian_perturbation : py_max(o.min_hessian_perturbation, __dmul_rn(o.perturb_dec_fact, t.del_w_last));
    return __dmul_rn(t.rec.del_w, t.del_w_last == 0.0 ? o.perturb_inc_fact_first : o.perturb_inc_fact);
}

// one thread: del_w and del_c of the trial, the differences the regularisation adds, the list.  (The close has already stopped the
// loop when this del_w is past max_hessian_perturbation; the first regularised trial is never refused, as on the host.)
__global__ void k_trial_schedule(TrialState* __restrict__ s, b2_inertia_options o, int32_t dual_always, double* __restrict__ list) {
    TrialState t = *s;
    const double del_w = next_del_w(t, o);
    const double del_c = (dual_always || t.rec.num_zero != 0) ? t.del_c : 0.0;
    t.dw = __dsub_rn(del_w, t.rec.del_w_prev);
    t.dc = __dsub_rn(del_c, t.rec.del_c_prev);
    t.rec.del_w = del_w;
    t.rec.del_w_prev = del_w;
    t.rec.del_c_prev = del_c;
    list[t.rec.trials] = del_w;
    t.rec.trials += 1;
    *s = t;
}

// b2_regularize_diagonal's pass (k_regularize) with dw, dc read from the device: reg += dw ; pr_diag += dw ; du_diag -= dc.
// SCALED: b2_scaled_regularize_diagonal's (k_scaled_regularize): pr_diag += dw (s s) with the scaling factor s of K2.5
template <bool SCALED>
__global__ void k_trial_regularize(const TrialState* __restrict__ s, int64_t n_tot, int64_t m, double* __restrict__ reg,
                                   double* __restrict__ pr, double* __restrict__ du, const double* __restrict__ sf) {
    const double dw = s->dw, dc = s->dc;
    GRID_STRIDE(i, n_tot + m) {
        if (SCALED) {
            if (i < n_tot) {
                const double f = sf[i];
                reg[i] = __dadd_rn(reg[i], dw);
                pr[i] = __dadd_rn(pr[i], __dmul_rn(dw, __dmul_rn(f, f)));
            } else {
                du[i - n_tot] = __dsub_rn(du[i - n_tot], dc);
            }
        } else {
            if (i < n_tot) { reg[i] += dw; pr[i] += dw; }
            else du[i - n_tot] -= dc;
        }
    }
}

// one thread after the factorisation: the inertia as b2_inertia_fetch reads it and the KKT type's test (as k_refine_test);
// only a right inertia runs the refinement
__global__ void k_trial_test(TrialState* __restrict__ s, b2_inertia_source src, int64_t expect_pos, int64_t expect_neg,
                             cudaGraphConditionalHandle c_if, cudaGraphConditionalHandle c_refine) {
    TrialState t = *s;
    const int32_t* c = src.counters_d;
    int64_t neg = 0, zero = 0;
    for (int k = 0; k < 2; ++k) {
        if (src.neg[k] >= 0) neg += c[src.neg[k]];
        if (src.zero[k] >= 0) zero += c[src.zero[k]];
    }
    t.rec.num_neg = neg; t.rec.num_zero = zero; t.rec.num_pos = src.n - neg - zero;
    t.fault = c[src.fail] != 0;
    t.rec.inertia_ok = !t.fault && zero == 0 && (expect_pos < 0 || t.rec.num_pos == expect_pos) && (expect_neg < 0 || neg == expect_neg);
    *s = t;
    cudaGraphSetConditional(c_if, t.rec.inertia_ok ? 1u : 0u);
    cudaGraphSetConditional(c_refine, 1u);
}

// one thread at the end of a trial: accept, go round again, fail or hand over; on stopping, the record and the list go to the host,
// the sequence number last (b2_inertia_loop_wait polls it)
__global__ void k_trial_close(TrialState* __restrict__ s, const b2_refine_record* __restrict__ refined, b2_inertia_options o,
                              double acceptable_tol, cudaGraphConditionalHandle c_loop, const double* __restrict__ list,
                              b2_inertia_record* out, double* list_out) {
    TrialState t = *s;
    int32_t status = 0;
    if (t.fault) {
        status = B2_TRIALS_FAULT;
    } else if (t.rec.inertia_ok) {
        t.rec.ir = refined->ir;
        t.rec.ratio = refined->ratio;            // 0 when ||b|| == 0, as solve_refine! leaves it
        if (t.rec.ratio < acceptable_tol) {
            status = B2_TRIALS_ACCEPTED;
            t.rec.ir_total += t.rec.ir;
        } else {
            status = B2_TRIALS_HANDOVER;
        }
    } else if (next_del_w(t, o) > o.max_hessian_perturbation) {
        status = B2_TRIALS_FAILED;
    }
    t.rec.status = status;
    *s = t;
    if (status) {
        for (int64_t k = 0; k < t.rec.trials; ++k) list_out[k] = list[k];
        b2_inertia_record r = t.rec;
        r.seq = t.rec.seq - 1;
        *out = r;
        __threadfence_system();
        *(volatile int64_t*)&out->seq = t.rec.seq;
    }
    cudaGraphSetConditional(c_loop, status ? 0u : 1u);
}

int fail_build(b2_inertia_loop* h, cudaStream_t st, cudaError_t e, const char* what) {
    abort_capture(st);
    h->drop();
    if (conditional_unsupported(e)) {
        set_error(std::string(what) + ": conditional CUDA graph nodes are not available (" + cudaGetErrorString(e) + ")");
        return B2_ERR_UNSUPPORTED;
    }
    return cuda_fail(e, what, __FILE__, __LINE__);
}

#define IL_TRY(call, what) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return fail_build(h, st, e__, what); } while (0)

// a conditional node of `type` after deps in g; its body graph in *body
cudaError_t add_conditional(cudaGraph_t g, const cudaGraphNode_t* deps, size_t ndeps, cudaGraphConditionalHandle c,
                            cudaGraphConditionalNodeType type, cudaGraphNode_t* node, cudaGraph_t* body) {
    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = c;
    p.conditional.type = type;
    p.conditional.size = 1;
    cudaError_t e = cudaGraphAddNode(node, g, deps, ndeps, &p);
    if (e == cudaSuccess) *body = p.conditional.phGraph_out[0];
    return e;
}

// ends the capture into the current graph and adds a conditional node after what it captured; *body: the node's body graph
cudaError_t close_with_conditional(cudaStream_t st, cudaGraphConditionalHandle c, cudaGraphConditionalNodeType type,
                                   cudaGraphNode_t* node, cudaGraph_t* body) {
    cudaStreamCaptureStatus cs;
    cudaGraph_t g = nullptr;
    const cudaGraphNode_t* deps = nullptr;
    size_t ndeps = 0;
    cudaError_t e = cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &ndeps);
    if (e == cudaSuccess) e = add_conditional(g, deps, ndeps, c, type, node, body);
    cudaGraph_t ended = nullptr;
    const cudaError_t e2 = cudaStreamEndCapture(st, &ended);
    return e != cudaSuccess ? e : e2;
}

}  // namespace

extern "C" {

int b2_inertia_trial_bound(const b2_inertia_options* o, int64_t* out) {
    if (!o || !out) { set_error("b2_inertia_trial_bound: invalid argument"); return B2_ERR_INVALID; }
    const double f = std::min(o->perturb_inc_fact_first, o->perturb_inc_fact);
    double d = std::min(o->min_hessian_perturbation, o->first_hessian_perturbation);
    const double mx = o->max_hessian_perturbation;
    if (!(f > 1.0) || !(d > 0.0) || !std::isfinite(f) || !std::isfinite(mx)) {
        set_error("b2_inertia_trial_bound: the del_w schedule of these options is unbounded");
        return B2_ERR_UNSUPPORTED;
    }
    // the first trial is never refused; every later one multiplies and is refused past the bound (the host's order of operations)
    int64_t n = 1;
    for (;;) {
        d = d * f;
        if (d > mx) break;
        if (++n > (int64_t(1) << 20)) { set_error("b2_inertia_trial_bound: more than 2^20 trials"); return B2_ERR_UNSUPPORTED; }
    }
    *out = n;
    return B2_OK;
}

int b2_inertia_loop_create(const b2_inertia_options* opt, b2_inertia_loop** out) {
    if (!opt || !out) { set_error("b2_inertia_loop_create: invalid argument"); return B2_ERR_INVALID; }
    int64_t cap = 0;
    const int rc = b2_inertia_trial_bound(opt, &cap);
    if (rc != B2_OK) return rc;
    b2_inertia_loop* h = new b2_inertia_loop();
    h->opt = *opt;
    h->cap = cap;
    cudaError_t e = h->state.alloc(1);
    if (e == cudaSuccess) e = h->del_w.alloc(cap);
    if (e == cudaSuccess) e = h->rrec.alloc(1);
    if (e == cudaSuccess) e = h->rout.alloc(1);
    if (e == cudaSuccess) e = cudaMemset(h->rrec.p, 0, sizeof(b2_refine_record));
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h->stage_h, sizeof(TrialState));
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h->rec_h, sizeof(b2_inertia_record));
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h->del_w_h, cap * sizeof(double));
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "b2_inertia_loop_create", __FILE__, __LINE__); }
    std::memset(h->stage_h, 0, sizeof(TrialState));
    std::memset(h->rec_h, 0, sizeof(b2_inertia_record));
    *out = h;
    return B2_OK;
}

int b2_inertia_loop_destroy(b2_inertia_loop* h) {
    delete h;
    return B2_OK;
}

namespace {
int inertia_loop_begin(b2_inertia_loop* h, int64_t n_tot, int64_t m, double* reg_d, double* pr_diag_d, double* du_diag_d,
                       const double* scaling_d, int32_t dual_always, void* stream) {
    cudaStream_t st = as_stream(stream);
    h->drop();
    IL_TRY(cudaGraphCreate(&h->graph, 0), "cudaGraphCreate");
    IL_TRY(cudaGraphConditionalHandleCreate(&h->c_loop, h->graph, 1, cudaGraphCondAssignDefault), "cudaGraphConditionalHandleCreate");
    IL_TRY(cudaGraphConditionalHandleCreate(&h->c_if, h->graph, 0, cudaGraphCondAssignDefault), "cudaGraphConditionalHandleCreate");
    IL_TRY(cudaGraphConditionalHandleCreate(&h->c_refine, h->graph, 1, cudaGraphCondAssignDefault), "cudaGraphConditionalHandleCreate");
    cudaGraphNode_t loop = nullptr;
    IL_TRY(add_conditional(h->graph, nullptr, 0, h->c_loop, cudaGraphCondTypeWhile, &loop, &h->body), "cudaGraphAddNode(WHILE)");
    IL_TRY(cudaStreamBeginCaptureToGraph(st, h->body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph(trial)");
    h->stage = 1;
    k_trial_schedule<<<1, 1, 0, st>>>(h->state.p, h->opt, dual_always ? 1 : 0, h->del_w.p);
    IL_TRY(cudaGetLastError(), "k_trial_schedule");
    if (n_tot + m) {
        if (scaling_d) k_trial_regularize<true><<<grid_elem(n_tot + m), 256, 0, st>>>(h->state.p, n_tot, m, reg_d, pr_diag_d, du_diag_d, scaling_d);
        else k_trial_regularize<false><<<grid_elem(n_tot + m), 256, 0, st>>>(h->state.p, n_tot, m, reg_d, pr_diag_d, du_diag_d, nullptr);
        IL_TRY(cudaGetLastError(), "k_trial_regularize");
    }
    return B2_OK;
}
}  // namespace

int b2_inertia_loop_begin(b2_inertia_loop* h, int64_t n_tot, int64_t m, double* reg_d, double* pr_diag_d, double* du_diag_d,
                          int32_t dual_always, void* stream) {
    if (!h || n_tot < 0 || m < 0 || (n_tot && (!reg_d || !pr_diag_d)) || (m && !du_diag_d)) {
        set_error("b2_inertia_loop_begin: invalid argument");
        return B2_ERR_INVALID;
    }
    return inertia_loop_begin(h, n_tot, m, reg_d, pr_diag_d, du_diag_d, nullptr, dual_always, stream);
}

int b2_inertia_loop_begin_scaled(b2_inertia_loop* h, int64_t n_tot, int64_t m, double* reg_d, double* pr_diag_d, double* du_diag_d,
                                 const double* scaling_d, int32_t dual_always, void* stream) {
    if (!h || n_tot < 0 || m < 0 || (n_tot && (!reg_d || !pr_diag_d || !scaling_d)) || (m && !du_diag_d)) {
        set_error("b2_inertia_loop_begin_scaled: invalid argument");
        return B2_ERR_INVALID;
    }
    return inertia_loop_begin(h, n_tot, m, reg_d, pr_diag_d, du_diag_d, scaling_d, dual_always, stream);
}

int b2_inertia_loop_refine(b2_inertia_loop* h, const b2_inertia_source* src, int64_t expect_pos, int64_t expect_neg, int64_t n,
                           const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream) {
    cudaStream_t st = as_stream(stream);
    if (!h || h->stage != 1 || !src || !src->counters_d || src->fail < 0 || src->neg[0] < 0 || src->zero[0] < 0 || n < 0 || !norms_d ||
        (n && (!b_d || !w_d || !x_d))) {
        if (h && h->stage) { abort_capture(st); h->drop(); }
        set_error("b2_inertia_loop_refine: invalid argument (or no b2_inertia_loop_begin before it)");
        return B2_ERR_INVALID;
    }
    h->src = *src; h->expect_pos = expect_pos; h->expect_neg = expect_neg; h->norms = norms_d;
    k_trial_test<<<1, 1, 0, st>>>(h->state.p, *src, expect_pos, expect_neg, h->c_if, h->c_refine);
    IL_TRY(cudaGetLastError(), "k_trial_test");
    cudaGraph_t refine = nullptr, steps = nullptr;
    cudaGraphNode_t loop = nullptr;
    IL_TRY(close_with_conditional(st, h->c_if, cudaGraphCondTypeIf, &h->if_node, &refine), "cudaGraphAddNode(IF)");
    IL_TRY(cudaStreamBeginCaptureToGraph(st, refine, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph(IF)");
    if (b2_richardson_begin(n, b_d, w_d, x_d, norms_d + 2, st) != B2_OK) return fail_build(h, st, cudaGetLastError(), "b2_richardson_begin");
    IL_TRY(close_with_conditional(st, h->c_refine, cudaGraphCondTypeWhile, &loop, &steps), "cudaGraphAddNode(WHILE refine)");
    IL_TRY(cudaStreamBeginCaptureToGraph(st, steps, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph(refine)");
    h->stage = 2;
    return B2_OK;
}

int b2_inertia_loop_end(b2_inertia_loop* h, int32_t max_iter, double tol, double acceptable_tol, void* stream) {
    cudaStream_t st = as_stream(stream);
    if (!h || h->stage != 2) {
        if (h && h->stage) { abort_capture(st); h->drop(); }
        set_error("b2_inertia_loop_end: no b2_inertia_loop_refine before it");
        return B2_ERR_INVALID;
    }
    IL_TRY(launch_refine_test(st, h->c_refine, h->norms, h->src, h->expect_pos, h->expect_neg, max_iter, tol, h->rrec.p, h->rout.p),
           "k_refine_test");
    cudaGraph_t g = nullptr;
    IL_TRY(cudaStreamEndCapture(st, &g), "cudaStreamEndCapture(refine)");
    IL_TRY(cudaStreamBeginCaptureToGraph(st, h->body, &h->if_node, nullptr, 1, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph(close)");
    k_trial_close<<<1, 1, 0, st>>>(h->state.p, h->rout.p, h->opt, acceptable_tol, h->c_loop, h->del_w.p, h->rec_h, h->del_w_h);
    IL_TRY(cudaGetLastError(), "k_trial_close");
    IL_TRY(cudaStreamEndCapture(st, &g), "cudaStreamEndCapture(trial)");
    IL_TRY(cudaGraphInstantiate(&h->exec, h->graph, 0), "cudaGraphInstantiate");
    h->stage = 3;
    return B2_OK;
}

int b2_inertia_loop_launch(b2_inertia_loop* h, double del_w_last, double del_c, int64_t num_zero, void* stream) {
    if (!h || !h->exec) { set_error("b2_inertia_loop_launch: no graph built"); return B2_ERR_INVALID; }
    if (h->rec_h->seq != h->launched) { set_error("b2_inertia_loop_launch: the last launch has not been waited for"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    TrialState t{};
    t.del_w_last = del_w_last;
    t.del_c = del_c;
    t.rec.num_zero = num_zero;
    t.rec.seq = h->launched + 1;
    *h->stage_h = t;
    B2_CUDA(cudaMemcpyAsync(h->state.p, h->stage_h, sizeof(TrialState), cudaMemcpyHostToDevice, st));
    B2_CUDA(cudaGraphLaunch(h->exec, st));
    h->stream = st;
    h->launched += 1;
    return B2_OK;
}

int b2_inertia_loop_wait(b2_inertia_loop* h) {
    if (!h || !h->launched) { set_error("b2_inertia_loop_wait: nothing launched"); return B2_ERR_INVALID; }
    const volatile int64_t* seq = &h->rec_h->seq;
    while (*seq != h->launched) {
        const cudaError_t e = cudaStreamQuery(h->stream);
        if (e == cudaSuccess) {
            if (*seq == h->launched) break;
            set_error("b2_inertia_loop_wait: the graph finished without its record");
            return B2_ERR_CUDA;
        }
        if (e != cudaErrorNotReady) return cuda_fail(e, "b2_inertia_loop_wait", __FILE__, __LINE__);
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return B2_OK;
}

int b2_inertia_loop_record(b2_inertia_loop* h, b2_inertia_record* out, double* del_w_out, int64_t cap) {
    if (!h || !out || cap < 0 || (cap && !del_w_out)) { set_error("b2_inertia_loop_record: invalid argument"); return B2_ERR_INVALID; }
    *out = *h->rec_h;
    const int64_t k = std::min(std::min(cap, out->trials), h->cap);
    if (k > 0) std::memcpy(del_w_out, h->del_w_h, (size_t)k * sizeof(double));
    return B2_OK;
}

}  // extern "C"
