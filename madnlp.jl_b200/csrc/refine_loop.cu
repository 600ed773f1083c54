// Richardson refinement of the first trial as ONE CUDA graph (RichardsonIterator.start / solve_refine, madnlp.jl_b200/richardson.py):
//     b2_richardson_begin ; WHILE { the caller's refinement step ; k_refine_test }
// The body runs under a conditional WHILE node (CUDA >= 12.4); k_refine_test applies solve_refine!'s stopping rule and the KKT
// type's inertia test on the device and sets the node's condition, so the host synchronises once per solve instead of once per
// refinement step.  The arithmetic of every step is the caller's, unchanged: a solve through this graph is bit-identical to the
// host loop.
#include <atomic>
#include <cstring>

#include "common.cuh"

using namespace b2;

struct b2_refine_loop {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraphNode_t node = nullptr;                // the WHILE node (its body is being captured between begin and end)
    cudaGraphConditionalHandle cond = 0;
    DevBuf<b2_refine_record> rec;                  // the record of the solve in progress; zero between solves
    b2_refine_record* rec_h = nullptr;             // pinned (and, with unified addressing, written by the device directly)
    const double* norms = nullptr;
    cudaStream_t stream = nullptr;                 // of the last launch
    int64_t launched = 0;                          // solves launched; rec_h->seq counts the ones finished
    void drop() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        exec = nullptr; graph = nullptr; node = nullptr;
    }
    ~b2_refine_loop() {
        drop();
        if (rec_h) cudaFreeHost(rec_h);
    }
};

namespace {

// one thread, after each refinement step.  RichardsonIterator.solve_refine's loop, operation for operation:
//     residual_ratio = norm_w / (min(norm_x, 1e6 * norm_b) + norm_b) ; ir += 1 ; stop if ir >= max_iter or ratio < tol
// Python's min(a, b) returns b only when b < a; the _rn intrinsics keep the compiler from contracting anything.
__global__ void k_refine_test(cudaGraphConditionalHandle cond, const double* __restrict__ norms, b2_inertia_source src,
                              int64_t expect_pos, int64_t expect_neg, int32_t max_iter, double tol, b2_refine_record* rec,
                              b2_refine_record* out) {
    const double nw = norms[0], nx = norms[1], nb = norms[2];
    b2_refine_record r = *rec;
    bool more = false;
    r.steps += 1;
    if (r.steps == 1) {
        // the step ran speculatively, before the host knew the inertia: read it as b2_inertia_fetch does
        const int32_t* c = src.counters_d;
        int64_t neg = 0, zero = 0;
        for (int k = 0; k < 2; ++k) {
            if (src.neg[k] >= 0) neg += c[src.neg[k]];
            if (src.zero[k] >= 0) zero += c[src.zero[k]];
        }
        r.num_neg = neg; r.num_zero = zero; r.num_pos = src.n - neg - zero;
        r.fail = c[src.fail];
        r.inertia_ok = r.fail == 0 && zero == 0 && (expect_pos < 0 || r.num_pos == expect_pos) && (expect_neg < 0 || neg == expect_neg);
        r.norm_b = nb;
    }
    r.norm_w = nw; r.norm_x = nx;
    if (r.inertia_ok && nb != 0.0) {
        const double c = __dmul_rn(1e6, nb);
        r.ratio = __ddiv_rn(nw, __dadd_rn(c < nx ? c : nx, nb));
        r.ir += 1;
        more = !(r.ir >= max_iter || r.ratio < tol);
    }
    if (more) {
        *rec = r;
    } else {
        // the last step: the record goes to the host, its sequence number last (b2_refine_loop_wait polls it), and the next solve
        // starts from zero
        *out = r;
        __threadfence_system();
        *(volatile int64_t*)&out->seq = r.seq + 1;
        b2_refine_record z{};
        z.seq = r.seq + 1;
        *rec = z;
    }
    cudaGraphSetConditional(cond, more ? 1u : 0u);
}

}  // namespace

namespace b2 {

bool conditional_unsupported(cudaError_t e) { return e == cudaErrorNotSupported || e == cudaErrorCallRequiresNewerDriver; }

void abort_capture(cudaStream_t st) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
        cudaGraph_t g = nullptr;
        cudaStreamEndCapture(st, &g);       // (capture-to-graph: g is the owner's own graph, dropped by the owner)
    }
    cudaGetLastError();
}

cudaError_t launch_refine_test(cudaStream_t st, cudaGraphConditionalHandle cond, const double* norms, const b2_inertia_source& src,
                               int64_t expect_pos, int64_t expect_neg, int32_t max_iter, double tol, b2_refine_record* rec,
                               b2_refine_record* out) {
    k_refine_test<<<1, 1, 0, st>>>(cond, norms, src, expect_pos, expect_neg, max_iter, tol, rec, out);
    return cudaGetLastError();
}

}  // namespace b2

namespace {

// leave no capture open on the stream and drop the half-built graph
void abort_build(b2_refine_loop* h, cudaStream_t st) {
    abort_capture(st);
    h->drop();
}

int fail_build(b2_refine_loop* h, cudaStream_t st, cudaError_t e, const char* what) {
    abort_build(h, st);
    if (conditional_unsupported(e)) {
        set_error(std::string(what) + ": conditional CUDA graph nodes are not available (" + cudaGetErrorString(e) + ")");
        return B2_ERR_UNSUPPORTED;
    }
    return cuda_fail(e, what, __FILE__, __LINE__);
}

#define RL_TRY(call, what) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return fail_build(h, st, e__, what); } while (0)

}  // namespace

extern "C" {

int b2_refine_loop_create(b2_refine_loop** out) {
    if (!out) { set_error("b2_refine_loop_create: invalid argument"); return B2_ERR_INVALID; }
    b2_refine_loop* h = new b2_refine_loop();
    cudaError_t e = h->rec.alloc(1);
    if (e == cudaSuccess) e = cudaMemset(h->rec.p, 0, sizeof(b2_refine_record));
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h->rec_h, sizeof(b2_refine_record));
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "b2_refine_loop_create", __FILE__, __LINE__); }
    std::memset(h->rec_h, 0, sizeof(b2_refine_record));
    *out = h;
    return B2_OK;
}

int b2_refine_loop_destroy(b2_refine_loop* h) {
    delete h;
    return B2_OK;
}

int b2_refine_loop_begin(b2_refine_loop* h, int64_t n, const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream) {
    if (!h || n < 0 || !norms_d || (n && (!b_d || !w_d || !x_d))) { set_error("b2_refine_loop_begin: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    h->drop();
    h->norms = norms_d;
    RL_TRY(cudaGraphCreate(&h->graph, 0), "cudaGraphCreate");
    RL_TRY(cudaStreamBeginCaptureToGraph(st, h->graph, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal), "cudaStreamBeginCaptureToGraph");
    if (b2_richardson_begin(n, b_d, w_d, x_d, norms_d + 2, st) != B2_OK) return fail_build(h, st, cudaGetLastError(), "b2_richardson_begin");
    cudaStreamCaptureStatus cs;
    cudaGraph_t g = nullptr;
    const cudaGraphNode_t* deps = nullptr;
    size_t ndeps = 0;
    RL_TRY(cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &ndeps), "cudaStreamGetCaptureInfo");
    RL_TRY(cudaGraphConditionalHandleCreate(&h->cond, h->graph, 1, cudaGraphCondAssignDefault), "cudaGraphConditionalHandleCreate");
    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = h->cond;
    p.conditional.type = cudaGraphCondTypeWhile;
    p.conditional.size = 1;
    RL_TRY(cudaGraphAddNode(&h->node, h->graph, deps, ndeps, &p), "cudaGraphAddNode(WHILE)");
    RL_TRY(cudaStreamEndCapture(st, &g), "cudaStreamEndCapture");
    RL_TRY(cudaStreamBeginCaptureToGraph(st, p.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal),
           "cudaStreamBeginCaptureToGraph(body)");
    return B2_OK;
}

int b2_refine_loop_end(b2_refine_loop* h, const b2_inertia_source* src, int64_t expect_pos, int64_t expect_neg, int32_t max_iter,
                       double tol, void* stream) {
    cudaStream_t st = as_stream(stream);
    if (!h || !h->node || !src || !src->counters_d || src->fail < 0 || src->neg[0] < 0 || src->zero[0] < 0) {
        if (h && h->node) abort_build(h, st);
        set_error("b2_refine_loop_end: invalid argument (or no b2_refine_loop_begin before it)");
        return B2_ERR_INVALID;
    }
    RL_TRY(launch_refine_test(st, h->cond, h->norms, *src, expect_pos, expect_neg, max_iter, tol, h->rec.p, h->rec_h), "k_refine_test");
    cudaGraph_t g = nullptr;
    RL_TRY(cudaStreamEndCapture(st, &g), "cudaStreamEndCapture(body)");
    RL_TRY(cudaGraphInstantiate(&h->exec, h->graph, 0), "cudaGraphInstantiate");
    return B2_OK;
}

int b2_refine_loop_launch(b2_refine_loop* h, void* stream) {
    if (!h || !h->exec) { set_error("b2_refine_loop_launch: no graph built"); return B2_ERR_INVALID; }
    B2_CUDA(cudaGraphLaunch(h->exec, as_stream(stream)));
    h->stream = as_stream(stream);
    h->launched += 1;
    return B2_OK;
}

int b2_refine_loop_wait(b2_refine_loop* h) {
    if (!h || !h->launched) { set_error("b2_refine_loop_wait: nothing launched"); return B2_ERR_INVALID; }
    const volatile int64_t* seq = &h->rec_h->seq;
    // the last test kernel's write reaches host memory before the graph's completion does: poll it, and the stream so that a
    // failed launch is reported rather than waited for
    while (*seq != h->launched) {
        const cudaError_t e = cudaStreamQuery(h->stream);
        if (e == cudaSuccess) {
            if (*seq == h->launched) break;
            set_error("b2_refine_loop_wait: the graph finished without its record");
            return B2_ERR_CUDA;
        }
        if (e != cudaErrorNotReady) return cuda_fail(e, "b2_refine_loop_wait", __FILE__, __LINE__);
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return B2_OK;
}

int b2_refine_loop_record(b2_refine_loop* h, b2_refine_record* out) {
    if (!h || !out) { set_error("b2_refine_loop_record: invalid argument"); return B2_ERR_INVALID; }
    *out = *h->rec_h;
    return B2_OK;
}

}  // extern "C"
