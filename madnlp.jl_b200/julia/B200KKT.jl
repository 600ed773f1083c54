# B200KKT.jl -- the shim a MadNLP.jl maintainer adds to drive libb200kkt.so (include/b200kkt.h) from MadNLP's
# existing plugin surface.  NOT RUN in this repository's CI (no Julia in the build image); it is the reference-side
# binding INTEGRATION.md describes, kept next to the library so that the C ABI and its consumer evolve together.
#
#   using MadNLP, MadNLPGPU, CUDA
#   include("B200KKT.jl"); using .B200KKT
#   madnlp(nlp; kkt_system = MadNLP.SparseCondensedKKTSystem, linear_solver = B200KKT.B200Solver,
#          equality_treatment = MadNLP.RelaxEquality, tol = 1e-4)
#
# Interface implemented (src/LinearSolvers/linearsolvers.jl:13-95; same list every plugin imports,
# lib/MadNLPHSL/src/MadNLPHSL.jl:3-32): constructor(csc; opt, logger), factorize!, solve_linear_system!, is_inertia,
# inertia, improve!, introduce, input_type, default_options, is_supported, is_async.
module B200KKT

import MadNLP
import MadNLP: AbstractLinearSolver, AbstractOptions, MadNLPLogger, SymbolicException, FactorizationException,
    SolveException, factorize!, solve_linear_system!, is_inertia, inertia, improve!, introduce, input_type,
    default_options, is_supported, is_async
using CUDA, CUDA.CUSPARSE
import Libdl
# (nothing here extends a method on types this module does not own without one of ITS types in the signature)

const libb200kkt = get(ENV, "B200KKT_LIB", "libb200kkt.so")

# mirror of `struct b2_options` (include/b200kkt.h)
Base.@kwdef mutable struct B200Options <: AbstractOptions
    b200_ordering::Int32 = 0            # B2_ORDER_METIS_ND
    b200_nemin::Int32 = 16
    b200_relax_zeros::Float64 = 0.25
    b200_pivot_eps::Float64 = 1e-13
    b200_use_cuda_graph::Int32 = 1
    b200_small_front_max::Int32 = 160
    b200_kkt_n_primal::Int32 = 0        # set by the KKT overloads below for SparseKKTSystem
    b200_fuse_max_fronts::Int32 = 8
    b200_dep_schedule::Int32 = 1
    b200_chain_merge_f::Int32 = 0
    b200_kkt_n_dual::Int32 = 0          # set by create_kkt_system(SparseUnreducedKKTSystem, ...) below
    b200_dense_pivoting::Int32 = 0      # B200DenseSolver only: 0 static (B2_DENSE_PIVOT_STATIC), 1 Bunch-Kaufman, as
                                        # lapack_algorithm = BUNCHKAUFMAN (B2_DENSE_PIVOT_BUNCH_KAUFMAN); B200Solver needs 0
    b200_sparse_pivoting::Int32 = 0     # B200Solver only: 0 static (B2_SPARSE_PIVOT_STATIC), 1 2x2 pivots on matched
                                        # primal-dual pairs (B2_SPARSE_PIVOT_PAIRS); B200DenseSolver needs 0
    b200_dense_algorithm::Int32 = 0     # B200DenseSolver only: 0 LDL' (B2_DENSE_ALG_LDLT), 1 LU with partial pivoting, as
                                        # lapack_algorithm = LU (B2_DENSE_ALG_LU, no inertia: InertiaAuto is InertiaFree);
                                        # B200Solver needs 0
end

struct CB2Options
    ordering::Int32; nemin::Int32; relax_zeros::Float64; pivot_eps::Float64
    use_cuda_graph::Int32; small_front_max::Int32; n_parts::Int32; part_rank::Int32
    kkt_n_primal::Int32; fuse_max_fronts::Int32; dep_schedule::Int32; chain_merge_f::Int32; kkt_n_dual::Int32; dense_pivoting::Int32
    sparse_pivoting::Int32; dense_algorithm::Int32
end
CB2Options(o::B200Options) = CB2Options(o.b200_ordering, o.b200_nemin, o.b200_relax_zeros, o.b200_pivot_eps,
    o.b200_use_cuda_graph, o.b200_small_front_max, 1, 0, o.b200_kkt_n_primal, o.b200_fuse_max_fronts, o.b200_dep_schedule, o.b200_chain_merge_f,
    o.b200_kkt_n_dual, o.b200_dense_pivoting, o.b200_sparse_pivoting, o.b200_dense_algorithm)

last_error() = unsafe_string(ccall((:b2_last_error, libb200kkt), Cstring, ()))
function check(rc::Cint, exc)
    rc == 0 && return
    rc == 3 && throw(SymbolicException())
    rc == 4 && throw(FactorizationException())
    rc == 5 && throw(SolveException())
    error("b200kkt error $rc: $(last_error())")
end

mutable struct B200Solver{T} <: AbstractLinearSolver{T}
    handle::Ptr{Cvoid}
    tril::CuSparseMatrixCSC{T,Int32}    # kept by reference: values are re-read on every factorize! (cudss.jl:154-158)
    opt::B200Options
    logger::MadNLPLogger
end

function B200Solver(csc::CuSparseMatrixCSC{Float64,Int32}; opt = B200Options(), logger = MadNLPLogger())
    n = size(csc, 1)
    colptr = Array(csc.colPtr) .- Int32(1)          # host, 0-based (analysis runs on the host, once)
    rowval = Array(csc.rowVal) .- Int32(1)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    copt = Ref(CB2Options(opt))
    rc = ccall((:b2_create, libb200kkt), Cint,
        (Int32, Int64, Ptr{Int32}, Ptr{Int32}, CuPtr{Float64}, Ptr{CB2Options}, Ptr{Int32}, Ptr{Ptr{Cvoid}}),
        n, length(rowval), colptr, rowval, pointer(csc.nzVal), copt, C_NULL, h)
    check(rc, SymbolicException)
    M = B200Solver{Float64}(h[], csc, opt, logger)
    finalizer(m -> ccall((:b2_destroy, libb200kkt), Cint, (Ptr{Cvoid},), m.handle), M)
    return M
end

stream_ptr() = Ptr{Cvoid}(UInt(CUDA.stream().handle))

function factorize!(M::B200Solver)
    check(ccall((:b2_factorize, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), M.handle, stream_ptr()), FactorizationException)
    return M
end

function solve_linear_system!(M::B200Solver{T}, x::CuVector{T}) where T
    check(ccall((:b2_solve, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, Int32, Ptr{Cvoid}), M.handle, pointer(x), 1, stream_ptr()), SolveException)
    return x
end

# the matrix method (src/LinearSolvers/linearsolvers.jl:102, CompactLBFGS's qn.H in src/IPM/factorization.jl:118): every column in
# one b2_solve, which walks the elimination tree once per 8 columns instead of once per column
function solve_linear_system!(M::B200Solver{T}, X::CuMatrix{T}) where T
    stride(X, 2) == size(X, 1) || throw(ArgumentError("solve_linear_system!: X needs contiguous columns (stride(X, 2) == size(X, 1))"))
    size(X, 2) == 0 && return X
    check(ccall((:b2_solve, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, Int32, Ptr{Cvoid}), M.handle, pointer(X), Int32(size(X, 2)), stream_ptr()),
          SolveException)
    return X
end

is_inertia(::B200Solver) = true
function inertia(M::B200Solver)
    p = Ref{Int64}(0); z = Ref{Int64}(0); n = Ref{Int64}(0)
    check(ccall((:b2_inertia, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Cvoid}),
        M.handle, p, z, n, stream_ptr()), FactorizationException)
    return (Int(p[]), Int(z[]), Int(n[]))       # (num_pos, num_zero, num_neg): the order src/IPM/solver.jl:626 destructures
end

function improve!(M::B200Solver)
    ch = Ref{Int32}(0)
    ccall((:b2_improve, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Int32}), M.handle, ch)
    return ch[] != 0
end

introduce(::B200Solver) = "b200kkt (sm_90a multifrontal LDL')"
input_type(::Type{<:B200Solver}) = :csc
default_options(::Type{<:B200Solver}) = B200Options()
is_supported(::Type{<:B200Solver}, ::Type{Float64}) = true
is_supported(::Type{<:B200Solver}, ::Type{Float32}) = false
is_async(::B200Solver) = true

# ---------------------------------------------------------------------------------------------------------------------
# KKT-level overloads.  Dispatch is on OUR solver type in the `LS` parameter of the stock KKT structs
#   SparseCondensedKKTSystem{T,VT,MT,QN,LS,...} (src/KKT/Sparse/condensed.jl:7)   with VT <: CuVector AND LS <: B200Solver
#   DenseCondensedKKTSystem{T,VT,MT,QN,LS,VI}   (src/KKT/Dense/condensed.jl:10)   with VT <: CuVector AND LS <: B200DenseSolver
#   DenseKKTSystem{T,VT,MT,QN,LS,VI}            (src/KKT/Dense/augmented.jl:10)   with VT <: CuVector AND LS <: B200DenseSolver
#   SparseUnreducedKKTSystem{T,VT,MT,QN,LS,...} (src/KKT/Sparse/unreduced.jl:8)   with VT <: CuVector AND LS <: B200Solver
# -- strictly more specific than MadNLPGPU's `VT <: AbstractGPUVector` methods (lib/MadNLPGPU/src/KKT/gpu_sparse.jl:308-382,
# gpu_dense.jl:86-138), so loading both packages is neither ambiguous nor type piracy (a type this module owns is in every
# signature).  The native plans live in the solver object (which this module owns), built lazily from the kkt's own maps at
# the first call: MadNLP's `ext` slot (get_sparse_condensed_ext, gpu_sparse.jl:100-130) keeps whatever MadNLPGPU put there.
# ---------------------------------------------------------------------------------------------------------------------
mutable struct CondensedPlans
    cond::Ptr{Cvoid}        # b2_condensed_plan   (pattern of tril(H) U diag U tril(Jt Jt') + the dptr/hptr/jptr maps)
    hess_plan::Ptr{Cvoid}   # b2_transfer_plan    hess_raw (COO) -> hess_com (CSC)
    jt_plan::Ptr{Cvoid}     # b2_transfer_plan    jt_coo         -> jt_csc
    hess_spmv::Ptr{Cvoid}   # b2_spmv_plan of hess_com
    jt_spmv::Ptr{Cvoid}     # b2_spmv_plan of jt_csc
    bounds::Ptr{Cvoid}      # b2_bounds (ind_lb / ind_ub and their inverse maps)
end

const _plans = IdDict{Any,CondensedPlans}()     # solver handle -> plans (freed with the solver)

const B200CondensedKKT{T} = MadNLP.SparseCondensedKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200Solver}

function plans(kkt::B200CondensedKKT{T}) where T
    get!(_plans, kkt.linear_solver) do
        n = size(kkt.hess_com, 1); m = size(kkt.jt_csc, 2)
        h0(v) = Array(v) .- one(eltype(v))                                   # host, 0-based
        hcp, hrv = h0(kkt.hess_com.colPtr), h0(kkt.hess_com.rowVal)
        jcp, jrv = h0(kkt.jt_csc.colPtr), h0(kkt.jt_csc.rowVal)
        cond = Ref{Ptr{Cvoid}}(C_NULL); nnz_aug = Ref{Int64}(0)
        check(ccall((:b2_condensed_symbolic, libb200kkt), Cint,
            (Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Ptr{Cvoid}}, Ptr{Int64}),
            n, m, hcp, hrv, jcp, jrv, cond, nnz_aug), SymbolicException)
        @assert nnz_aug[] == length(MadNLP.nzval(kkt.aug_com))               # same pattern as build_condensed_aug_symbolic
        tplan(map_d) = begin
            mp = Array(map_d) .- 1; h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2_transfer_plan_create, libb200kkt), Cint, (Int64, Int64, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
                length(mp), maximum(mp; init = -1) + 1, mp, h), SymbolicException); h[]
        end
        splan(nr, nc, cp, rv) = begin
            h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2_spmv_plan_create, libb200kkt), Cint, (Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Ptr{Cvoid}}), nr, nc, cp, rv, h), SymbolicException); h[]
        end
        lb = Array(kkt.ind_lb) .- 1; ub = Array(kkt.ind_ub) .- 1; b = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b2_bounds_create, libb200kkt), Cint, (Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
            length(kkt.pr_diag), length(lb), length(ub), lb, ub, b), SymbolicException)
        CondensedPlans(cond[], tplan(kkt.hess_csc_map), tplan(kkt.jt_csc_map), splan(n, n, hcp, hrv), splan(n, m, jcp, jrv), b[])
    end
end

function MadNLP.build_kkt!(kkt::B200CondensedKKT{T}) where T
    p = plans(kkt)
    check(ccall((:b2_condensed_assemble, libb200kkt), Cint,
        (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.cond, pointer(MadNLP.nzval(kkt.aug_com)), pointer(kkt.pr_diag), pointer(kkt.du_diag),
        pointer(MadNLP.nzval(kkt.hess_com)), pointer(MadNLP.nzval(kkt.jt_csc)), pointer(kkt.diag_buffer), stream_ptr()), FactorizationException)
end

function MadNLP.compress_hessian!(kkt::B200CondensedKKT{T}) where T
    check(ccall((:b2_transfer, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        plans(kkt).hess_plan, pointer(MadNLP.nzval(kkt.hess_com)), pointer(kkt.hess_raw.V), stream_ptr()), FactorizationException)
end

function MadNLP.compress_jacobian!(kkt::B200CondensedKKT{T}) where T
    check(ccall((:b2_transfer, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        plans(kkt).jt_plan, pointer(MadNLP.nzval(kkt.jt_csc)), pointer(kkt.jt_coo.V), stream_ptr()), FactorizationException)
end

# solve_kkt! (src/IPM/factorization.jl:143-167): pre -> b2_solve -> post
function MadNLP.solve_kkt!(kkt::B200CondensedKKT{T}, w::MadNLP.AbstractKKTVector) where T
    p = plans(kkt); n = size(kkt.hess_com, 1); m = size(kkt.jt_csc, 2); wv = MadNLP.full(w)
    check(ccall((:b2_condensed_solve_pre, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.bounds, p.jt_spmv, n, m, pointer(MadNLP.nzval(kkt.jt_csc)), pointer(kkt.pr_diag), pointer(kkt.diag_buffer),
        pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(kkt.buffer), pointer(wv), stream_ptr()), SolveException)
    solve_linear_system!(kkt.linear_solver, view(wv, 1:n))
    check(ccall((:b2_condensed_solve_post, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.bounds, p.jt_spmv, n, m, pointer(MadNLP.nzval(kkt.jt_csc)), pointer(kkt.pr_diag), pointer(kkt.diag_buffer),
        pointer(kkt.l_lower), pointer(kkt.u_lower), pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(kkt.buffer), pointer(wv), stream_ptr()), SolveException)
    return w
end
solve_linear_system!(M::B200Solver{T}, x::SubArray{T,1,<:CuVector{T}}) where T =
    (check(ccall((:b2_solve, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, Int32, Ptr{Cvoid}), M.handle, pointer(x), 1, stream_ptr()), SolveException); x)

# mul!(w, kkt, x, alpha, beta) (src/IPM/factorization.jl:303-324) incl. _kktmul!: ONE kernel instead of 3 SpMV + broadcasts
function MadNLP.mul!(w::MadNLP.AbstractKKTVector{T}, kkt::B200CondensedKKT{T}, x::MadNLP.AbstractKKTVector, alpha = one(T), beta = zero(T)) where T
    p = plans(kkt); n = size(kkt.hess_com, 1); m = size(kkt.jt_csc, 2)
    check(ccall((:b2_condensed_kkt_mul, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T},
         Cdouble, Cdouble, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.bounds, p.hess_spmv, p.jt_spmv, n, m, pointer(MadNLP.nzval(kkt.hess_com)), pointer(MadNLP.nzval(kkt.jt_csc)),
        pointer(kkt.reg), pointer(kkt.du_diag), pointer(kkt.l_lower), pointer(kkt.u_lower), pointer(kkt.l_diag), pointer(kkt.u_diag),
        alpha, beta, pointer(MadNLP.full(x)), pointer(MadNLP.full(w)), stream_ptr()), SolveException)
    return w
end

# ---------------------------------------------------------------------------------------------------------------------
# Dense back-end: role of LapackCUDASolver (lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cusolver.jl:150-187), plus inertia
# ---------------------------------------------------------------------------------------------------------------------
mutable struct B200DenseSolver{T} <: AbstractLinearSolver{T}
    handle::Ptr{Cvoid}
    A::CuMatrix{T}                      # kept by reference (src/LinearSolvers/lapack.jl:40); lower triangle is read
    kkt_plan::Ptr{Cvoid}                # b2d_kkt (index sets of the DenseCondensed wrappers), created on first use
    bounds::Ptr{Cvoid}
    opt::B200Options
    logger::MadNLPLogger
end
function B200DenseSolver(A::CuMatrix{Float64}; opt = B200Options(), logger = MadNLPLogger())
    N = size(A, 1); h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b2d_create, libb200kkt), Cint, (Int32, Int32, CuPtr{Float64}, Ptr{CB2Options}, Ptr{Ptr{Cvoid}}),
        N, stride(A, 2), pointer(A), Ref(CB2Options(opt)), h), SymbolicException)
    M = B200DenseSolver{Float64}(h[], A, C_NULL, C_NULL, opt, logger)
    finalizer(m -> ccall((:b2d_destroy, libb200kkt), Cint, (Ptr{Cvoid},), m.handle), M)
    return M
end
factorize!(M::B200DenseSolver) = (check(ccall((:b2d_factorize, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), M.handle, stream_ptr()), FactorizationException); M)
solve_linear_system!(M::B200DenseSolver{T}, x::CuVector{T}) where T =
    (check(ccall((:b2d_solve, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, Int32, Ptr{Cvoid}), M.handle, pointer(x), 1, stream_ptr()), SolveException); x)
is_inertia(M::B200DenseSolver) = M.opt.b200_dense_algorithm == 0     # LU reports no inertia (lapack_common.jl:91)
function inertia(M::B200DenseSolver)
    M.opt.b200_dense_algorithm == 0 || error("B200DenseSolver: an LU factorisation (b200_dense_algorithm = 1) reports no inertia")
    p = Ref{Int64}(0); z = Ref{Int64}(0); n = Ref{Int64}(0)
    check(ccall((:b2d_inertia, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Cvoid}), M.handle, p, z, n, stream_ptr()), FactorizationException)
    return (Int(p[]), Int(z[]), Int(n[]))
end
improve!(::B200DenseSolver) = false
introduce(M::B200DenseSolver) = M.opt.b200_dense_algorithm == 1 ? "b200kkt dense LU (partial pivoting)" :
    M.opt.b200_dense_pivoting == 1 ? "b200kkt dense LDL' (Bunch-Kaufman pivoting)" : "b200kkt dense LDL' (DMMA)"
input_type(::Type{<:B200DenseSolver}) = :dense
default_options(::Type{<:B200DenseSolver}) = B200Options()
is_supported(::Type{<:B200DenseSolver}, ::Type{Float64}) = true
is_async(::B200DenseSolver) = true

const B200DenseKKT{T} = MadNLP.DenseCondensedKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200DenseSolver}
const B200DenseAugKKT{T} = MadNLP.DenseKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200DenseSolver}
const B200AnyDenseKKT{T} = Union{B200DenseKKT{T},B200DenseAugKKT{T}}     # AbstractDenseKKTSystem with our solver

function dense_plans(kkt::B200AnyDenseKKT{T}) where T
    M = kkt.linear_solver
    if M.kkt_plan == C_NULL
        n = size(kkt.hess, 1); m = size(kkt.jac, 1); ii = Array(kkt.ind_ineq) .- 1; h = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b2d_kkt_create, libb200kkt), Cint, (Int32, Int32, Int32, Ptr{Int64}, Ptr{Ptr{Cvoid}}), n, m, length(ii), ii, h), SymbolicException)
        M.kkt_plan = h[]
        lb = Array(kkt.ind_lb) .- 1; ub = Array(kkt.ind_ub) .- 1; b = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b2_bounds_create, libb200kkt), Cint, (Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
            length(kkt.pr_diag), length(lb), length(ub), lb, ub, b), SymbolicException)
        M.bounds = b[]
    end
    return M.kkt_plan, M.bounds
end

# build_kkt!(::DenseCondensedKKTSystem) (src/KKT/Dense/condensed.jl:157-186): one fused DMMA SYRK + epilogue
function MadNLP.build_kkt!(kkt::B200DenseKKT{T}) where T
    n = size(kkt.hess, 1); m = size(kkt.jac, 1)
    check(ccall((:b2d_condensed_assemble, libb200kkt), Cint,
        (Int32, Int32, Int32, Int32, CuPtr{Int64}, CuPtr{Int64}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        n, m, kkt.n_ineq, kkt.n_eq, pointer(kkt.etc[:b200_ind_ineq0]), pointer(kkt.etc[:b200_ind_eq0]), pointer(kkt.hess), pointer(kkt.jac),
        pointer(kkt.pr_diag), pointer(kkt.du_diag), pointer(kkt.diag_buffer), pointer(kkt.aug_com), stream_ptr()), FactorizationException)
end
# (kkt.etc is the Dict{Symbol,Any} scratch slot of the struct, Dense/condensed.jl:49: the 0-based device copies of ind_ineq / ind_eq
#  are stored there once:  kkt.etc[:b200_ind_ineq0] = CuVector(kkt.ind_ineq .- 1) ...)

# solve_kkt!(::DenseCondensedKKTSystem) (src/IPM/factorization.jl:190-229)
function MadNLP.solve_kkt!(kkt::B200DenseKKT{T}, w::MadNLP.AbstractKKTVector) where T
    kp, bp = dense_plans(kkt); wv = MadNLP.full(w)
    check(ccall((:b2d_kkt_solve_pre, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        kp, bp, pointer(kkt.jac), pointer(kkt.pr_diag), pointer(kkt.diag_buffer), pointer(kkt.l_diag), pointer(kkt.u_diag),
        pointer(kkt.buffer), pointer(kkt.pd_buffer), pointer(wv), stream_ptr()), SolveException)
    solve_linear_system!(kkt.linear_solver, kkt.pd_buffer)
    check(ccall((:b2d_kkt_solve_post, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        kp, bp, pointer(kkt.jac), pointer(kkt.pr_diag), pointer(kkt.diag_buffer), pointer(kkt.l_lower), pointer(kkt.u_lower),
        pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(kkt.buffer), pointer(kkt.pd_buffer), pointer(wv), stream_ptr()), SolveException)
    return w
end

# mul!(w, ::AbstractDenseKKTSystem, x, alpha, beta) (src/IPM/factorization.jl:303-324): the same formula for both dense KKT types
function MadNLP.mul!(w::MadNLP.AbstractKKTVector{T}, kkt::B200AnyDenseKKT{T}, x::MadNLP.AbstractKKTVector, alpha = one(T), beta = zero(T)) where T
    kp, bp = dense_plans(kkt)
    check(ccall((:b2d_kkt_mul, libb200kkt), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        kp, bp, pointer(kkt.hess), pointer(kkt.jac), pointer(kkt.reg), pointer(kkt.du_diag), pointer(kkt.l_lower), pointer(kkt.u_lower),
        pointer(kkt.l_diag), pointer(kkt.u_diag), alpha, beta, pointer(MadNLP.full(x)), pointer(MadNLP.full(w)), stream_ptr()), SolveException)
    return w
end

# ---------------------------------------------------------------------------------------------------------------------
# DenseKKTSystem (src/KKT/Dense/augmented.jl): the augmented matrix of order n + ns + m, assembled by one kernel and factorised
# whole by B200DenseSolver.  kkt.etc (augmented.jl:39) holds the 0-based device copy of ind_ineq, made on first use.
# ---------------------------------------------------------------------------------------------------------------------
ind_ineq0(kkt::B200DenseAugKKT) = get!(() -> CuVector{Int64}(Array(kkt.ind_ineq) .- 1), kkt.etc, :b200_ind_ineq0)

# build_kkt! (augmented.jl:116-156): every element of the lower triangle written, so the one-time fill! is not relied on
function MadNLP.build_kkt!(kkt::B200DenseAugKKT{T}) where T
    n = size(kkt.hess, 1); m = size(kkt.jac, 1)
    check(ccall((:b2d_aug_assemble, libb200kkt), Cint,
        (Int32, Int32, Int32, CuPtr{Int64}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        n, m, length(kkt.ind_ineq), pointer(ind_ineq0(kkt)), pointer(kkt.hess), pointer(kkt.jac), pointer(kkt.pr_diag),
        pointer(kkt.du_diag), pointer(kkt.diag_hess), pointer(kkt.aug_com), stream_ptr()), FactorizationException)
end

# compress_hessian! (augmented.jl:158-161) = diag!(diag_hess, hess)
function MadNLP.compress_hessian!(kkt::B200DenseAugKKT{T}) where T
    check(ccall((:b2d_copy_diag, libb200kkt), Cint, (Int32, Int32, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        size(kkt.hess, 1), stride(kkt.hess, 2), pointer(kkt.hess), pointer(kkt.diag_hess), stream_ptr()), FactorizationException)
end

# solve_kkt!(::AbstractReducedKKTSystem) (src/IPM/factorization.jl:41-46): reduce_rhs! -> solve on primal_dual(w) -> finish_aug_solve!;
# primal_dual(w) is the leading n + ns + m entries of full(w)
function MadNLP.solve_kkt!(kkt::B200DenseAugKKT{T}, w::MadNLP.AbstractKKTVector) where T
    _, bp = dense_plans(kkt); wv = MadNLP.full(w); m = size(kkt.jac, 1)
    check(ccall((:b2_reduce_rhs, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        bp, m, pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(wv), stream_ptr()), SolveException)
    check(ccall((:b2d_solve, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, Int32, Ptr{Cvoid}),
        kkt.linear_solver.handle, pointer(wv), 1, stream_ptr()), SolveException)
    check(ccall((:b2_finish_aug_solve, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        bp, m, pointer(kkt.l_lower), pointer(kkt.u_lower), pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(wv), stream_ptr()), SolveException)
    return w
end

# mul!(y, ::DenseKKTSystem, x) (augmented.jl:98-100) = _symv!('L', 1, aug_com, x, 0, y)
function MadNLP.mul!(y::CuVector{T}, kkt::B200DenseAugKKT{T}, x::CuVector{T}) where T
    N = size(kkt.aug_com, 1)
    check(ccall((:b2d_symv_lower, libb200kkt), Cint, (Int32, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}),
        N, stride(kkt.aug_com, 2), pointer(kkt.aug_com), pointer(x), pointer(y), one(T), zero(T), stream_ptr()), SolveException)
    return y
end

# ---------------------------------------------------------------------------------------------------------------------
# SparseUnreducedKKTSystem (src/KKT/Sparse/unreduced.jl) with B200Solver.  The analysis must know which rows are bound duals
# (b2_options.kkt_n_dual), so create_kkt_system fills kkt_n_primal = n_tot and kkt_n_dual = m when they were left at 0 and then
# runs the stock constructor.  Plans (transfer maps, SpMV plans, bounds) live beside the solver, as for the condensed type.
# ---------------------------------------------------------------------------------------------------------------------
const B200UnreducedKKT{T} = MadNLP.SparseUnreducedKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200Solver}
const B200ScaledKKT{T} = MadNLP.ScaledSparseKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200Solver}

function MadNLP.create_kkt_system(::Type{MadNLP.SparseUnreducedKKTSystem}, cb::MadNLP.SparseCallback, linear_solver::Type{<:B200Solver};
                                  opt_linear_solver = default_options(linear_solver), kwargs...)
    n_tot = cb.nvar + length(cb.ind_ineq)
    opt_linear_solver.b200_kkt_n_primal == 0 && (opt_linear_solver.b200_kkt_n_primal = n_tot)
    opt_linear_solver.b200_kkt_n_dual == 0 && (opt_linear_solver.b200_kkt_n_dual = cb.ncon)
    return invoke(MadNLP.create_kkt_system, Tuple{Type{MadNLP.SparseUnreducedKKTSystem},MadNLP.SparseCallback,Type},
                  MadNLP.SparseUnreducedKKTSystem, cb, linear_solver; opt_linear_solver = opt_linear_solver, kwargs...)
end

mutable struct UnreducedPlans
    aug_plan::Ptr{Cvoid}; hess_plan::Ptr{Cvoid}; jac_plan::Ptr{Cvoid}   # b2_transfer_plan: aug_raw / hess_raw / jac_raw -> CSC
    hess_spmv::Ptr{Cvoid}; jac_spmv::Ptr{Cvoid}                         # b2_spmv_plan of hess_com (n_tot x n_tot) / jac_com (m x n_tot)
    bounds::Ptr{Cvoid}
end
const _uplans = IdDict{Any,UnreducedPlans}()

function uplans(kkt::Union{B200UnreducedKKT{T},B200ScaledKKT{T}}) where T   # (K2.5: the same plans)
    get!(_uplans, kkt.linear_solver) do
        h0(v) = Array(v) .- one(eltype(v))
        tplan(map_d, nnz_csc) = begin
            mp = Array(map_d) .- 1; h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2_transfer_plan_create, libb200kkt), Cint, (Int64, Int64, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
                length(mp), nnz_csc, mp, h), SymbolicException); h[]
        end
        splan(A) = begin
            h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2_spmv_plan_create, libb200kkt), Cint, (Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Ptr{Cvoid}}),
                size(A, 1), size(A, 2), h0(A.colPtr), h0(A.rowVal), h), SymbolicException); h[]
        end
        lb = Array(kkt.ind_lb) .- 1; ub = Array(kkt.ind_ub) .- 1; b = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b2_bounds_create, libb200kkt), Cint, (Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
            length(kkt.pr_diag), length(lb), length(ub), lb, ub, b), SymbolicException)
        nz(A) = length(MadNLP.nzval(A))
        UnreducedPlans(tplan(kkt.aug_csc_map, nz(kkt.aug_com)), tplan(kkt.hess_csc_map, nz(kkt.hess_com)),
                       tplan(kkt.jac_csc_map, nz(kkt.jac_com)), splan(kkt.hess_com), splan(kkt.jac_com), b[])
    end
end

_transfer(plan, dst, src) = check(ccall((:b2_transfer, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Ptr{Cvoid}),
    plan, pointer(dst), pointer(src), stream_ptr()), FactorizationException)

# build_kkt! (unreduced.jl:178-180) = transfer!(aug_com, aug_raw, aug_csc_map)
MadNLP.build_kkt!(kkt::B200UnreducedKKT) = _transfer(uplans(kkt).aug_plan, MadNLP.nzval(kkt.aug_com), kkt.aug_raw.V)
MadNLP.compress_hessian!(kkt::B200UnreducedKKT) = _transfer(uplans(kkt).hess_plan, MadNLP.nzval(kkt.hess_com), kkt.hess_raw.V)
# compress_jacobian! (Sparse/utils.jl:36-40): slack entries -1, then transfer!
function MadNLP.compress_jacobian!(kkt::B200UnreducedKKT{T}) where T
    ns = length(kkt.ind_ineq)
    ns > 0 && check(ccall((:b2_fill, libb200kkt), Cint, (Int64, Cdouble, CuPtr{T}, Ptr{Cvoid}),
        ns, -one(T), pointer(kkt.jac, length(kkt.jac) - ns + 1), stream_ptr()), FactorizationException)
    _transfer(uplans(kkt).jac_plan, MadNLP.nzval(kkt.jac_com), kkt.jac_raw.V)
end

# _set_aug_diagonal!(::AbstractUnreducedKKTSystem) (src/IPM/kernels.jl:29-34): one launch
function MadNLP._set_aug_diagonal!(kkt::B200UnreducedKKT{T}) where T
    check(ccall((:b2_set_aug_diagonal_unreduced, libb200kkt), Cint,
        (Int64, Int64, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        length(kkt.pr_diag), length(kkt.l_lower), length(kkt.u_lower), pointer(kkt.reg), pointer(kkt.l_lower), pointer(kkt.u_lower),
        pointer(kkt.pr_diag), pointer(kkt.l_lower_aug), pointer(kkt.u_lower_aug), stream_ptr()), FactorizationException)
    return
end

# solve_kkt! (src/IPM/factorization.jl:29-39): scale the bound-dual blocks -> b2_solve on full(w) -> scale back
function MadNLP.solve_kkt!(kkt::B200UnreducedKKT{T}, w::MadNLP.AbstractKKTVector) where T
    wv = MadNLP.full(w)
    args = (length(kkt.pr_diag), length(kkt.du_diag), length(kkt.l_lower), length(kkt.u_lower))
    sig = (Int64, Int64, Int64, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid})
    check(ccall((:b2_unreduced_solve_pre, libb200kkt), Cint, sig, args..., pointer(kkt.l_lower_aug), pointer(kkt.u_lower_aug),
        pointer(wv), stream_ptr()), SolveException)
    solve_linear_system!(kkt.linear_solver, wv)
    check(ccall((:b2_unreduced_solve_post, libb200kkt), Cint, sig, args..., pointer(kkt.l_lower_aug), pointer(kkt.u_lower_aug),
        pointer(wv), stream_ptr()), SolveException)
    return w
end

# mul! (src/IPM/factorization.jl:231-237): symmetric Hessian, J' y, J x, then _kktmul!
function MadNLP.mul!(w::MadNLP.AbstractKKTVector{T}, kkt::B200UnreducedKKT{T}, x::MadNLP.AbstractKKTVector, alpha = one(T), beta = zero(T)) where T
    p = uplans(kkt); st = stream_ptr(); xv = MadNLP.full(x); wv = MadNLP.full(w)
    spmv(name, plan, nz, xp, yp, b) = check(ccall((name, libb200kkt), Cint,
        (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}), plan, pointer(nz), xp, yp, alpha, b, st), SolveException)
    spmv(:b2_spmv_symlower, p.hess_spmv, MadNLP.nzval(kkt.hess_com), pointer(xv), pointer(wv), beta)
    spmv(:b2_spmv_t, p.jac_spmv, MadNLP.nzval(kkt.jac_com), pointer(MadNLP.dual(x)), pointer(wv), one(T))
    spmv(:b2_spmv_n, p.jac_spmv, MadNLP.nzval(kkt.jac_com), pointer(xv), pointer(MadNLP.dual(w)), beta)
    check(ccall((:b2_kktmul, libb200kkt), Cint,
        (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.bounds, length(kkt.du_diag), pointer(kkt.reg), pointer(kkt.du_diag), pointer(kkt.l_lower), pointer(kkt.u_lower),
        pointer(kkt.l_diag), pointer(kkt.u_diag), alpha, beta, pointer(xv), pointer(wv), st), SolveException)
    return w
end

# jtprod! (Sparse/utils.jl:28-30): y = jac_com' x
function MadNLP.jtprod!(y::CuVector{T}, kkt::B200UnreducedKKT{T}, x::CuVector{T}) where T
    check(ccall((:b2_spmv_t, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}),
        uplans(kkt).jac_spmv, pointer(MadNLP.nzval(kkt.jac_com)), pointer(x), pointer(y), one(T), zero(T), stream_ptr()), SolveException)
    return y
end

# ---------------------------------------------------------------------------------------------------------------------
# ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl) with B200Solver.  The layout is SparseKKTSystem's, so
# create_kkt_system fills kkt_n_primal = n_tot as for K2 and runs the stock constructor; the plans are the unreduced type's (uplans)
# plus aug_com's pattern on the device, which b2_scaled_transfer reads.  build_kkt! scales V's sources on their way into aug_com: the
# constructor's scaled_aug_raw is never written.  l_diag = x - xl and u_diag = xu - x (positive), as the reference has them.
# ---------------------------------------------------------------------------------------------------------------------
function MadNLP.create_kkt_system(::Type{MadNLP.ScaledSparseKKTSystem}, cb::MadNLP.SparseCallback, linear_solver::Type{<:B200Solver};
                                  opt_linear_solver = default_options(linear_solver), kwargs...)
    opt_linear_solver.b200_kkt_n_primal == 0 && (opt_linear_solver.b200_kkt_n_primal = cb.nvar + length(cb.ind_ineq))
    return invoke(MadNLP.create_kkt_system, Tuple{Type{MadNLP.ScaledSparseKKTSystem},MadNLP.SparseCallback,Type},
                  MadNLP.ScaledSparseKKTSystem, cb, linear_solver; opt_linear_solver = opt_linear_solver, kwargs...)
end

const _scaled_pattern = IdDict{Any,Tuple{CuVector{Int32},CuVector{Int32}}}()
scaled_pattern(kkt::B200ScaledKKT) = get!(_scaled_pattern, kkt.linear_solver) do
    (CuVector{Int32}(Array(kkt.aug_com.colPtr) .- 1), CuVector{Int32}(Array(kkt.aug_com.rowVal) .- 1))
end

# build_kkt! (scaled_augmented.jl:209-236): one pass over aug_com's slots, each COO source scaled before the slot's sum
function MadNLP.build_kkt!(kkt::B200ScaledKKT{T}) where T
    cp, rv = scaled_pattern(kkt)
    check(ccall((:b2_scaled_transfer, libb200kkt), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Int32}, CuPtr{Int32}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        uplans(kkt).aug_plan, size(kkt.aug_com, 1), length(kkt.pr_diag), pointer(cp), pointer(rv), pointer(kkt.scaling_factor),
        pointer(MadNLP.nzval(kkt.aug_com)), pointer(kkt.aug_raw.V), stream_ptr()), FactorizationException)
end
MadNLP.compress_hessian!(kkt::B200ScaledKKT) = _transfer(uplans(kkt).hess_plan, MadNLP.nzval(kkt.hess_com), kkt.hess_raw.V)
function MadNLP.compress_jacobian!(kkt::B200ScaledKKT{T}) where T
    ns = length(kkt.ind_ineq)
    ns > 0 && check(ccall((:b2_fill, libb200kkt), Cint, (Int64, Cdouble, CuPtr{T}, Ptr{Cvoid}),
        ns, -one(T), pointer(kkt.jac, length(kkt.jac) - ns + 1), stream_ptr()), FactorizationException)
    _transfer(uplans(kkt).jac_plan, MadNLP.nzval(kkt.jac_com), kkt.jac_raw.V)
end

# _set_aug_diagonal! (src/IPM/kernels.jl:47-68): pr_diag and scaling_factor in one launch
function MadNLP._set_aug_diagonal!(kkt::B200ScaledKKT{T}) where T
    check(ccall((:b2_scaled_set_aug_diagonal, libb200kkt), Cint, (Ptr{Cvoid}, ntuple(_ -> CuPtr{T}, 7)..., Ptr{Cvoid}),
        uplans(kkt).bounds, pointer(kkt.reg), pointer(kkt.l_lower), pointer(kkt.l_diag), pointer(kkt.u_lower), pointer(kkt.u_diag),
        pointer(kkt.pr_diag), pointer(kkt.scaling_factor), stream_ptr()), FactorizationException)
    return
end

# set_aug_diagonal! (src/IPM/kernels.jl:36-45): reg, du_diag, l_lower = zl_r, u_lower = zu_r, l_diag = x_lr - xl_r, u_diag = xu_r - x_ur
# in one launch, then _set_aug_diagonal!
function MadNLP.set_aug_diagonal!(kkt::B200ScaledKKT{T}, solver::MadNLP.AbstractMadNLPSolver{T}) where T
    o = MadNLP.get_opt(solver)
    v(f) = pointer(MadNLP.full(f(solver)))
    check(ccall((:b2_set_aug_diagonal_iterate_scaled, libb200kkt), Cint, (Ptr{Cvoid}, Int64, Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 11)..., Ptr{Cvoid}),
        uplans(kkt).bounds, length(kkt.du_diag), o.default_primal_regularization, o.default_dual_regularization, v(MadNLP.get_x),
        v(MadNLP.get_xl), v(MadNLP.get_xu), v(MadNLP.get_zl), v(MadNLP.get_zu), pointer(kkt.reg), pointer(kkt.du_diag),
        pointer(kkt.l_lower), pointer(kkt.u_lower), pointer(kkt.l_diag), pointer(kkt.u_diag), stream_ptr()), FactorizationException)
    MadNLP._set_aug_diagonal!(kkt)
end

# regularize_diagonal! (scaled_augmented.jl:238-242): reg += primal; pr_diag += primal s^2; du_diag -= dual
function MadNLP.regularize_diagonal!(kkt::B200ScaledKKT{T}, primal, dual) where T
    check(ccall((:b2_scaled_regularize_diagonal, libb200kkt), Cint, (Int64, Int64, Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 4)..., Ptr{Cvoid}),
        length(kkt.pr_diag), length(kkt.du_diag), primal, dual, pointer(kkt.scaling_factor), pointer(kkt.reg), pointer(kkt.pr_diag),
        pointer(kkt.du_diag), stream_ptr()), FactorizationException)
end

# solve_kkt! (src/IPM/factorization.jl:48-74): one launch on each side of b2_solve on primal_dual(w)
function MadNLP.solve_kkt!(kkt::B200ScaledKKT{T}, w::MadNLP.AbstractKKTVector) where T
    wv = MadNLP.full(w); b = uplans(kkt).bounds; m = length(kkt.du_diag)
    check(ccall((:b2_scaled_solve_pre, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        b, m, pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(kkt.scaling_factor), pointer(wv), stream_ptr()), SolveException)
    solve_linear_system!(kkt.linear_solver, MadNLP.primal_dual(w))
    check(ccall((:b2_scaled_solve_post, libb200kkt), Cint, (Ptr{Cvoid}, Int64, ntuple(_ -> CuPtr{T}, 6)..., Ptr{Cvoid}),
        b, m, pointer(kkt.l_lower), pointer(kkt.u_lower), pointer(kkt.l_diag), pointer(kkt.u_diag), pointer(kkt.scaling_factor),
        pointer(wv), stream_ptr()), SolveException)
    return w
end

# mul! (src/IPM/factorization.jl:239-251): the three SpMVs, then the diagonal and bound part with K2.5's signs
function MadNLP.mul!(w::MadNLP.AbstractKKTVector{T}, kkt::B200ScaledKKT{T}, x::MadNLP.AbstractKKTVector, alpha = one(T), beta = zero(T)) where T
    p = uplans(kkt); st = stream_ptr(); xv = MadNLP.full(x); wv = MadNLP.full(w)
    spmv(name, plan, nz, xp, yp, b) = check(ccall((name, libb200kkt), Cint,
        (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}), plan, pointer(nz), xp, yp, alpha, b, st), SolveException)
    spmv(:b2_spmv_symlower, p.hess_spmv, MadNLP.nzval(kkt.hess_com), pointer(xv), pointer(wv), beta)
    spmv(:b2_spmv_t, p.jac_spmv, MadNLP.nzval(kkt.jac_com), pointer(MadNLP.dual(x)), pointer(wv), one(T))
    spmv(:b2_spmv_n, p.jac_spmv, MadNLP.nzval(kkt.jac_com), pointer(xv), pointer(MadNLP.dual(w)), beta)
    check(ccall((:b2_scaled_kktmul, libb200kkt), Cint,
        (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        p.bounds, length(kkt.du_diag), pointer(kkt.reg), pointer(kkt.du_diag), pointer(kkt.l_lower), pointer(kkt.u_lower),
        pointer(kkt.l_diag), pointer(kkt.u_diag), alpha, beta, pointer(xv), pointer(wv), st), SolveException)
    return w
end

function MadNLP.jtprod!(y::CuVector{T}, kkt::B200ScaledKKT{T}, x::CuVector{T}) where T
    check(ccall((:b2_spmv_t, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}),
        uplans(kkt).jac_spmv, pointer(MadNLP.nzval(kkt.jac_com)), pointer(x), pointer(y), one(T), zero(T), stream_ptr()), SolveException)
    return y
end

# ---------------------------------------------------------------------------------------------------------------------
# Optional: the vector passes of RichardsonIterator (src/LinearSolvers/backsolve.jl:36-52) as single launches.
#   b200_richardson_begin!(b, w, x, norms)   norms[3] = ||b||_inf ; x = 0 ; w = b
#   b200_richardson_update!(b, w, x, norms)  x += w ; w = b ; norms[1] = 0 ; norms[2] = ||x||_inf
# followed by mul!(w, kkt, x, -1, 1) through b2_condensed_kkt_mul_norm (accumulates ||w||_inf into norms[1]); one
# 24-byte D2H copy then carries the three norms of the stopping rule.
# ---------------------------------------------------------------------------------------------------------------------
function b200_richardson_begin!(b::CuVector{T}, w::CuVector{T}, x::CuVector{T}, norms::CuVector{T}) where T
    check(ccall((:b2_richardson_begin, libb200kkt), Cint, (Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        length(b), pointer(b), pointer(w), pointer(x), pointer(norms, 3), stream_ptr()), SolveException)
end
function b200_richardson_update!(b::CuVector{T}, w::CuVector{T}, x::CuVector{T}, norms::CuVector{T}) where T
    check(ccall((:b2_richardson_update, libb200kkt), Cint, (Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
        length(b), pointer(b), pointer(w), pointer(x), pointer(norms), stream_ptr()), SolveException)
end

# ---------------------------------------------------------------------------------------------------------------------
# B200KrylovIterator: restarted GMRES preconditioned on the RIGHT by solve_kkt! (csrc/krylov.cu, madnlp.jl_b200/krylov.py), an
# alternative to RichardsonIterator:  madnlp(nlp; iterator = B200KKT.B200KrylovIterator, ...).  It stops and accepts with
# Richardson's residual ratio (tol^(5/4), tol^(5/8)), unlike MadNLPKrylov, which preconditions on the left and stops on the
# absolute norm of the preconditioned residual.  solve_kkt! and mul! are MadNLP's own (they dispatch to this package's overloads);
# everything else goes through the b2_krylov_* entries.  NOT RUN here, like the rest of this file.
# ---------------------------------------------------------------------------------------------------------------------
Base.@kwdef mutable struct B200KrylovOptions <: AbstractOptions
    krylov_restart::Int = 5
    krylov_max_iter::Int = 10
    krylov_tol::Float64 = 1e-10
    krylov_acceptable_tol::Float64 = 1e-5
end

mutable struct B200KrylovIterator{T, KKT} <: MadNLP.AbstractIterator{T}
    kkt::KKT
    opt::B200KrylovOptions
    cnt::Any
    logger::Any
    handle::Ptr{Cvoid}
    Z::Vector{Any}                     # UnreducedKKTVectors over the rows of Z
    state::CuVector{T}                 # wraps the handle's state (B2_KRYLOV_STATE_LEN doubles)
    rec::Vector{T}                     # page-locked host copy of the record (CUDA.pin)
end

const B2_KRYLOV_REC, B2_KRYLOV_STATE_LEN = 344, 352
const KREC_EST, KREC_H, KREC_NORM_W, KREC_NORM_X, KREC_NORM_B, KREC_NORM_B2 = 1, 2, 3, 4, 5, 6    # 1-based

default_options(::Type{B200KrylovIterator}, tol) = B200KrylovOptions(krylov_tol = tol^(5/4), krylov_acceptable_tol = tol^(5/8))

function B200KrylovIterator(kkt; opt = B200KrylovOptions(), logger = MadNLP.MadNLPLogger(), cnt = nothing)
    T = eltype(kkt.pr_diag)
    N = length(kkt.pr_diag) + length(kkt.du_diag) + length(kkt.l_diag) + length(kkt.u_diag)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b2_krylov_create, libb200kkt), Cint, (Int64, Int32, Ptr{Ptr{Cvoid}}), N, opt.krylov_restart, h), SolveException)
    V = Ref{Ptr{Cvoid}}(C_NULL); Zp = Ref{Ptr{Cvoid}}(C_NULL); S = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b2_krylov_buffers, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Ptr{Cvoid}}, Ptr{Ptr{Cvoid}}, Ptr{Ptr{Cvoid}}), h[], V, Zp, S),
          SolveException)
    wrap(p, n) = unsafe_wrap(CuArray, CuPtr{T}(UInt(p)), n)
    n, m, nlb, nub = length(kkt.pr_diag), length(kkt.du_diag), length(kkt.l_diag), length(kkt.u_diag)
    # the fields of MadNLP.UnreducedKKTVector (src/KKT/rhs.jl), built over row k of Z as its allocating constructor builds them
    function zvec(k)
        values = wrap(Zp[] + (k - 1) * N * sizeof(T), N)
        x = MadNLP._madnlp_unsafe_wrap(values, n + m)
        xp = MadNLP._madnlp_unsafe_wrap(values, n)
        xl = MadNLP._madnlp_unsafe_wrap(values, m, n + 1)
        xzl = MadNLP._madnlp_unsafe_wrap(values, nlb, n + m + 1)
        xzu = MadNLP._madnlp_unsafe_wrap(values, nub, n + m + nlb + 1)
        return MadNLP.UnreducedKKTVector(values, x, xp, view(xp, kkt.ind_lb), view(xp, kkt.ind_ub), xl, xzl, xzu)
    end
    Z = [zvec(k) for k in 1:opt.krylov_restart]
    it = B200KrylovIterator{T, typeof(kkt)}(kkt, opt, cnt, logger, h[], Z, wrap(S[], B2_KRYLOV_STATE_LEN),
                                            CUDA.pin(Vector{T}(undef, 8)))
    finalizer(x -> ccall((:b2_krylov_destroy, libb200kkt), Cint, (Ptr{Cvoid},), x.handle), it)
    return it
end

function _krylov_record!(it::B200KrylovIterator)
    copyto!(it.rec, 1, it.state, B2_KRYLOV_REC + 1, 8)       # synchronises
    return it.rec
end

function MadNLP.solve_refine!(x::MadNLP.AbstractKKTVector{T}, it::B200KrylovIterator{T}, b::MadNLP.AbstractKKTVector{T},
                              w::MadNLP.AbstractKKTVector{T}) where T
    kkt, o, h = it.kkt, it.opt, it.handle
    xv, bv, wv = MadNLP.full(x), MadNLP.full(b), MadNLP.full(w)
    ir = 0
    check(ccall((:b2_krylov_begin, libb200kkt), Cint, (Ptr{Cvoid}, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                h, 1, pointer(bv), pointer(xv), pointer(wv), stream_ptr()), SolveException)
    norm_b = norm_b2 = -one(T)
    ratio = zero(T)
    while true
        k = 0
        while true
            check(ccall((:b2_krylov_scale, libb200kkt), Cint, (Ptr{Cvoid}, Int32, CuPtr{T}, Ptr{Cvoid}), h, k, pointer(wv), stream_ptr()),
                  SolveException)
            MadNLP.solve_kkt!(kkt, it.Z[k + 1])
            MadNLP.mul!(w, kkt, it.Z[k + 1], one(T), zero(T))
            check(ccall((:b2_krylov_orthogonalize, libb200kkt), Cint, (Ptr{Cvoid}, Int32, CuPtr{T}, Ptr{Cvoid}), h, k, pointer(wv),
                        stream_ptr()), SolveException)
            rec = _krylov_record!(it)
            # ||b|| arrives with the first step's record (one read per Arnoldi iteration); for b = 0 that step ran on zeros
            if norm_b < 0
                norm_b, norm_b2 = rec[KREC_NORM_B], rec[KREC_NORM_B2]
                norm_b == 0 && (it.cnt !== nothing && (it.cnt.ir = 0); return true)
            end
            ir += 1
            (k + 1 == o.krylov_restart || ir >= o.krylov_max_iter || rec[KREC_H] == 0 ||
             rec[KREC_EST] <= o.krylov_tol * norm_b2) && break
            k += 1
        end
        check(ccall((:b2_krylov_close, libb200kkt), Cint, (Ptr{Cvoid}, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                    h, k + 1, pointer(bv), pointer(xv), pointer(wv), stream_ptr()), SolveException)
        MadNLP.mul!(w, kkt, x, -one(T), one(T))
        check(ccall((:b2_norm_inf, libb200kkt), Cint, (Int64, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), length(wv), pointer(wv),
                    pointer(it.state, B2_KRYLOV_REC + KREC_NORM_W), stream_ptr()), SolveException)
        rec = _krylov_record!(it)
        ratio = rec[KREC_NORM_W] / (min(rec[KREC_NORM_X], 1e6 * norm_b) + norm_b)
        (ratio < o.krylov_tol || ir >= o.krylov_max_iter) && break
        check(ccall((:b2_krylov_begin, libb200kkt), Cint, (Ptr{Cvoid}, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                    h, 0, C_NULL, C_NULL, pointer(wv), stream_ptr()), SolveException)
    end
    it.cnt !== nothing && (it.cnt.ir = ir)
    return ratio < o.krylov_acceptable_tol
end

# inertia read split in two (queue more work behind factorize!, block once): b2_inertia_enqueue / b2_inertia_fetch
inertia_enqueue!(M::B200Solver) = check(ccall((:b2_inertia_enqueue, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), M.handle, stream_ptr()), FactorizationException)
function inertia_fetch(M::B200Solver)
    p = Ref{Int64}(0); z = Ref{Int64}(0); n = Ref{Int64}(0)
    check(ccall((:b2_inertia_fetch, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}), M.handle, p, z, n), FactorizationException)
    return (Int(p[]), Int(z[]), Int(n[]))
end

# ---------------------------------------------------------------------------------------------------------------------
# hessian_approximation = CompactLBFGS with SparseKKTSystem (src/quasi_newton.jl:212-437, src/IPM/factorization.jl:76-139,
# 253-276).  Not executed here (no Julia in the build image).  The stock CompactLBFGS is CONSTRUCTED with its
# `additional_buffers` slot already holding a B200LBFGSState (a type this module owns), so its fourth type parameter is
# B200LBFGSState from the start: init!/update! dispatch on CompactLBFGS{T,VT,MT,<:B200LBFGSState} and the KKT overloads on
# QN <: that type with LS <: B200Solver -- no type piracy.  The create_kkt_system overload below hands the generic constructor
# the marker B200CompactLBFGS (a subtype of AbstractQuasiNewton, so build_hessian_structure takes the diagonal pattern,
# Sparse/utils.jl:18-26), whose create_quasi_newton method builds that struct.  The state lives on the device; the host-side
# counters of the stock struct are not maintained (b2_lbfgs_state reads them).
# ---------------------------------------------------------------------------------------------------------------------
mutable struct B200LBFGSState
    handle::Ptr{Cvoid}
    n::Int
    max_mem::Int
    H::CuMatrix{Float64}          # N x 2 max_history: E, then C^{-1} E after factorize_kkt!
end

function B200LBFGSState(n, N, opt::MadNLP.QuasiNewtonOptions)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b2_lbfgs_create, libb200kkt), Cint, (Int64, Int32, Int32, Float64, Float64, Float64, Ptr{Ptr{Cvoid}}),
                n, opt.max_history, Int32(opt.init_strategy), opt.init_value, opt.sigma_min, opt.sigma_max, h), SymbolicException)
    st = B200LBFGSState(h[], n, opt.max_history, CUDA.zeros(Float64, N, 2 * opt.max_history))
    finalizer(x -> ccall((:b2_lbfgs_destroy, libb200kkt), Cint, (Ptr{Cvoid},), x.handle), st)
    return st
end

# marker passed as hessian_approximation to the generic constructor; never instantiated
abstract type B200CompactLBFGS <: MadNLP.AbstractQuasiNewton{Float64, CuVector{Float64}} end

# the stock struct, field for field as create_quasi_newton(::Type{CompactLBFGS}, ...) builds it (quasi_newton.jl:242-277),
# except additional_buffers
function MadNLP.create_quasi_newton(::Type{B200CompactLBFGS}, cb::MadNLP.AbstractCallback{T,VT}, n;
        options = MadNLP.QuasiNewtonOptions{T}()) where {T, VT<:CuVector{T}}
    N = cb.nvar + length(cb.ind_ineq) + cb.ncon                   # order of the augmented system
    vec() = fill!(MadNLP.create_array(cb, n), zero(T))
    mat(r, c) = fill!(MadNLP.create_array(cb, r, c), zero(T))
    return MadNLP.CompactLBFGS(
        options.init_strategy, vec(), vec(), vec(), vec(), vec(),
        T(options.init_value), T(options.sigma_min), T(options.sigma_max), options.max_history, 0, 0,
        mat(n, 0), mat(n, 0), mat(0, 0), mat(0, 0), mat(0, 0), mat(0, 0), mat(0, 0), mat(0, 0), mat(0, 0), mat(0, 0),
        fill!(MadNLP.create_array(cb, 0), zero(T)), fill!(MadNLP.create_array(cb, 0), zero(T)),
        fill!(MadNLP.create_array(cb, 0), zero(T)),
        B200LBFGSState(n, N, options),
        false,
    )
end

const B200LBFGS{T,VT,MT} = MadNLP.CompactLBFGS{T,VT,MT,<:B200LBFGSState}
const B200LBFGSKKT{T} = MadNLP.SparseKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN<:B200LBFGS,LS<:B200Solver}

function MadNLP.create_kkt_system(::Type{MadNLP.SparseKKTSystem}, cb::MadNLP.SparseCallback{T,VT}, ::Type{LS};
        opt_linear_solver = default_options(LS), hessian_approximation = MadNLP.ExactHessian,
        qn_options = MadNLP.QuasiNewtonOptions()) where {T, VT<:CuVector{T}, LS<:B200Solver}
    qn = hessian_approximation <: MadNLP.CompactLBFGS ? B200CompactLBFGS : hessian_approximation
    return invoke(MadNLP.create_kkt_system, Tuple{Type{MadNLP.SparseKKTSystem}, MadNLP.SparseCallback{T,VT}, Type},
                  MadNLP.SparseKKTSystem, cb, LS; opt_linear_solver, hessian_approximation = qn, qn_options)
end

MadNLP.init!(qn::B200LBFGS{T}, Bk::CuVector{T}, g0::CuVector{T}, f0::T) where T =
    check(ccall((:b2_lbfgs_init, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, Float64, Ptr{Cvoid}),
                qn.additional_buffers.handle, pointer(Bk), pointer(g0), f0, stream_ptr()), FactorizationException)

function MadNLP.update!(qn::B200LBFGS{T}, Bk::CuVector{T}, sk::CuVector{T}, yk::CuVector{T}) where T
    check(ccall((:b2_lbfgs_update, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                qn.additional_buffers.handle, pointer(Bk), pointer(sk), pointer(yk), stream_ptr()), FactorizationException)
    return true          # whether the pair was kept is decided on the device (b2_lbfgs_state)
end

function MadNLP.factorize_kkt!(kkt::B200LBFGSKKT)
    factorize!(kkt.linear_solver)
    st = kkt.quasi_newton.additional_buffers
    check(ccall((:b2_lbfgs_smw_prepare, libb200kkt), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, CuPtr{Float64}, Ptr{Cvoid}),
                st.handle, kkt.linear_solver.handle, size(st.H, 1), pointer(st.H), stream_ptr()), FactorizationException)
    return
end

function MadNLP.solve_kkt!(kkt::B200LBFGSKKT, w::MadNLP.AbstractKKTVector)
    st = kkt.quasi_newton.additional_buffers
    MadNLP.reduce_rhs!(kkt, w)
    w_ = MadNLP.primal_dual(w)
    solve_linear_system!(kkt.linear_solver, w_)
    check(ccall((:b2_lbfgs_smw_apply, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{Float64}, CuPtr{Float64}, Ptr{Cvoid}),
                st.handle, size(st.H, 1), pointer(st.H), pointer(w_), stream_ptr()), SolveException)
    MadNLP.finish_aug_solve!(kkt, w)
    return w
end

function MadNLP.mul!(w::MadNLP.AbstractKKTVector{T}, kkt::B200LBFGSKKT, x::MadNLP.AbstractKKTVector, alpha = one(T), beta = zero(T)) where T
    mul!(MadNLP.primal(w), Symmetric(kkt.hess_com, :L), MadNLP.primal(x), alpha, beta)
    mul!(MadNLP.primal(w), kkt.jac_com', MadNLP.dual(x), alpha, one(T))
    mul!(MadNLP.dual(w), kkt.jac_com, MadNLP.primal(x), alpha, beta)
    check(ccall((:b2_lbfgs_kkt_mul_lowrank, libb200kkt), Cint, (Ptr{Cvoid}, Float64, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                kkt.quasi_newton.additional_buffers.handle, alpha, pointer(MadNLP.full(x)), pointer(MadNLP.full(w)), stream_ptr()),
          SolveException)
    MadNLP._kktmul!(w, x, kkt.reg, kkt.du_diag, kkt.l_lower, kkt.u_lower, kkt.l_diag, kkt.u_diag, alpha, beta)
    return w
end

# ---------------------------------------------------------------------------------------------------------------------
# hessian_approximation = BFGS / DampedBFGS with DenseKKTSystem and DenseCondensedKKTSystem (src/quasi_newton.jl:71-201, 425-437).
# Not executed here (no Julia in the build image).  The create_kkt_system overloads below swap the stock markers for
# B200BFGS / B200DampedBFGS, types this module owns that hold a b2d_qn handle, and `invoke` the generic constructor, which calls
# their create_quasi_newton methods.  They carry the fields eval_lag_hess_wrapper! reads (sk, yk, last_g, last_x, last_jv,
# src/IPM/callbacks.jl:146-192); bsk, r, is_instantiated and the decision live on the device (b2d_qn_state reads them).  Bk is the
# KKT system's `hess`, updated in place on its lower triangle, the only one the dense KKT kernels read.
# ---------------------------------------------------------------------------------------------------------------------
abstract type B200DenseQuasiNewton{T,VT} <: MadNLP.AbstractQuasiNewton{T,VT} end

for (name, kind) in ((:B200BFGS, 1), (:B200DampedBFGS, 2))
    @eval begin
        mutable struct $name{T,VT<:CuVector{T}} <: B200DenseQuasiNewton{T,VT}
            handle::Ptr{Cvoid}
            init_strategy::MadNLP.BFGSInitStrategy      # stored and unused, as in the reference
            sk::VT
            yk::VT
            last_g::VT
            last_x::VT
            last_jv::VT
        end
        function MadNLP.create_quasi_newton(::Type{$name}, cb::MadNLP.AbstractCallback{T,VT}, n;
                options = MadNLP.QuasiNewtonOptions{T}()) where {T, VT<:CuVector{T}}
            h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2d_qn_create, libb200kkt), Cint, (Int64, Int32, Ptr{Ptr{Cvoid}}), n, Int32($kind), h), SymbolicException)
            vec() = fill!(MadNLP.create_array(cb, n), zero(T))
            qn = $name{T,VT}(h[], options.init_strategy, vec(), vec(), vec(), vec(), vec())
            finalizer(x -> ccall((:b2d_qn_destroy, libb200kkt), Cint, (Ptr{Cvoid},), x.handle), qn)
            return qn
        end
    end
end

_b200_dense_qn(qn) = qn <: MadNLP.DampedBFGS ? B200DampedBFGS : qn <: MadNLP.BFGS ? B200BFGS : qn

for KKT in (:DenseKKTSystem, :DenseCondensedKKTSystem)
    @eval function MadNLP.create_kkt_system(::Type{MadNLP.$KKT}, cb::MadNLP.AbstractCallback{T,VT}, ::Type{LS};
            opt_linear_solver = default_options(LS), hessian_approximation = MadNLP.ExactHessian,
            qn_options = MadNLP.QuasiNewtonOptions()) where {T, VT<:CuVector{T}, LS<:B200DenseSolver}
        return invoke(MadNLP.create_kkt_system, Tuple{Type{MadNLP.$KKT}, MadNLP.AbstractCallback{T,VT}, Type},
                      MadNLP.$KKT, cb, LS; opt_linear_solver, hessian_approximation = _b200_dense_qn(hessian_approximation),
                      qn_options)
    end
end

MadNLP.init!(qn::B200DenseQuasiNewton{T}, Bk::CuMatrix{T}, g0::CuVector{T}, f0::T) where T =
    check(ccall((:b2d_qn_init, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, Float64, Ptr{Cvoid}),
                qn.handle, pointer(Bk), pointer(g0), f0, stream_ptr()), FactorizationException)

function MadNLP.update!(qn::B200DenseQuasiNewton{T}, Bk::CuMatrix{T}, sk::CuVector{T}, yk::CuVector{T}) where T
    check(ccall((:b2d_qn_update, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                qn.handle, pointer(Bk), pointer(sk), pointer(yk), stream_ptr()), FactorizationException)
    return true          # whether BFGS skipped the pair is decided on the device (b2d_qn_state)
end

# ---------------------------------------------------------------- inertia_correction_method = InertiaFree
# mul_hess_blk! (src/IPM/factorization.jl:326-350) and curv_test (src/IPM/solver.jl:785-788) for every KKT type above, dispatched on
# the KKT's linear solver (B200Solver / B200DenseSolver, owned here): the Hessian product (b2_spmv_symlower on hess_com, b2d_symv_lower
# on hess), then b2_mul_hess_blk_tail, which with a result buffer also reduces the four dot products and takes the decision on the
# device.  curv_test reads the 6-double result with one copy.  set_g_ifr! and set_aug_rhs_ifr! stay MadNLP's broadcasts on the
# solver's own vectors; b2_set_g_ifr / b2_set_aug_rhs_ifr are their one-launch equivalents.  Like the rest of this file, NOT RUN.
const B200SparseAugKKT{T} = MadNLP.SparseKKTSystem{T,VT,MT,QN,LS} where {VT<:CuVector{T},MT,QN,LS<:B200Solver}
const B200IFRKKT{T} = Union{B200SparseAugKKT{T},B200UnreducedKKT{T},B200CondensedKKT{T},B200AnyDenseKKT{T}}
# the types whose restoration phase and solve sites run here: the inertia-free ones and ScaledSparseKKTSystem, which has no mul_hess_blk!
const B200RRKKT{T} = Union{B200IFRKKT{T},B200ScaledKKT{T}}

mutable struct IFRPlans
    hess_spmv::Ptr{Cvoid}        # b2_spmv_plan of hess_com (C_NULL for the dense types)
    bounds::Ptr{Cvoid}           # b2_bounds over n_tot (its curvature-test scratch is used)
    result::CuVector{Float64}    # B2_CURV_RESULT_LEN = 6: wx't, wx'n, g'n, t't, lhs, pass
    result_h::Vector{Float64}
end
const _ifr_plans = IdDict{Any,IFRPlans}()      # linear solver -> plans

function ifr_plans(kkt::B200RRKKT)
    get!(_ifr_plans, kkt.linear_solver) do
        sp = C_NULL
        if !(kkt isa B200AnyDenseKKT)
            H = kkt.hess_com
            cp = Int32.(Array(H.colPtr) .- 1); rv = Int32.(Array(H.rowVal) .- 1)
            h = Ref{Ptr{Cvoid}}(C_NULL)
            check(ccall((:b2_spmv_plan_create, libb200kkt), Cint, (Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Ptr{Cvoid}}),
                        size(H, 1), size(H, 2), cp, rv, h), SymbolicException)
            sp = h[]
        end
        lb = Int64.(Array(kkt.ind_lb) .- 1); ub = Int64.(Array(kkt.ind_ub) .- 1)
        b = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b2_bounds_create, libb200kkt), Cint, (Int64, Int64, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Ptr{Cvoid}}),
                    length(kkt.pr_diag), length(lb), length(ub), lb, ub, b), SymbolicException)
        IFRPlans(sp, b[], CUDA.zeros(Float64, 6), zeros(Float64, 6))
    end
end

function _hess_blk!(wx::CuVector{T}, kkt::B200IFRKKT{T}, t::CuVector{T}, n, g, tol, result) where T
    p = ifr_plans(kkt)
    if kkt isa B200AnyDenseKKT
        nh = size(kkt.hess, 1)
        check(ccall((:b2d_symv_lower, libb200kkt), Cint, (Int32, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}),
                    nh, nh, pointer(kkt.hess), pointer(t), pointer(wx), one(T), zero(T), stream_ptr()), SolveException)
    else
        nh = size(kkt.hess_com, 1)
        check(ccall((:b2_spmv_symlower, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, Ptr{Cvoid}),
                    p.hess_spmv, pointer(MadNLP.nzval(kkt.hess_com)), pointer(t), pointer(wx), one(T), zero(T), stream_ptr()), SolveException)
    end
    ptr_or_null(v) = v === nothing ? CuPtr{T}(0) : pointer(v)
    check(ccall((:b2_mul_hess_blk_tail, libb200kkt), Cint,
                (Ptr{Cvoid}, Int64, Int32, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T},
                 Cdouble, CuPtr{T}, Ptr{Cvoid}),
                p.bounds, nh, Int32(kkt isa B200UnreducedKKT), pointer(kkt.pr_diag), pointer(kkt.l_lower), pointer(kkt.l_diag),
                pointer(kkt.u_lower), pointer(kkt.u_diag), pointer(t), pointer(wx), ptr_or_null(n), ptr_or_null(g), Float64(tol),
                ptr_or_null(result), stream_ptr()), SolveException)
    return wx
end

MadNLP.mul_hess_blk!(wx::CuVector{T}, kkt::B200IFRKKT{T}, t::CuVector{T}) where T = _hess_blk!(wx, kkt, t, nothing, nothing, 0.0, nothing)

function MadNLP.curv_test(t::CuVector{T}, n::CuVector{T}, g::CuVector{T}, kkt::B200IFRKKT{T}, wx::CuVector{T}, inertia_free_tol) where T
    p = ifr_plans(kkt)
    _hess_blk!(wx, kkt, t, n, g, inertia_free_tol, p.result)
    copyto!(p.result_h, p.result)                  # the one synchronising read of the test
    return p.result_h[6] == 1.0
end

# ---------------------------------------------------------------- feasibility restoration (robust!, src/IPM/solver.jl:413-540)
# set_aug_RR!, set_aug_rhs_RR! and set_f_RR! / initialize_robust_restorer! dispatch on a KKT system with our linear solver (directly, or
# through the KKTSystem parameter of MadNLPSolver).  finish_aug_solve_RR! and the _R reductions take plain vectors in the reference, so
# they cannot be overloaded without type piracy: they are this module's functions with the KKT system as first argument, and robust! /
# filter_line_search_RR! call them instead (one line per call site, INTEGRATION.md).  The b2_bounds object and a result slot come from
# ifr_plans.  Every vector is the solver's own full vector (zl / zu via full(...), +-Inf bounds); indices 0-based on the device side.
# Like the rest of this file, NOT RUN.
const B200RRSolver{T} = MadNLP.MadNLPSolver{T,VT,VI,KKT} where {VT,VI,KKT<:B200RRKKT{T}}
_ptr(v) = pointer(v)
_sp() = stream_ptr()

function MadNLP.set_aug_RR!(kkt::B200RRKKT{T}, solver::MadNLP.AbstractMadNLPSolver, RR::MadNLP.RobustRestorer) where T
    p, o = ifr_plans(kkt), MadNLP.get_opt(solver)
    x, xl, xu = MadNLP.full(MadNLP.get_x(solver)), MadNLP.full(MadNLP.get_xl(solver)), MadNLP.full(MadNLP.get_xu(solver))
    zl, zu = MadNLP.full(MadNLP.get_zl(solver)), MadNLP.full(MadNLP.get_zu(solver))
    # ScaledSparseKKTSystem's set_aug_RR! (kernels.jl:89-104) writes l_diag = x - xl and u_diag = xu - x
    entry = kkt isa B200ScaledKKT ? :b2_set_aug_rr_scaled : :b2_set_aug_rr
    check(ccall((entry, libb200kkt), Cint,
                (Ptr{Cvoid}, Int64, Cdouble, Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 16)..., Ptr{Cvoid}),
                p.bounds, length(RR.pp), o.default_primal_regularization, o.default_dual_regularization, RR.zeta, _ptr(RR.D_R),
                _ptr(RR.pp), _ptr(RR.nn), _ptr(RR.zp), _ptr(RR.zn), _ptr(x), _ptr(xl), _ptr(xu), _ptr(zl), _ptr(zu), _ptr(kkt.reg),
                _ptr(kkt.du_diag), _ptr(kkt.l_lower), _ptr(kkt.u_lower), _ptr(kkt.l_diag), _ptr(kkt.u_diag), _sp()), SolveException)
    MadNLP._set_aug_diagonal!(kkt)                 # each type's own (the unreduced one takes the square roots)
    return
end

function MadNLP.set_aug_rhs_RR!(solver::MadNLP.AbstractMadNLPSolver, kkt::B200RRKKT{T}, RR::MadNLP.RobustRestorer, rho) where T
    pl = ifr_plans(kkt)
    x, xl, xu = MadNLP.full(MadNLP.get_x(solver)), MadNLP.full(MadNLP.get_xl(solver)), MadNLP.full(MadNLP.get_xu(solver))
    zl, zu = MadNLP.full(MadNLP.get_zl(solver)), MadNLP.full(MadNLP.get_zu(solver))
    check(ccall((:b2_set_aug_rhs_rr, libb200kkt), Cint, (Ptr{Cvoid}, Int64, ntuple(_ -> CuPtr{T}, 13)..., Cdouble, Cdouble, CuPtr{T}, Ptr{Cvoid}),
                pl.bounds, length(RR.pp), _ptr(x), _ptr(xl), _ptr(xu), _ptr(zl), _ptr(zu), _ptr(MadNLP.get_jacl(solver)), _ptr(RR.f_R),
                _ptr(MadNLP.get_c(solver)), _ptr(MadNLP.get_y(solver)), _ptr(RR.pp), _ptr(RR.nn), _ptr(RR.zp), _ptr(RR.zn), RR.mu_R,
                Float64(rho), _ptr(MadNLP.full(MadNLP.get_p(solver))), _sp()), SolveException)
    return
end

function MadNLP.set_f_RR!(solver::B200RRSolver{T}, RR::MadNLP.RobustRestorer) where T
    x = MadNLP.full(MadNLP.get_x(solver))
    check(ccall((:b2_set_f_rr, libb200kkt), Cint, (Int64, Cdouble, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                length(x), RR.zeta, _ptr(RR.D_R), _ptr(x), _ptr(RR.x_ref), _ptr(RR.f_R), _sp()), SolveException)
    return
end

# initialize_robust_restorer! (src/IPM/restoration.jl:39-75): the two norms of c in one read, then one launch (b2_rr_init) and the
# obj_val_R reduction
function MadNLP.initialize_robust_restorer!(solver::B200RRSolver{T}) where T
    MadNLP.get_RR(solver) === nothing && MadNLP.set_RR!(solver, MadNLP.RobustRestorer(solver))
    RR::MadNLP.RobustRestorer = MadNLP.get_RR(solver)
    kkt, o, c = MadNLP.get_kkt(solver), MadNLP.get_opt(solver), MadNLP.get_c(solver)
    pl = ifr_plans(kkt)
    r = CUDA.zeros(T, 2)
    check(ccall((:b2_get_theta, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), pl.bounds, length(c), _ptr(c),
                _ptr(r), _sp()), SolveException)
    check(ccall((:b2_norm_inf, libb200kkt), Cint, (Int64, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), length(c), _ptr(c), _ptr(r) + sizeof(T), _sp()),
          SolveException)
    rh = Array(r)
    RR.theta_ref = rh[1]
    RR.mu_R = max(MadNLP.get_mu(solver), rh[2])
    RR.tau_R = max(o.tau_min, 1 - RR.mu_R)
    RR.zeta = sqrt(RR.mu_R)
    x = MadNLP.full(MadNLP.get_x(solver))
    zl, zu = MadNLP.full(MadNLP.get_zl(solver)), MadNLP.full(MadNLP.get_zu(solver))
    check(ccall((:b2_rr_init, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 10)..., Ptr{Cvoid}),
                pl.bounds, length(c), _ptr(x), _ptr(c), RR.mu_R, o.rho, _ptr(RR.x_ref), _ptr(RR.D_R), _ptr(RR.f_R), _ptr(RR.pp),
                _ptr(RR.nn), _ptr(RR.zp), _ptr(RR.zn), _ptr(MadNLP.get_y(solver)), _ptr(zl), _ptr(zu), _sp()), SolveException)
    RR.obj_val_R = get_obj_val_R(kkt, RR.pp, RR.nn, RR.D_R, x, RR.x_ref, o.rho, RR.zeta)
    empty!(RR.filter)
    push!(RR.filter, (MadNLP.get_theta_max(solver), -Inf))
    MadNLP.get_cnt(solver).t = 0
    MadNLP.set_del_w!(solver, zero(T))
end

# finish_aug_solve_RR!(dpp, dnn, dzp, dzn, l, dl, pp, nn, zp, zn, mu_R, rho) (src/IPM/kernels.jl:251-257)
function finish_aug_solve_RR!(kkt::B200RRKKT{T}, dpp, dnn, dzp, dzn, l, dl, pp, nn, zp, zn, mu_R, rho) where T
    check(ccall((:b2_finish_aug_solve_rr, libb200kkt), Cint, (Int64, ntuple(_ -> CuPtr{T}, 6)..., Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 4)...,
                Ptr{Cvoid}), length(l), _ptr(l), _ptr(dl), _ptr(pp), _ptr(nn), _ptr(zp), _ptr(zn), mu_R, rho, _ptr(dpp), _ptr(dnn),
                _ptr(dzp), _ptr(dzn), _sp()), SolveException)
    return
end

# the reductions (kernels.jl:390-636): one launch each into the plans' result slot, then one read.  Arguments as in the reference
# (vectors full length: x, xl, xu, zl, zu, f_R, jacl, dx n_tot; c, l, pp, nn, zp, zn and steps m; dzl / dzu compressed).
function _reduce(kkt::B200RRKKT{T}, sym::Symbol, argt::Tuple, args...) where T
    pl = ifr_plans(kkt)
    check(ccall(Libdl.dlsym(Libdl.dlopen(libb200kkt), sym), Cint, (Ptr{Cvoid}, argt..., CuPtr{T}, Ptr{Cvoid}), pl.bounds, args...,
                _ptr(pl.result), _sp()), SolveException)
    return Array(view(pl.result, 1:1))[1]
end
const _V = CuPtr{Float64}
get_theta(kkt::B200RRKKT, c) = _reduce(kkt, :b2_get_theta, (Int64, _V), length(c), _ptr(c))
get_theta_R(kkt::B200RRKKT, c, p, n) = _reduce(kkt, :b2_get_theta_r, (Int64, _V, _V, _V), length(c), _ptr(c), _ptr(p), _ptr(n))
get_inf_pr_R(kkt::B200RRKKT, c, p, n) = _reduce(kkt, :b2_get_inf_pr_r, (Int64, _V, _V, _V), length(c), _ptr(c), _ptr(p), _ptr(n))
get_obj_val_R(kkt::B200RRKKT, p, n, D_R, x, x_ref, rho, zeta) =
    _reduce(kkt, :b2_get_obj_val_r, (Int64, _V, _V, _V, _V, _V, Cdouble, Cdouble), length(p), _ptr(p), _ptr(n), _ptr(D_R), _ptr(x),
            _ptr(x_ref), rho, zeta)
get_inf_du_R(kkt::B200RRKKT, f_R, l, zl, zu, jacl, zp, zn, rho, sd) =
    _reduce(kkt, :b2_get_inf_du_r, (Int64, ntuple(_ -> _V, 7)..., Cdouble, Cdouble), length(l), _ptr(f_R), _ptr(l), _ptr(zl), _ptr(zu),
            _ptr(jacl), _ptr(zp), _ptr(zn), rho, sd)
get_inf_compl_R(kkt::B200RRKKT, x, xl, xu, zl, zu, pp, zp, nn, zn, mu_R, sc) =
    _reduce(kkt, :b2_get_inf_compl_r, (Int64, ntuple(_ -> _V, 9)..., Cdouble, Cdouble), length(pp), _ptr(x), _ptr(xl), _ptr(xu), _ptr(zl),
            _ptr(zu), _ptr(pp), _ptr(zp), _ptr(nn), _ptr(zn), mu_R, sc)
get_alpha_max_R(kkt::B200RRKKT, x, xl, xu, dx, pp, dpp, nn, dnn, tau_R) =
    _reduce(kkt, :b2_get_alpha_max_r, (Int64, ntuple(_ -> _V, 8)..., Cdouble), length(pp), _ptr(x), _ptr(xl), _ptr(xu), _ptr(dx), _ptr(pp),
            _ptr(dpp), _ptr(nn), _ptr(dnn), tau_R)
get_alpha_z_R(kkt::B200RRKKT, zl, zu, dzl, dzu, zp, dzp, zn, dzn, tau_R) =
    _reduce(kkt, :b2_get_alpha_z_r, (Int64, ntuple(_ -> _V, 8)..., Cdouble), length(zp), _ptr(zl), _ptr(zu), _ptr(dzl), _ptr(dzu), _ptr(zp),
            _ptr(dzp), _ptr(zn), _ptr(dzn), tau_R)
get_varphi_R(kkt::B200RRKKT, obj_val, x, xl, xu, pp, nn, mu_R) =
    _reduce(kkt, :b2_get_varphi_r, (Int64, Cdouble, ntuple(_ -> _V, 5)..., Cdouble), length(pp), obj_val, _ptr(x), _ptr(xl), _ptr(xu),
            _ptr(pp), _ptr(nn), mu_R)
get_varphi_d_R(kkt::B200RRKKT, f_R, x, xl, xu, dx, pp, nn, dpp, dnn, mu_R, rho) =
    _reduce(kkt, :b2_get_varphi_d_r, (Int64, ntuple(_ -> _V, 9)..., Cdouble, Cdouble), length(pp), _ptr(f_R), _ptr(x), _ptr(xl), _ptr(xu),
            _ptr(dx), _ptr(pp), _ptr(nn), _ptr(dpp), _ptr(dnn), mu_R, rho)

# ---- the other solve sites (src/IPM/solver.jl): initialize_dual with DualInitializeLeastSquares (:86-97), robust!'s return to the regular
# phase (:518-530), second_order_correction (:547-608) and restore! (:300-411).  The factorisation and the refined solve stay MadNLP's
# (factorize_wrapper!, solve_refine_wrapper!); the right-hand sides, the y rule, get_F, restore!'s step and the trial point are one launch
# each (csrc/solve_sites.cu), with every step length read by the kernels from device memory.  The filter tests, the callbacks and the
# counters stay MadNLP's.  robust! calls b200_reinitialize_dual! in place of its exit block (one line, INTEGRATION.md).  Like the rest of
# this file, NOT RUN.
function _set_initial_rhs!(solver::B200RRSolver{T}) where T
    pl, m = ifr_plans(MadNLP.get_kkt(solver)), length(MadNLP.get_c(solver))
    check(ccall((:b2_set_initial_rhs, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), pl.bounds, m,
                _ptr(MadNLP.full(MadNLP.get_f(solver))), _ptr(MadNLP.full(MadNLP.get_zl(solver))), _ptr(MadNLP.full(MadNLP.get_zu(solver))),
                _ptr(MadNLP.full(MadNLP.get_p(solver))), _sp()), SolveException)
end

function _dual_init_select!(solver::B200RRSolver{T}, solved::Bool) where T
    pl, y = ifr_plans(MadNLP.get_kkt(solver)), MadNLP.get_y(solver)
    check(ccall((:b2_dual_init_select, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, Int32, Cdouble, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}),
                pl.bounds, length(y), _ptr(MadNLP.dual(MadNLP.get_d(solver))), Int32(solved), MadNLP.get_opt(solver).constr_mult_init_max,
                _ptr(y), _ptr(pl.result), _sp()), SolveException)
    return
end

# set_aug_rhs!(solver, kkt, w, mu) + dual_inf_perturbation!; w = c, or c_trial + alpha c when c_trial !== nothing
function _set_aug_rhs_perturbed!(solver::B200RRSolver{T}, c, c_trial, alpha) where T
    pl, o = ifr_plans(MadNLP.get_kkt(solver)), MadNLP.get_opt(solver)
    v = map(MadNLP.full, (MadNLP.get_x(solver), MadNLP.get_xl(solver), MadNLP.get_xu(solver), MadNLP.get_f(solver), MadNLP.get_zl(solver),
                          MadNLP.get_zu(solver)))
    llb = CuVector{Int64}(MadNLP.get_ind_llb(solver) .- 1); uub = CuVector{Int64}(MadNLP.get_ind_uub(solver) .- 1)
    check(ccall((:b2_set_aug_rhs_perturbed, libb200kkt), Cint,
                (Ptr{Cvoid}, Int64, ntuple(_ -> CuPtr{T}, 9)..., Cdouble, Cdouble, Cdouble, Int64, CuPtr{Int64}, Int64, CuPtr{Int64}, CuPtr{T},
                 Ptr{Cvoid}), pl.bounds, length(c), map(_ptr, v)..., _ptr(MadNLP.get_jacl(solver)), _ptr(c),
                c_trial === nothing ? CU_NULL : _ptr(c_trial), Float64(alpha), MadNLP.get_mu(solver), o.kappa_d, length(llb), _ptr(llb),
                length(uub), _ptr(uub), _ptr(MadNLP.full(MadNLP.get_p(solver))), _sp()), SolveException)
end

function MadNLP.initialize_dual(solver::B200RRSolver{T}, ::Type{MadNLP.DualInitializeLeastSquares}) where T
    _set_initial_rhs!(solver)
    MadNLP.factorize_wrapper!(solver)
    is_solved = MadNLP.solve_refine_wrapper!(MadNLP.get_d(solver), solver, MadNLP.get_p(solver), MadNLP.get__w4(solver))
    _dual_init_select!(solver, is_solved)
end

# robust!'s exit block (solver.jl:518-530), in its order: no compress_hessian!, so a dense augmented system keeps its stale diag_hess
function b200_reinitialize_dual!(solver::B200RRSolver{T}) where T
    _set_initial_rhs!(solver)
    MadNLP.initialize!(MadNLP.get_kkt(solver))
    MadNLP.factorize_wrapper!(solver)
    MadNLP.solve_refine_wrapper!(MadNLP.get_d(solver), solver, MadNLP.get_p(solver), MadNLP.get__w4(solver))
    _dual_init_select!(solver, true)
end

function MadNLP.second_order_correction(solver::B200RRSolver{T}, alpha_max, theta, varphi, theta_trial, varphi_d,
                                        switching_condition::Bool) where T
    o, kkt, pl = MadNLP.get_opt(solver), MadNLP.get_kkt(solver), ifr_plans(MadNLP.get_kkt(solver))
    w1 = MadNLP.get__w1(solver)
    x, xl, xu = MadNLP.full(MadNLP.get_x(solver)), MadNLP.full(MadNLP.get_xl(solver)), MadNLP.full(MadNLP.get_xu(solver))
    theta_soc_old = theta_trial
    for p = 1:o.max_soc
        # pass 1: wy = c_trial + alpha_max c on the fly; later passes: wy = dual(_w1), the previous correction's dual part (as the reference)
        p == 1 ? _set_aug_rhs_perturbed!(solver, MadNLP.get_c(solver), MadNLP.get_c_trial(solver), alpha_max) :
                 _set_aug_rhs_perturbed!(solver, MadNLP.dual(w1), nothing, zero(T))
        MadNLP.solve_refine_wrapper!(w1, solver, MadNLP.get_p(solver), MadNLP.get__w4(solver))
        check(ccall((:b2_get_alpha_max, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, CuPtr{T}, Ptr{Cvoid}),
                    pl.bounds, _ptr(x), _ptr(xl), _ptr(xu), _ptr(MadNLP.primal(w1)), MadNLP.get_tau(solver), _ptr(pl.result), _sp()), SolveException)
        check(ccall((:b2_soc_trial, libb200kkt), Cint, (Int64, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), length(x), _ptr(pl.result),
                    _ptr(x), _ptr(MadNLP.primal(w1)), _ptr(MadNLP.full(MadNLP.get_x_trial(solver))), _sp()), SolveException)
        alpha_soc = Array(view(pl.result, 1:1))[1]
        MadNLP.eval_cons_wrapper!(solver, MadNLP.get_c_trial(solver), MadNLP.get_x_trial(solver))
        MadNLP.set_obj_val_trial!(solver, MadNLP.eval_f_wrapper(solver, MadNLP.get_x_trial(solver)))
        theta_soc = get_theta(kkt, MadNLP.get_c_trial(solver))
        varphi_soc = MadNLP.get_varphi(MadNLP.get_obj_val_trial(solver), MadNLP.get_x_trial_lr(solver), MadNLP.get_xl_r(solver),
                                       MadNLP.get_xu_r(solver), MadNLP.get_x_trial_ur(solver), MadNLP.get_mu(solver))
        !MadNLP.is_filter_acceptable(MadNLP.get_filter(solver), theta_soc, varphi_soc) && break
        if theta <= MadNLP.get_theta_min(solver) && switching_condition
            if MadNLP.is_armijo(varphi_soc, varphi, o.eta_phi, MadNLP.get_alpha(solver), varphi_d)
                MadNLP.set_ftype!(solver, "F"); MadNLP.set_alpha!(solver, alpha_soc)
                return true
            end
        elseif MadNLP.is_sufficient_progress(theta_soc, theta, o.gamma_theta, varphi_soc, varphi, o.gamma_phi, MadNLP.has_constraints(solver))
            MadNLP.set_ftype!(solver, "H"); MadNLP.set_alpha!(solver, alpha_soc)
            return true
        end
        theta_soc > o.kappa_soc * theta_soc_old && break
        theta_soc_old = theta_soc
    end
    return false
end

function MadNLP.restore!(solver::B200RRSolver{T}) where T
    o, kkt, pl = MadNLP.get_opt(solver), MadNLP.get_kkt(solver), ifr_plans(MadNLP.get_kkt(solver))
    MadNLP.set_del_w!(solver, zero(T))
    w1, w2, d = MadNLP.get__w1(solver), MadNLP.get__w2(solver), MadNLP.get_d(solver)
    x, xl, xu = MadNLP.full(MadNLP.get_x(solver)), MadNLP.full(MadNLP.get_xl(solver)), MadNLP.full(MadNLP.get_xu(solver))
    zl, zu, f = MadNLP.full(MadNLP.get_zl(solver)), MadNLP.full(MadNLP.get_zu(solver)), MadNLP.full(MadNLP.get_f(solver))
    y, c, jacl = MadNLP.get_y(solver), MadNLP.get_c(solver), MadNLP.get_jacl(solver)
    copyto!(MadNLP.primal(w1), MadNLP.primal(MadNLP.get_x(solver))); copyto!(MadNLP.dual(w1), y); copyto!(MadNLP.dual(w2), c)
    get_F() = _reduce(kkt, :b2_get_pd_error, (Int64, ntuple(_ -> _V, 8)..., Cdouble), length(c), _ptr(c), _ptr(f), _ptr(zl), _ptr(zu),
                      _ptr(jacl), _ptr(x), _ptr(xl), _ptr(xu), MadNLP.get_mu(solver))
    F = get_F()
    MadNLP.set_alpha_z!(solver, zero(T)); MadNLP.set_ftype!(solver, "R")
    a = CUDA.zeros(T, 3)                                   # alpha_max, alpha_z, alpha
    while true
        check(ccall((:b2_get_alpha_max, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, CuPtr{T}, Ptr{Cvoid}),
                    pl.bounds, _ptr(x), _ptr(xl), _ptr(xu), _ptr(MadNLP.primal(d)), MadNLP.get_tau(solver), _ptr(a), _sp()), SolveException)
        check(ccall((:b2_get_alpha_z, libb200kkt), Cint, (Ptr{Cvoid}, CuPtr{T}, CuPtr{T}, CuPtr{T}, CuPtr{T}, Cdouble, CuPtr{T}, Ptr{Cvoid}),
                    pl.bounds, _ptr(zl), _ptr(zu), _ptr(MadNLP.dual_lb(d)), _ptr(MadNLP.dual_ub(d)), MadNLP.get_tau(solver), _ptr(a) + sizeof(T),
                    _sp()), SolveException)
        check(ccall((:b2_restore_update, libb200kkt), Cint, (Ptr{Cvoid}, Int64, ntuple(_ -> CuPtr{T}, 11)..., Ptr{Cvoid}), pl.bounds,
                    length(y), _ptr(a), _ptr(a) + sizeof(T), _ptr(a) + 2 * sizeof(T), _ptr(MadNLP.primal(d)), _ptr(MadNLP.dual(d)),
                    _ptr(MadNLP.dual_lb(d)), _ptr(MadNLP.dual_ub(d)), _ptr(x), _ptr(y), _ptr(zl), _ptr(zu), _sp()), SolveException)
        MadNLP.set_alpha!(solver, Array(view(a, 3:3))[1])
        MadNLP.eval_cons_wrapper!(solver, c, MadNLP.get_x(solver))
        MadNLP.eval_grad_f_wrapper!(solver, MadNLP.get_f(solver), MadNLP.get_x(solver))
        MadNLP.set_obj_val!(solver, MadNLP.eval_f_wrapper(solver, MadNLP.get_x(solver)))
        !o.jacobian_constant && MadNLP.eval_jac_wrapper!(solver, kkt, MadNLP.get_x(solver))
        MadNLP.jtprod!(jacl, kkt, y)
        F_trial = get_F()
        if F_trial > o.soft_resto_pderror_reduction_factor * F
            copyto!(MadNLP.primal(MadNLP.get_x(solver)), MadNLP.primal(w1)); copyto!(y, MadNLP.dual(w1)); copyto!(c, MadNLP.dual(w2))
            return MadNLP.ROBUST
        end
        MadNLP.adjust_boundary!(MadNLP.get_x_lr(solver), MadNLP.get_xl_r(solver), MadNLP.get_x_ur(solver), MadNLP.get_xu_r(solver),
                                MadNLP.get_mu(solver))
        F = F_trial
        theta = get_theta(kkt, c)
        varphi = MadNLP.get_varphi(MadNLP.get_obj_val(solver), MadNLP.get_x_lr(solver), MadNLP.get_xl_r(solver), MadNLP.get_xu_r(solver),
                                   MadNLP.get_x_ur(solver), MadNLP.get_mu(solver))
        MadNLP.get_cnt(solver).k += 1
        !(MadNLP.get_intermediate_callback(solver)(solver, MadNLP.UserCallbackRestore())::Bool) && return MadNLP.USER_REQUESTED_STOP
        MadNLP.is_filter_acceptable(MadNLP.get_filter(solver), theta, varphi) ? (return MadNLP.REGULAR) : (MadNLP.get_cnt(solver).t += 1)
        MadNLP.get_cnt(solver).k >= o.max_iter && return MadNLP.MAXIMUM_ITERATIONS_EXCEEDED
        time() - MadNLP.get_cnt(solver).start_time >= o.max_wall_time && return MadNLP.MAXIMUM_WALLTIME_EXCEEDED
        sd = MadNLP.get_sd(y, MadNLP.get_zl_r(solver), MadNLP.get_zu_r(solver), o.s_max)
        sc = MadNLP.get_sc(MadNLP.get_zl_r(solver), MadNLP.get_zu_r(solver), o.s_max)
        MadNLP.set_inf_pr!(solver, MadNLP.get_inf_pr(c))
        MadNLP.set_inf_du!(solver, MadNLP.get_inf_du(MadNLP.primal(MadNLP.get_f(solver)), MadNLP.primal(MadNLP.get_zl(solver)),
                                                     MadNLP.primal(MadNLP.get_zu(solver)), jacl, sd))
        cl = (MadNLP.get_x_lr(solver), MadNLP.get_xl_r(solver), MadNLP.get_zl_r(solver), MadNLP.get_xu_r(solver), MadNLP.get_x_ur(solver),
              MadNLP.get_zu_r(solver))
        MadNLP.set_inf_compl!(solver, MadNLP.get_inf_compl(cl..., zero(T), sc))
        MadNLP.set_inf_compl_mu!(solver, MadNLP.get_inf_compl(cl..., MadNLP.get_mu(solver), sc))
        MadNLP.print_iter(solver)
        !o.hessian_constant && MadNLP.eval_lag_hess_wrapper!(solver, kkt, MadNLP.get_x(solver), y)
        entry = kkt isa B200ScaledKKT ? :b2_set_aug_diagonal_iterate_scaled : :b2_set_aug_diagonal_iterate   # K2.5's bound signs
        check(ccall((entry, libb200kkt), Cint, (Ptr{Cvoid}, Int64, Cdouble, Cdouble, ntuple(_ -> CuPtr{T}, 11)..., Ptr{Cvoid}),
                    pl.bounds, length(y), o.default_primal_regularization, o.default_dual_regularization, _ptr(x), _ptr(xl), _ptr(xu),
                    _ptr(zl), _ptr(zu), _ptr(kkt.reg), _ptr(kkt.du_diag), _ptr(kkt.l_lower), _ptr(kkt.u_lower), _ptr(kkt.l_diag),
                    _ptr(kkt.u_diag), _sp()), SolveException)
        MadNLP._set_aug_diagonal!(kkt)
        _set_aug_rhs_perturbed!(solver, c, nothing, zero(T))
        MadNLP.factorize_wrapper!(solver)
        MadNLP.solve_refine_wrapper!(d, solver, MadNLP.get_p(solver), MadNLP.get__w4(solver))
        MadNLP.set_ftype!(solver, "f")
    end
end

# ---- the adaptive barrier rules (get_adaptive_mu, src/IPM/barrier.jl:260-316) for the solvers this module owns.  The quality-function
# rule keeps the reference's sequence (set_aug_rhs! with mu = 0, the two solves into _w3 / _w4 without refinement, on the factor the
# solver holds) and moves the norms, the average complementarity, the centering right-hand side and the whole search to the device:
# the host reads mu once.  _check_progress, the mode switch and _update_monotone! stay MadNLP's.  Like the rest of this file, NOT RUN.
const B2_QF_TRACE = 8
function MadNLP.get_adaptive_mu(solver::B200RRSolver{T}, barrier::MadNLP.QualityFunctionUpdate{T}) where T
    MadNLP.get_nlb(solver) + MadNLP.get_nub(solver) == 0 && return barrier.mu_min
    kkt, o = MadNLP.get_kkt(solver), MadNLP.get_opt(solver)
    pl = ifr_plans(kkt)
    x, xl, xu = MadNLP.full(MadNLP.get_x(solver)), MadNLP.full(MadNLP.get_xl(solver)), MadNLP.full(MadNLP.get_xu(solver))
    zl, zu = MadNLP.full(MadNLP.get_zl(solver)), MadNLP.full(MadNLP.get_zu(solver))
    p, m = MadNLP.get_p(solver), length(MadNLP.get_c(solver))
    step_aff, step_cen = MadNLP.get__w3(solver), MadNLP.get__w4(solver)
    scal = CuVector{T}([MadNLP.get_tau(solver), zero(T), zero(T), zero(T)])   # B2_QF_TAU, _NRM_PRIMAL, _NRM_DUAL, _MU_AVG
    MadNLP.set_aug_rhs!(solver, kkt, MadNLP.get_c(solver), zero(T))
    check(ccall((:b2_primal_dual_norm2, libb200kkt), Cint, (Ptr{Cvoid}, Int64, CuPtr{T}, CuPtr{T}, Ptr{Cvoid}), pl.bounds, m,
                _ptr(MadNLP.full(p)), _ptr(scal) + sizeof(T), _sp()), SolveException)
    copyto!(MadNLP.full(step_aff), MadNLP.full(p))
    MadNLP.solve_kkt!(kkt, step_aff)
    check(ccall((:b2_get_average_complementarity, libb200kkt), Cint, (Ptr{Cvoid}, ntuple(_ -> CuPtr{T}, 6)..., Ptr{Cvoid}), pl.bounds,
                _ptr(x), _ptr(xl), _ptr(xu), _ptr(zl), _ptr(zu), _ptr(scal) + 3 * sizeof(T), _sp()), SolveException)
    llb = CuVector{Int64}(MadNLP.get_ind_llb(solver) .- 1); uub = CuVector{Int64}(MadNLP.get_ind_uub(solver) .- 1)
    check(ccall((:b2_set_centering_aug_rhs, libb200kkt), Cint,
                (Ptr{Cvoid}, Int64, Int64, CuPtr{Int64}, Int64, CuPtr{Int64}, CuPtr{T}, Cdouble, CuPtr{T}, Ptr{Cvoid}), pl.bounds, m,
                length(llb), _ptr(llb), length(uub), _ptr(uub), _ptr(scal) + 3 * sizeof(T), o.kappa_d, _ptr(MadNLP.full(p)), _sp()),
          SolveException)
    copyto!(MadNLP.full(step_cen), MadNLP.full(p))
    MadNLP.solve_kkt!(kkt, step_cen)
    res = CUDA.zeros(T, B2_QF_TRACE + 4 * (6 + barrier.max_gs_iter))
    check(ccall((:b2_qf_search, libb200kkt), Cint,
                (Ptr{Cvoid}, Int64, ntuple(_ -> CuPtr{T}, 8)..., Cdouble, Cdouble, Cdouble, Cdouble, Cdouble, Int32, CuPtr{T}, Ptr{Cvoid}),
                pl.bounds, m, _ptr(x), _ptr(xl), _ptr(xu), _ptr(zl), _ptr(zu), _ptr(MadNLP.full(step_aff)), _ptr(MadNLP.full(step_cen)),
                _ptr(scal), barrier.sigma_min, barrier.sigma_max, barrier.mu_min, barrier.mu_max, barrier.sigma_tol,
                Int32(barrier.max_gs_iter), _ptr(res), _sp()), SolveException)
    barrier.n_update += 1
    return Array(view(res, 2:2))[1]                    # B2_QF_MU
end

function MadNLP.get_adaptive_mu(solver::B200RRSolver{T}, barrier::MadNLP.LOQOUpdate{T}) where T
    MadNLP.get_nlb(solver) + MadNLP.get_nub(solver) == 0 && return barrier.mu_min
    kkt = MadNLP.get_kkt(solver)
    v = map(MadNLP.full, (MadNLP.get_x(solver), MadNLP.get_xl(solver), MadNLP.get_xu(solver), MadNLP.get_zl(solver), MadNLP.get_zu(solver)))
    mu = _reduce(kkt, :b2_get_average_complementarity, ntuple(_ -> _V, 5), map(_ptr, v)...)
    min_cc = _reduce(kkt, :b2_get_min_complementarity, ntuple(_ -> _V, 5), map(_ptr, v)...)
    xi = min_cc / mu
    sigma = barrier.gamma * min((1 - barrier.r) * ((1 - xi) / xi), 2)^3
    return clamp(sigma * mu, barrier.mu_min, barrier.mu_max)
end

end # module
