"""ctypes binding of the C ABI in include/b200kkt.h (libb200kkt.so, built in-tree by csrc/Makefile).

This is the same boundary a MadNLP.jl maintainer would bind with `ccall` (INTEGRATION.md); the Python host
layer above it only mirrors the reference's plugin interface.  There is NO fallback: if the shared library is
missing the import fails loudly, and every numeric entry point needs a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200kkt.so")

B2_OK = 0
B2_ERR_INVALID, B2_ERR_CUDA, B2_ERR_SYMBOLIC, B2_ERR_FACTORIZATION, B2_ERR_SOLVE, B2_ERR_NO_DEVICE, B2_ERR_UNSUPPORTED = 1, 2, 3, 4, 5, 6, 7
ORDER_METIS_ND, ORDER_MINDEG, ORDER_NATURAL, ORDER_USER = 0, 1, 2, 3
QN_BFGS, QN_DAMPED_BFGS = 1, 2
B2_DENSE_PIVOT_STATIC, B2_DENSE_PIVOT_BUNCH_KAUFMAN = 0, 1
B2_DENSE_ALG_LDLT, B2_DENSE_ALG_LU = 0, 1
B2_SPARSE_PIVOT_STATIC, B2_SPARSE_PIVOT_PAIRS = 0, 1
B2_PIVOT_1X1, B2_PIVOT_1X1_PERTURBED, B2_PIVOT_2X2_FIRST, B2_PIVOT_2X2_SECOND = 0, 1, 2, 3
# layout of b2_mul_hess_blk_tail's curvature-test result (B2_CURV_* in include/b200kkt.h)
CURV_WXT, CURV_WXN, CURV_GN, CURV_TT, CURV_LHS, CURV_PASS, CURV_RESULT_LEN = 0, 1, 2, 3, 4, 5, 6
# layout of b2_dual_init_select's result (B2_DUAL_INIT_* in include/b200kkt.h)
DUAL_INIT_NORM, DUAL_INIT_COPY, DUAL_INIT_RESULT_LEN = 0, 1, 2
# the adaptive barrier's scalar array and b2_qf_search's result (B2_QF_* in include/b200kkt.h)
QF_TAU, QF_NRM_PRIMAL, QF_NRM_DUAL, QF_MU_AVG, QF_SCAL_LEN = 0, 1, 2, 3, 4
QF_SIGMA, QF_MU, QF_N_EVAL, QF_N_GS_ITER, QF_TOL_EXIT, QF_TRACE, QF_MAX_GS_ITER = 0, 1, 2, 3, 4, 8, 64
# the Krylov iterator's state (B2_KRYLOV_* in include/b200kkt.h): offsets of y, of the record, and the record's entries
KRYLOV_MAX_RESTART, KRYLOV_Y, KRYLOV_REC, KRYLOV_REC_LEN, KRYLOV_STATE_LEN = 16, 321, 344, 8, 352
KREC_EST, KREC_H, KREC_NORM_W, KREC_NORM_X, KREC_NORM_B, KREC_NORM_B2 = 0, 1, 2, 3, 4, 5


def qf_result_len(max_gs_iter):
    return QF_TRACE + 4 * (6 + max_gs_iter)


class B2Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200kkt error {code}: {msg}")
        self.code = code


# exception types of the reference (src/LinearSolvers/linearsolvers.jl:133-137)
class SymbolicException(B2Error):
    pass


class FactorizationException(B2Error):
    pass


class SolveException(B2Error):
    pass


class InertiaException(RuntimeError):
    pass


class _Pivoting(C.Structure):
    _fields_ = [("dense_pivoting", C.c_int32), ("sparse_pivoting", C.c_int32), ("dense_algorithm", C.c_int32)]


class _OptionsTail(C.Union):
    """the three int32 after kkt_n_dual: `dense_pivoting`, `sparse_pivoting` and `dense_algorithm` (include/b200kkt.h).
    `reserved` keeps the view of all three at the offset it always had, so that code which reads `Options.reserved` still finds
    it there."""
    _anonymous_ = ("_pivoting",)
    _fields_ = [("_pivoting", _Pivoting), ("reserved", C.c_int32 * 3)]


class Options(C.Structure):
    _anonymous_ = ("_tail",)
    _fields_ = [
        ("ordering", C.c_int32), ("nemin", C.c_int32), ("relax_zeros", C.c_double), ("pivot_eps", C.c_double),
        ("use_cuda_graph", C.c_int32), ("small_front_max", C.c_int32), ("n_parts", C.c_int32), ("part_rank", C.c_int32),
        ("kkt_n_primal", C.c_int32), ("fuse_max_fronts", C.c_int32), ("dep_schedule", C.c_int32), ("chain_merge_f", C.c_int32), ("kkt_n_dual", C.c_int32),
        ("_tail", _OptionsTail),
    ]


class Stats(C.Structure):
    _fields_ = [(k, C.c_int64) for k in (
        "n", "nnz_a", "nnz_l", "flops", "n_supernodes", "n_levels", "max_front", "n_small_fronts", "n_big_fronts",
        "factor_bytes", "workspace_bytes", "sep_rows", "n_factor_launches", "n_solve_launches", "n_perturbed")]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class InertiaSource(C.Structure):
    """b2_inertia_source: where a solver's factorisation leaves its pivot counts on the device"""
    _fields_ = [("counters_d", C.c_void_p), ("n", C.c_int64), ("neg", C.c_int32 * 2), ("zero", C.c_int32 * 2), ("fail", C.c_int32),
                ("reserved", C.c_int32)]


class RefineRecord(C.Structure):
    """b2_refine_record: what one launch of a refinement-loop graph leaves in pinned host memory"""
    _fields_ = [("ratio", C.c_double), ("norm_w", C.c_double), ("norm_x", C.c_double), ("norm_b", C.c_double), ("ir", C.c_int64),
                ("steps", C.c_int64), ("num_pos", C.c_int64), ("num_zero", C.c_int64), ("num_neg", C.c_int64), ("inertia_ok", C.c_int32),
                ("fail", C.c_int32), ("seq", C.c_int64)]


class InertiaSchedule(C.Structure):
    """b2_inertia_options: the del_w schedule of inertia_correction! (MadNLP's options of these names)"""
    _fields_ = [(k, C.c_double) for k in ("first_hessian_perturbation", "min_hessian_perturbation", "max_hessian_perturbation",
                                          "perturb_inc_fact_first", "perturb_inc_fact", "perturb_dec_fact")]


TRIALS_ACCEPTED, TRIALS_FAILED, TRIALS_HANDOVER, TRIALS_FAULT = 1, 2, 3, 4


class InertiaRecord(C.Structure):
    """b2_inertia_record: what one launch of an inertia-correction graph leaves in pinned host memory"""
    _fields_ = [("status", C.c_int32), ("inertia_ok", C.c_int32), ("trials", C.c_int64), ("del_w", C.c_double),
                ("del_w_prev", C.c_double), ("del_c_prev", C.c_double), ("num_pos", C.c_int64), ("num_zero", C.c_int64),
                ("num_neg", C.c_int64), ("ir", C.c_int64), ("ratio", C.c_double), ("ir_total", C.c_int64), ("seq", C.c_int64)]


class SymbolicSizes(C.Structure):
    _fields_ = [(k, C.c_int64) for k in (
        "n", "n_supernodes", "n_rows", "n_children", "n_rel", "n_amap", "n_levels", "lval_size", "cb_size")]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"(or `make -C madnlp.jl_b200/csrc`). The GPU KKT path has no CPU fallback.")
    return C.CDLL(LIB_PATH)


lib = _load()

_p = C.c_void_p
_i32, _i64, _f64 = C.c_int32, C.c_int64, C.c_double
_PP = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); every symbol declared in include/b200kkt.h appears here
PROTOTYPES = {
    "b2_last_error": (C.c_char_p, []),
    "b2_version": (C.c_int, []),
    "b2_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "b2_options_default": (C.c_int, [C.POINTER(Options)]),
    "b2_create": (C.c_int, [_i32, _i64, _p, _p, _p, C.POINTER(Options), _p, _PP]),
    "b2_create_symbolic_only": (C.c_int, [_i32, _i64, _p, _p, C.POINTER(Options), _p, _PP]),
    "b2_destroy": (C.c_int, [_p]),
    "b2_set_values_ptr": (C.c_int, [_p, _p]),
    "b2_factorize": (C.c_int, [_p, _p]),
    "b2_inertia": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), _p]),
    "b2_inertia_enqueue": (C.c_int, [_p, _p]),
    "b2_inertia_fetch": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "b2_solve": (C.c_int, [_p, _p, _i32, _p]),
    "b2_improve": (C.c_int, [_p, C.POINTER(_i32)]),
    "b2_get_stats": (C.c_int, [_p, C.POINTER(Stats)]),
    "b2_get_perm": (C.c_int, [_p, _p]),
    "b2_exchange_buffer": (C.c_int, [_p, _PP, C.POINTER(_i64), C.POINTER(_i64)]),
    "b2_exchange_vector": (C.c_int, [_p, _PP, C.POINTER(_i64)]),
    "b2_inertia_parts": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), _p]),
    "b2_factorize_local": (C.c_int, [_p, _p]),
    "b2_factorize_top": (C.c_int, [_p, _p]),
    "b2_solve_fwd_local": (C.c_int, [_p, _p, _p]),
    "b2_solve_top": (C.c_int, [_p, _p, _p]),
    "b2_solve_bwd_local": (C.c_int, [_p, _p, _p]),
    "b2_owned_mask": (C.c_int, [_p, _p]),
    "b2_symbolic_query": (C.c_int, [_p, C.POINTER(SymbolicSizes)]),
    "b2_symbolic_export": (C.c_int, [_p] + [_p] * 13),
    "b2_symbolic_owner": (C.c_int, [_p, _p]),
    "b2_symbolic_exchange": (C.c_int, [_p, _p, C.POINTER(_i64), C.POINTER(_i64)]),
    "b2_debug_get_factor": (C.c_int, [_p, _p, _p]),
    "b2_symbolic_pairs": (C.c_int, [_p, _p]),
    "b2_get_pivot_blocks": (C.c_int, [_p, _p, _p, _p]),
    "b2_debug_profile_front": (C.c_int, [_p, _i32, _i32, _p]),
    "b2d_debug_trace": (C.c_int, [_p, _p, _i64, C.POINTER(_i64)]),
    "b2_debug_trace": (C.c_int, [_p, _p, _p, _p, _p, _i64, C.POINTER(_i64)]),
    "b2_debug_trace_solve": (C.c_int, [_p, _p, _i64, C.POINTER(_i64)]),
    "b2_debug_dep_order": (C.c_int, [_p, _p, _i64, C.POINTER(_i64)]),
    "b2d_create": (C.c_int, [_i32, _i32, _p, C.POINTER(Options), _PP]),
    "b2d_destroy": (C.c_int, [_p]),
    "b2d_factorize": (C.c_int, [_p, _p]),
    "b2d_inertia": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), _p]),
    "b2d_inertia_enqueue": (C.c_int, [_p, _p]),
    "b2d_inertia_fetch": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "b2d_solve": (C.c_int, [_p, _p, _i32, _p]),
    "b2d_get_pivots": (C.c_int, [_p, _p, _p, _p]),
    "b2d_get_lu": (C.c_int, [_p, _p, _p, _p]),
    "b2_condensed_symbolic_device": (C.c_int, [_i32, _i32, _p, _p, _p, _p, _PP, C.POINTER(_i64), _p]),
    "b2_coo_to_csc_device": (C.c_int, [_i32, _i32, _i64, _p, _p, _p, _p, _p, C.POINTER(_i64), _p]),
    "b2d_ozaki_plan_create": (C.c_int, [_i32, _i32, _PP]),
    "b2d_ozaki_plan_destroy": (C.c_int, [_p]),
    "b2d_condensed_assemble_ozaki": (C.c_int, [_p, _i32, _i32, _i32, _i32] + [_p] * 9),
    "b2d_ozaki_plan_status": (C.c_int, [_p, C.POINTER(_i32), _p]),
    "b2d_kkt_create": (C.c_int, [_i32, _i32, _i32, _p, _PP]),
    "b2d_kkt_destroy": (C.c_int, [_p]),
    "b2d_kkt_solve_pre": (C.c_int, [_p] * 10 + [_p]),
    "b2d_kkt_solve_post": (C.c_int, [_p] * 12 + [_p]),
    "b2d_kkt_mul": (C.c_int, [_p] * 10 + [_f64, _f64, _p, _p, _p]),
    "b2d_gemv_n": (C.c_int, [_i32, _i32, _i32, _p, _p, _p, _f64, _f64, _p]),
    "b2d_gemv_t": (C.c_int, [_i32, _i32, _i32, _p, _p, _p, _f64, _f64, _p]),
    "b2d_symv_lower": (C.c_int, [_i32, _i32, _p, _p, _p, _f64, _f64, _p]),
    "b2_coo_to_csc": (C.c_int, [_i32, _i32, _i64, _p, _p, _p, _p, _p, C.POINTER(_i64)]),
    "b2_transfer_plan_create": (C.c_int, [_i64, _i64, _p, _PP]),
    "b2_transfer_plan_destroy": (C.c_int, [_p]),
    "b2_transfer": (C.c_int, [_p, _p, _p, _p]),
    "b2_condensed_symbolic": (C.c_int, [_i32, _i32, _p, _p, _p, _p, _PP, C.POINTER(_i64)]),
    "b2_condensed_pattern": (C.c_int, [_p, _p, _p]),
    "b2_condensed_plan_sizes": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "b2_condensed_plan_destroy": (C.c_int, [_p]),
    "b2_condensed_assemble": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p]),
    "b2d_condensed_assemble": (C.c_int, [_i32, _i32, _i32, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b2d_aug_assemble": (C.c_int, [_i32, _i32, _i32] + [_p] * 8),
    "b2d_copy_diag": (C.c_int, [_i32, _i32, _p, _p, _p]),
    "b2_bounds_create": (C.c_int, [_i64, _i64, _i64, _p, _p, _PP]),
    "b2_bounds_destroy": (C.c_int, [_p]),
    "b2_set_aug_diagonal": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_set_aug_diagonal_unreduced": (C.c_int, [_i64, _i64, _i64] + [_p] * 7),
    "b2_unreduced_solve_pre": (C.c_int, [_i64, _i64, _i64, _i64, _p, _p, _p, _p]),
    "b2_unreduced_solve_post": (C.c_int, [_i64, _i64, _i64, _i64, _p, _p, _p, _p]),
    "b2_regularize_diagonal": (C.c_int, [_i64, _i64, _f64, _f64, _p, _p, _p, _p]),
    "b2_scaled_set_aug_diagonal": (C.c_int, [_p] + [_p] * 7 + [_p]),
    "b2_scaled_transfer": (C.c_int, [_p, _i64, _i64, _p, _p, _p, _p, _p, _p]),
    "b2_scaled_solve_pre": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "b2_scaled_solve_post": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p, _p]),
    "b2_scaled_kktmul": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p, _p]),
    "b2_scaled_regularize_diagonal": (C.c_int, [_i64, _i64, _f64, _f64, _p, _p, _p, _p, _p]),
    "b2_reduce_rhs": (C.c_int, [_p, _i64, _p, _p, _p, _p]),
    "b2_finish_aug_solve": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p]),
    "b2_spmv_plan_create": (C.c_int, [_i32, _i32, _p, _p, _PP]),
    "b2_spmv_plan_destroy": (C.c_int, [_p]),
    "b2_spmv_n": (C.c_int, [_p, _p, _p, _p, _f64, _f64, _p]),
    "b2_spmv_t": (C.c_int, [_p, _p, _p, _p, _f64, _f64, _p]),
    "b2_spmv_symlower": (C.c_int, [_p, _p, _p, _p, _f64, _f64, _p]),
    "b2_kktmul": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p, _p]),
    "b2_condensed_solve_pre": (C.c_int, [_p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_condensed_solve_post": (C.c_int, [_p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_condensed_kkt_mul": (C.c_int, [_p, _p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p, _p]),
    "b2_condensed_kkt_mul_norm": (C.c_int, [_p, _p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p, _p, _p]),
    "b2_condensed_refine_pre": (C.c_int, [_p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_condensed_solve_post_update": (C.c_int, [_p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_condensed_kkt_mul_norm_y": (C.c_int, [_p, _p, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p, _p, _p, _p]),
    "b2_get_alpha_max": (C.c_int, [_p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_get_alpha_z": (C.c_int, [_p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_get_varphi": (C.c_int, [_p, _f64, _p, _p, _p, _f64, _p, _p]),
    "b2_get_varphi_d": (C.c_int, [_p, _p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_get_inf_du": (C.c_int, [_p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_get_inf_compl": (C.c_int, [_p, _p, _p, _p, _p, _p, _f64, _f64, _p, _p]),
    "b2_get_average_complementarity": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_get_min_complementarity": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p]),
    "b2_get_rel_search_norm": (C.c_int, [_p, _i64, _p, _p, _p, _p]),
    "b2_get_sd": (C.c_int, [_p, _i64, _p, _p, _p, _f64, _p, _p]),
    "b2_get_sc": (C.c_int, [_p, _p, _p, _f64, _p, _p]),
    "b2_set_aug_rhs": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_set_g_ifr": (C.c_int, [_i64, _p, _p, _p, _p, _p, _f64, _p, _p]),
    "b2_set_aug_rhs_ifr": (C.c_int, [_i64, _i64, _i64, _i64, _p, _p, _p]),
    "b2_mul_hess_blk_tail": (C.c_int, [_p, _i64, _i32] + [_p] * 9 + [_f64, _p, _p]),
    "b2_rr_init": (C.c_int, [_p, _i64, _p, _p, _f64, _f64] + [_p] * 10 + [_p]),
    "b2_set_aug_rr": (C.c_int, [_p, _i64, _f64, _f64, _f64] + [_p] * 16 + [_p]),
    "b2_set_aug_rr_scaled": (C.c_int, [_p, _i64, _f64, _f64, _f64] + [_p] * 16 + [_p]),
    "b2_set_aug_rhs_rr": (C.c_int, [_p, _i64] + [_p] * 13 + [_f64, _f64, _p, _p]),
    "b2_finish_aug_solve_rr": (C.c_int, [_i64] + [_p] * 6 + [_f64, _f64] + [_p] * 4 + [_p]),
    "b2_set_f_rr": (C.c_int, [_i64, _f64, _p, _p, _p, _p, _p]),
    "b2_reset_bound_dual": (C.c_int, [_i64, _p, _p, _f64, _f64, _p]),
    "b2_reset_bound_dual_lu": (C.c_int, [_p] + [_p] * 5 + [_f64, _f64, _p]),
    "b2_adjust_boundary": (C.c_int, [_p, _p, _p, _p, _f64, _p]),
    "b2_get_theta": (C.c_int, [_p, _i64, _p, _p, _p]),
    "b2_get_theta_r": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "b2_get_inf_pr_r": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "b2_get_obj_val_r": (C.c_int, [_p, _i64] + [_p] * 5 + [_f64, _f64, _p, _p]),
    "b2_get_inf_du_r": (C.c_int, [_p, _i64] + [_p] * 7 + [_f64, _f64, _p, _p]),
    "b2_get_inf_compl_r": (C.c_int, [_p, _i64] + [_p] * 9 + [_f64, _f64, _p, _p]),
    "b2_get_alpha_max_r": (C.c_int, [_p, _i64] + [_p] * 8 + [_f64, _p, _p]),
    "b2_get_alpha_z_r": (C.c_int, [_p, _i64] + [_p] * 8 + [_f64, _p, _p]),
    "b2_get_varphi_r": (C.c_int, [_p, _i64, _f64] + [_p] * 5 + [_f64, _p, _p]),
    "b2_get_varphi_d_r": (C.c_int, [_p, _i64] + [_p] * 9 + [_f64, _f64, _p, _p]),
    "b2_set_aug_diagonal_iterate": (C.c_int, [_p, _i64, _f64, _f64] + [_p] * 11 + [_p]),
    "b2_set_aug_diagonal_iterate_scaled": (C.c_int, [_p, _i64, _f64, _f64] + [_p] * 11 + [_p]),
    "b2_set_aug_rhs_perturbed": (C.c_int, [_p, _i64] + [_p] * 9 + [_f64, _f64, _f64, _i64, _p, _i64, _p, _p, _p]),
    "b2_set_initial_rhs": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "b2_dual_init_select": (C.c_int, [_p, _i64, _p, _i32, _f64, _p, _p, _p]),
    "b2_get_pd_error": (C.c_int, [_p, _i64] + [_p] * 8 + [_f64, _p, _p]),
    "b2_restore_update": (C.c_int, [_p, _i64] + [_p] * 11 + [_p]),
    "b2_soc_trial": (C.c_int, [_i64, _p, _p, _p, _p, _p]),
    "b2_primal_dual_norm2": (C.c_int, [_p, _i64, _p, _p, _p]),
    "b2_set_centering_aug_rhs": (C.c_int, [_p, _i64, _i64, _p, _i64, _p, _p, _f64, _p, _p]),
    "b2_qf_search": (C.c_int, [_p, _i64] + [_p] * 8 + [_f64] * 5 + [_i32, _p, _p]),
    "b2_richardson_begin": (C.c_int, [_i64, _p, _p, _p, _p, _p]),
    "b2_richardson_update": (C.c_int, [_i64, _p, _p, _p, _p, _p]),
    "b2_copy_many": (C.c_int, [_i32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(_i64), _p]),
    "b2_norm_inf": (C.c_int, [_i64, _p, _p, _p]),
    "b2_axpy": (C.c_int, [_i64, _f64, _p, _p, _p]),
    "b2_copy": (C.c_int, [_i64, _p, _p, _p]),
    "b2_fill": (C.c_int, [_i64, _f64, _p, _p]),
    "b2_lbfgs_create": (C.c_int, [_i64, _i32, _i32, _f64, _f64, _f64, _PP]),
    "b2_lbfgs_destroy": (C.c_int, [_p]),
    "b2_lbfgs_state": (C.c_int, [_p, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_f64), _p]),
    "b2_lbfgs_init": (C.c_int, [_p, _p, _p, _f64, _p]),
    "b2_lbfgs_update": (C.c_int, [_p, _p, _p, _p, _p]),
    "b2_lbfgs_smw_prepare": (C.c_int, [_p, _p, _i64, _p, _p]),
    "b2_lbfgs_smw_apply": (C.c_int, [_p, _i64, _p, _p, _p]),
    "b2_lbfgs_kkt_mul_lowrank": (C.c_int, [_p, _f64, _p, _p, _p]),
    "b2_lbfgs_debug_get": (C.c_int, [_p, _i32, _p, C.POINTER(_i64), _p]),
    "b2_lbfgs_debug_ipiv": (C.c_int, [_p, _p, _p]),
    "b2_debug_bk_factor": (C.c_int, [_i32, _p, _p, _p]),
    "b2_debug_bk_solve": (C.c_int, [_i32, _p, _p, _p, _p]),
    "b2d_qn_create": (C.c_int, [_i64, _i32, _PP]),
    "b2d_qn_destroy": (C.c_int, [_p]),
    "b2d_qn_init": (C.c_int, [_p, _p, _p, _f64, _p]),
    "b2d_qn_update": (C.c_int, [_p, _p, _p, _p, _p]),
    "b2d_qn_rank2": (C.c_int, [_p, _p, _p, _p]),
    "b2d_qn_state": (C.c_int, [_p, C.POINTER(_i32), C.POINTER(_i32), _p, _p]),
    "b2d_qn_debug_vectors": (C.c_int, [_p, _p, _p, _p]),
    "b2_krylov_create": (C.c_int, [_i64, _i32, _PP]),
    "b2_krylov_destroy": (C.c_int, [_p]),
    "b2_krylov_buffers": (C.c_int, [_p, _PP, _PP, _PP]),
    "b2_krylov_begin": (C.c_int, [_p, _i32, _p, _p, _p, _p]),
    "b2_krylov_scale": (C.c_int, [_p, _i32, _p, _p]),
    "b2_krylov_orthogonalize": (C.c_int, [_p, _i32, _p, _p]),
    "b2_krylov_close": (C.c_int, [_p, _i32, _p, _p, _p, _p]),
    "b2_inertia_source_get": (C.c_int, [_p, C.POINTER(InertiaSource)]),
    "b2_refine_loop_create": (C.c_int, [_PP]),
    "b2_refine_loop_destroy": (C.c_int, [_p]),
    "b2_refine_loop_begin": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "b2_refine_loop_end": (C.c_int, [_p, C.POINTER(InertiaSource), _i64, _i64, _i32, _f64, _p]),
    "b2_refine_loop_launch": (C.c_int, [_p, _p]),
    "b2_refine_loop_wait": (C.c_int, [_p]),
    "b2_refine_loop_record": (C.c_int, [_p, C.POINTER(RefineRecord)]),
    "b2_inertia_trial_bound": (C.c_int, [C.POINTER(InertiaSchedule), C.POINTER(_i64)]),
    "b2_inertia_loop_create": (C.c_int, [C.POINTER(InertiaSchedule), _PP]),
    "b2_inertia_loop_destroy": (C.c_int, [_p]),
    "b2_inertia_loop_begin": (C.c_int, [_p, _i64, _i64, _p, _p, _p, _i32, _p]),
    "b2_inertia_loop_begin_scaled": (C.c_int, [_p, _i64, _i64, _p, _p, _p, _p, _i32, _p]),
    "b2_inertia_loop_refine": (C.c_int, [_p, C.POINTER(InertiaSource), _i64, _i64, _i64, _p, _p, _p, _p, _p]),
    "b2_inertia_loop_end": (C.c_int, [_p, _i32, _f64, _f64, _p]),
    "b2_inertia_loop_launch": (C.c_int, [_p, _f64, _f64, _i64, _p]),
    "b2_inertia_loop_wait": (C.c_int, [_p]),
    "b2_inertia_loop_record": (C.c_int, [_p, C.POINTER(InertiaRecord), _p, _i64]),
}

for _name, (_res, _args) in PROTOTYPES.items():
    _fn = getattr(lib, _name)          # AttributeError here = header/library mismatch: fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


def last_error() -> str:
    return (lib.b2_last_error() or b"").decode()


_EXC = {B2_ERR_SYMBOLIC: SymbolicException, B2_ERR_FACTORIZATION: FactorizationException, B2_ERR_SOLVE: SolveException}


def check(rc: int):
    if rc != B2_OK:
        raise _EXC.get(rc, B2Error)(rc, last_error())


def device_count() -> int:
    n = C.c_int(0)
    rc = lib.b2_device_count(C.byref(n))
    return n.value if rc == B2_OK else 0


def require_device():
    if device_count() == 0:
        raise B2Error(B2_ERR_NO_DEVICE, "no CUDA device visible; the GPU KKT path has no CPU fallback")


def default_options(**kw) -> Options:
    o = Options()
    check(lib.b2_options_default(C.byref(o)))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise TypeError(f"unknown b2 option {k!r}")
        setattr(o, k, v)
    return o


def ptr(t):
    """device/host pointer of a torch tensor or numpy array (or None)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def copy_many(pairs, stream=None):
    """b2_copy_many: copy every (src, dst) pair of float64 device tensors of one length each in ONE launch; at most 16 pairs (the
    entry refuses more)."""
    n = len(pairs)
    src = (C.c_void_p * n)(*[s.data_ptr() for s, _ in pairs])
    dst = (C.c_void_p * n)(*[d.data_ptr() for _, d in pairs])
    ns = (C.c_int64 * n)(*[d.numel() for _, d in pairs])
    check(lib.b2_copy_many(n, src, dst, ns, stream_ptr(stream)))


def stream_ptr(stream=None):
    if stream is None:
        import torch
        return torch.cuda.current_stream().cuda_stream
    return getattr(stream, "cuda_stream", stream)
