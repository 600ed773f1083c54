"""madnlp.jl_b200 -- H100-native KKT hot path for MadNLP-style interior-point solvers.

Only what the hot path needs lives here (SURVEY.md section 8):
  csrc/           hand-written sm_90a CUDA kernels + the C ABI (include/b200kkt.h) -> libb200kkt.so
  capi.py         ctypes binding of that ABI (the same boundary Julia would `ccall`)
  linear_solvers  mirror of MadNLP's AbstractLinearSolver surface (B200SparseSolver, B200DenseSolver)
  kkt             mirror of the AbstractKKTSystem surface (SparseKKTSystem, SparseUnreducedKKTSystem,
                  SparseCondensedKKTSystem, DenseCondensedKKTSystem, DenseKKTSystem, UnreducedKKTVector), and
                  SolverVectors, the one holder of the solver's iterate on the device
  quasi_newton    ExactHessian / CompactLBFGS (the device L-BFGS state SparseKKTSystem uses) / BFGS / DampedBFGS (the
                  device dense quasi-Newton states of DenseKKTSystem and DenseCondensedKKTSystem)
  richardson, ipm the refinement loop and the `regular!` call-order replay used for the IPM-level metric, with the
                  InertiaBased (default), InertiaFree and InertiaIgnore regularisations
  krylov          KrylovIterator: restarted GMRES refinement preconditioned on the right by the KKT solve (ipm's
                  `iterator = "KrylovIterator"`)
  capture         the eager -> capture -> replay rule every CUDA graph of the host layer follows
  restoration     RobustRestorer: the feasibility restoration phase's state, kernels and reductions on the device
  barrier         the barrier update rules; AdaptiveBarrier: the quality-function and LOQO rules' new mu on the device
  workloads       synthetic generators for the configurations named in BASELINE.json
  julia/          the Julia shim a MadNLP.jl maintainer would add (cannot be run in this image)

Importing this package requires the built shared library; there is no CPU fallback.
"""
from . import capi  # noqa: F401  (fails loudly if libb200kkt.so is missing)
from . import workloads  # noqa: F401


def __getattr__(name):
    # torch-dependent modules are imported lazily so that CPU-only tooling (ABI checks, symbolic analysis)
    # does not pay for `import torch`.
    import importlib
    if name in ("kkt", "linear_solvers", "quasi_newton", "richardson", "krylov", "ipm", "parallel", "restoration", "barrier",
                "capture"):
        return importlib.import_module(f".{name}", __name__)
    raise AttributeError(name)
