"""CPU checks of the inertia-correction graph's host side (csrc/inertia_loop.cu): the ctypes mirrors of b2_inertia_record and
b2_inertia_options have the header's layout, and the trial bound that sizes the del_w list is never below the number of trials the
host schedule (IPMLinearAlgebra._trials_from) can take."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import madnlp_jl_b200 as pkg
from madnlp_jl_b200.ipm import InertiaOptions, inertia_trial_bound

capi = pkg.capi
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CC = shutil.which("cc") or shutil.which("gcc")


@pytest.mark.skipif(CC is None, reason="no C compiler")
@pytest.mark.parametrize("struct, cls", [("b2_inertia_record", capi.InertiaRecord), ("b2_inertia_options", capi.InertiaSchedule)])
def test_struct_layout_matches_the_header(tmp_path, struct, cls):
    fields = [name for name, _ in cls._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200kkt.h"\nint main(void) {\n'
                   f'    printf("%zu\\n", sizeof({struct}));\n'
                   + "".join(f'    printf("%zu\\n", offsetof({struct}, {f}));\n' for f in fields) + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([CC, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(cls)] + [getattr(cls, f).offset for f in fields]


def _host_trials(o, del_w_last):
    """the number of regularised trials of IPMLinearAlgebra._trials_from when no trial is accepted"""
    trials = 0
    del_w = 0.0
    while True:
        if trials == 0:
            del_w = o.first_hessian_perturbation if del_w_last == 0.0 else max(o.min_hessian_perturbation, o.perturb_dec_fact * del_w_last)
        else:
            del_w *= o.perturb_inc_fact_first if del_w_last == 0.0 else o.perturb_inc_fact
            if del_w > o.max_hessian_perturbation:
                return trials
        trials += 1


@pytest.mark.parametrize("opts", [{}, dict(max_hessian_perturbation=1.0), dict(perturb_inc_fact=1.5, min_hessian_perturbation=1e-12),
                                  dict(first_hessian_perturbation=1e-30, perturb_inc_fact_first=3.0),
                                  dict(max_hessian_perturbation=1e-25)])
def test_trial_bound_covers_the_host_schedule(opts):
    o = InertiaOptions(**opts)
    bound = inertia_trial_bound(o)
    worst = 0
    for del_w_last in (0.0, 1e-300, 1e-21, 3e-20, 1e-8, 0.5, 7.0, 1e10, 1e30):
        n = _host_trials(o, del_w_last)
        assert n <= bound, (del_w_last, n, bound)
        worst = max(worst, n)
    # from min_hessian_perturbation with the smaller factor the bound is reached: del_w_last so small that the first del_w is the minimum
    if o.min_hessian_perturbation <= o.first_hessian_perturbation and o.perturb_inc_fact <= o.perturb_inc_fact_first:
        assert worst == bound


@pytest.mark.parametrize("opts", [dict(perturb_inc_fact=1.0), dict(perturb_inc_fact_first=0.5), dict(min_hessian_perturbation=0.0),
                                  dict(max_hessian_perturbation=float("inf")), dict(perturb_inc_fact=1.0 + 2.0 ** -40)])
def test_unbounded_schedule_keeps_the_host_loop(opts):
    assert inertia_trial_bound(InertiaOptions(**opts)) is None
