"""Source checks of the CUDA headers (CPU; needs nvcc, which cross-compiles for sm_90a without a device): every header compiles
on its own, and the inline-PTX primitives are written in csrc/ptx.cuh only."""
import concurrent.futures as cf
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "madnlp.jl_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
HEADERS = sorted(os.path.basename(p) for p in glob.glob(os.path.join(CSRC, "*.cuh")))

# instructions that belong in ptx.cuh, and the inline uses that stay with their one kernel
PRIMITIVES = ("mbarrier.", "cp.async", "ld.acquire", "ld.relaxed", "st.release", "st.relaxed", "rcp.approx", "griddepcontrol",
              "%globaltimer", "%smid")
ALLOWED = {
    ("warp_kernels.cuh", "rcp.approx.ftz.f64"): "pivot_iter's reciprocal, interleaved with the pending update (B2_TIE)",
    ("ozaki_kernels.cuh", "cp.async.bulk.tensor.3d"): "the TMA tensor load of the Ozaki SYRK",
}


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_every_header_compiles_alone(tmp_path):
    def compile_one(h):
        tu = tmp_path / (h + ".cu")
        tu.write_text(f'#include "{h}"\n')
        r = subprocess.run([NVCC, "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                            "-I", CSRC, "-c", str(tu), "-o", str(tmp_path / (h + ".o"))], capture_output=True, text=True)
        return h, r.returncode, r.stderr

    assert len(HEADERS) >= 12
    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        failed = [(h, err) for h, rc, err in ex.map(compile_one, HEADERS) if rc != 0]
    assert not failed, "\n".join(f"{h}:\n{err}" for h, err in failed)


_TOKEN = re.compile(r'"(?:\\.|[^"\\\n])*"|//[^\n]*|/\*.*?\*/', re.S)


def _asm_strings(src):
    """the string literals inside each asm(...) statement of a C++ source, comments removed"""
    strings = [(m.start(), m.group()[1:-1]) for m in _TOKEN.finditer(src) if m.group().startswith('"')]
    bare = _TOKEN.sub(lambda m: " " * len(m.group()), src)      # same offsets, no strings or comments
    out = []
    for m in re.finditer(r"\basm\s*(?:volatile\s*)?\(", bare):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(bare[i], 0)
            i += 1
        out.append("".join(s for pos, s in strings if m.end() <= pos < i))
    return out


def test_ptx_primitives_live_in_ptx_cuh():
    stray, allowed_seen = [], set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        name = os.path.basename(path)
        if name == "ptx.cuh":
            continue
        for asm in _asm_strings(open(path).read()):
            hits = [p for p in PRIMITIVES if p in asm]
            if not hits:
                continue
            key = next(((f, s) for f, s in ALLOWED if f == name and s in asm), None)
            if key:
                allowed_seen.add(key)
            else:
                stray.append(f"{name}: {hits} in {asm[:80]!r}")
    assert not stray, "inline PTX primitives outside ptx.cuh:\n" + "\n".join(stray)
    assert allowed_seen == set(ALLOWED), f"stale allowlist entries: {set(ALLOWED) - allowed_seen}"
    ptx = "".join(_asm_strings(open(os.path.join(CSRC, "ptx.cuh")).read()))
    for p in PRIMITIVES:
        assert p in ptx, f"{p} is not defined in ptx.cuh"
