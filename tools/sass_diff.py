#!/usr/bin/env python
"""Compare the SASS of two builds of libb200kkt.so kernel by kernel.

    python tools/sass_diff.py old/libb200kkt.so new/libb200kkt.so

Each kernel's instructions come from `cuobjdump -sass`, without addresses and encodings, and with the per-build hashes of
anonymous-namespace names (`_GLOBAL__N__<hash>_<len>_<file>_<hash>`) removed.  Prints the kernels found in only one build and those
whose instructions differ; exits 1 if there are any.
"""
import os
import re
import subprocess
import sys

ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_(\d+_.+?)_[0-9a-f]{8}(?=\d)")
ADDR = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s*")
ENC = re.compile(r"\s*/\* 0x[0-9a-f]{16} \*/\s*$")


def kernels(lib):
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", lib], check=True, capture_output=True, text=True).stdout
    out, name = {}, None
    for line in ANON.sub(r"_GLOBAL__N__\1", text).splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            while name in out:                    # (the same kernel compiled into two translation units)
                name += "'"
            out[name] = []
        elif name is not None and ADDR.match(line):
            out[name].append(ENC.sub("", ADDR.sub("", line)).strip())
    return out


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    only_a, only_b = sorted(a.keys() - b.keys()), sorted(b.keys() - a.keys())
    both = sorted(a.keys() & b.keys())
    diff = [k for k in both if a[k] != b[k]]
    for k in only_a:
        print(f"only in {sys.argv[1]}: {k}")
    for k in only_b:
        print(f"only in {sys.argv[2]}: {k}")
    for k in diff:
        print(f"differs ({len(a[k])} -> {len(b[k])} instructions): {k}")
    print(f"{len(a)} / {len(b)} kernels, {len(both)} matched, {len(diff)} differing")
    sys.exit(1 if only_a or only_b or diff else 0)


if __name__ == "__main__":
    main()
