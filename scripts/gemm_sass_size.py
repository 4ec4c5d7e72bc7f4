#!/usr/bin/env python
"""SASS size of every gemm_tc_kernel instantiation: instructions and BRA instructions per kernel, from `cuobjdump -sass`
of the built objects (run `python -m gligen_b200.build` first; nvcc's cuobjdump and c++filt are used, no GPU).

    python scripts/gemm_sass_size.py [OBJ ...]        # default: gligen_b200/_build/gemm_tc*.o

One line per kernel: kind, <BN, GEGLU, CTA2, PP>, instructions, BRAs.  The epilogue is unrolled over the whole tile, so
these counts follow its length (DESIGN §5)."""
from __future__ import annotations

import glob
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
INSN = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")


def demangle(names):
    if not shutil.which("c++filt"):
        return names
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    return r.stdout.splitlines()


def sass_counts(obj):
    """{mangled kernel name: (instructions, BRAs)} of the gemm_tc_kernel functions in one object."""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    counts, name = {}, None
    for line in out.splitlines():
        if "Function : " in line:
            name = line.split("Function : ", 1)[1].strip()
            if "gemm_tc_kernel" not in name:
                name = None
            else:
                counts[name] = [0, 0]
            continue
        if name is None:
            continue
        m = INSN.search(line)
        if m:
            counts[name][0] += 1
            counts[name][1] += m.group(2) == "BRA"
    return counts


def main(argv):
    objs = argv or sorted(glob.glob(os.path.join(ROOT, "gligen_b200", "_build", "gemm_tc*.o")))
    if not objs:
        sys.exit("no objects: run `python -m gligen_b200.build` first")
    rows = {}
    for obj in objs:
        rows.update(sass_counts(obj))
    names = demangle(list(rows))
    table = []
    for (mangled, (n, bra)), name in zip(rows.items(), names):
        m = re.search(r"glg::(?:(\w+)::)?gemm_tc_kernel<([^>]*)>", name)
        kind, tmpl = (m.group(1) or "-", m.group(2).replace(" ", "")) if m else ("?", name)
        table.append((tmpl, kind, n, bra))
    table.sort(key=lambda r: (r[0], r[1]))
    print(f"{'<BN,GEGLU,CTA2,PP>':<24} {'kind':<26} {'instructions':>12} {'BRA':>6}")
    for tmpl, kind, n, bra in table:
        print(f"{tmpl:<24} {kind:<26} {n:>12} {bra:>6}")


if __name__ == "__main__":
    main(sys.argv[1:])
