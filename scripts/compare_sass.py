#!/usr/bin/env python
"""Compare the device code of one CUDA source file in two source trees, kernel by kernel, without a GPU.

Each side is compiled for sm_90a as the library is (-O3, -Xptxas -v, one cubin).  For every kernel the
`cuobjdump -sass` body and ptxas's register / shared-memory / spill report must be identical on both sides; kernels
present on one side only are listed.  --rename OLD NEW rewrites the old side's demangled names (Python regex
substitution) so that a renamed kernel is compared with its new name.  Exit status 0 when everything matches.

For example, the change that made K3's walk a template parameter (k3_heap_cat<T,B,C,G> -> k3_heap<T,B,C,G,1>):

    git archive <parent> variantcalling_b200/csrc include | tar -x -C /tmp/parent
    python scripts/compare_sass.py /tmp/parent/variantcalling_b200/csrc variantcalling_b200/csrc \\
        --rename 'k3_(heap|infer)_cat<([^>]*)>' 'k3_\\1<\\2, (int)1>' \\
        --rename 'k3_heap<((?:\\(int\\)\\d+, ){3}\\(int\\)\\d+)>' 'k3_heap<\\1, (int)0>' \\
        --rename 'k3_infer<(\\(int\\)\\d+)>' 'k3_infer<\\1, (int)0>'
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin"]


def demangle(names):
    out = subprocess.run([os.path.join(CUDA, "bin", "cu++filt")], input="\n".join(names), capture_output=True,
                         text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def kernels(csrc, source, tmp, renames):
    """name -> (sass body, ptxas resource report) of every kernel in csrc/source."""
    cubin = os.path.join(tmp, "k.cubin")
    r = subprocess.run([os.path.join(CUDA, "bin", "nvcc"), *FLAGS, source, "-o", cubin], cwd=csrc, capture_output=True,
                       text=True)
    if r.returncode:
        sys.exit(r.stderr)
    report, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            report[cur] = []
        elif cur and re.search(r"stack frame|Used \d+ registers", line):
            report[cur].append(line.split(":", 1)[-1].strip())
    names = demangle(list(report))
    sass = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    bodies = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        head, _, body = chunk.partition("\n")
        bodies[head.strip()] = body
    out = {}
    for mangled, res in report.items():
        name = names[mangled]
        for old, new in renames:
            name = re.sub(old, new, name)
        out[name] = (bodies[mangled], res)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("old_csrc")
    ap.add_argument("new_csrc")
    ap.add_argument("--source", default="kernels.cu")
    ap.add_argument("--rename", nargs=2, action="append", default=[], metavar=("OLD", "NEW"))
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        old = kernels(os.path.abspath(a.old_csrc), a.source, tmp, a.rename)
        new = kernels(os.path.abspath(a.new_csrc), a.source, tmp, [])
    bad = 0
    for name in sorted(set(old) | set(new)):
        if name not in new or name not in old:
            print(f"only in {'old' if name in old else 'new'}: {name}")
            bad += 1
        elif old[name] != new[name]:
            what = "sass" if old[name][0] != new[name][0] else f"resources {old[name][1]} -> {new[name][1]}"
            print(f"differs ({what}): {name}")
            bad += 1
        else:
            print(f"identical: {name}  [{'; '.join(new[name][1])}]")
    print(f"{len(old)} old kernels, {len(new)} new kernels, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
