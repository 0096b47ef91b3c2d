#!/usr/bin/env python
"""Compares the SASS of the chaining kernels in two builds of csrc/chain.cu, ignoring symbol names.  Every kernel of the first
object must have a twin in the second with the same instructions.  The second build's instantiations whose cDNA template argument
is true (spliced chaining) are skipped, so the check says whether the non-cDNA kernels are still the same code.

  nvcc -gencode arch=compute_90a,code=sm_90a <the flags of winnowmap_b200/build.py> -x cu -c csrc/chain.cu -o new.o   (old.o likewise)
  python tools/compare_sass.py old.o new.o

Exits 1 when a kernel differs or has no twin."""
import re
import subprocess
import sys


def kernels(obj):
    """{mangled name: instruction lines} of an object's SASS."""
    txt = subprocess.check_output(["/usr/local/cuda/bin/cuobjdump", "-sass", obj], text=True)
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur and re.search(r"/\*[0-9a-f]{4}\*/", line):
            out[cur].append(re.sub(r"\b\w*_Z\w+", "SYM", line.strip()))
    return out


def key(mangled):
    """The demangled kernel name with its template arguments but without the cDNA flag and the parameter list."""
    d = subprocess.check_output(["c++filt", mangled], text=True).strip()
    d = re.sub(r"\(.*\)$", "", d).replace(", false>", ">").replace("<false>", "")
    return re.sub(r"^void ", "", d), "true>" in d


def main():
    old = {key(n)[0]: v for n, v in kernels(sys.argv[1]).items()}
    new = {}
    for n, v in kernels(sys.argv[2]).items():
        k, cdna = key(n)
        if not cdna:
            new[k] = v
    ok = True
    for k in sorted(set(old) | set(new)):
        if k not in old or k not in new:
            print(f"no twin: {k} (in old: {k in old}, in new: {k in new})")
            ok = False
            continue
        same = old[k] == new[k]
        print(f"{'same' if same else 'DIFFERENT'} {len(old[k])} instructions {k}")
        ok &= same
    print("all kernels identical" if ok else "kernels differ")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
