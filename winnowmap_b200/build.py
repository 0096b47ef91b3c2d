"""Builds winnowmap_b200/libwinnowmap_b200.so (CUDA kernels + C ABI) in-tree with nvcc for
sm_90a (H100), and next to it the command-line executable winnowmap_b200/winnowmap-b200, which finds the .so through an
$ORIGIN rpath.  No JIT cache: both are built once by build() and loaded from the tree."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libwinnowmap_b200.so")
EXE = os.path.join(HERE, "winnowmap-b200")
EXE_SRC = os.path.join(HERE, "cli", "main.c")
NVCC = os.environ.get("WM_NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# -fmad=false: the reference is built without FMA contraction (Makefile:4); chaining and the
# minimizer weights use double/float expressions whose roundings must match.
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-fmad=false", "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fopenmp",
         "-ccbin", "/usr/bin/g++", "-Xptxas", "-v"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


def needs_build():
    if not os.path.exists(SO) or not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(SO), os.path.getmtime(EXE_SRC)):
        return True
    t = os.path.getmtime(SO)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src) + ".o")
        objs.append(obj)
        if (not force) and os.path.exists(obj) and os.path.getmtime(obj) > max(
                [os.path.getmtime(src)] + [os.path.getmtime(h) for h in glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))]):
            continue
        cmd = [NVCC] + ARCH + FLAGS + ["-x", "cu", "-dc" if False else "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(HERE, "build", "ptxas.log"), "a") as f:
        f.write("\n".join(log))
    if verbose:
        sys.stderr.write("\n".join(log))
    cmd = [NVCC] + ARCH + ["-shared", "-o", SO] + objs + ["-ccbin", "/usr/bin/g++", "-lpthread", "-lz", "-lgomp"]
    subprocess.check_call(cmd)
    build_exe()
    return SO


def build_exe():
    """winnowmap_b200/winnowmap-b200: main() only calls wm_cli_main of the .so beside it"""
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-I", os.path.join(HERE, "..", "include"), EXE_SRC, "-o", EXE, "-L", HERE,
                           "-lwinnowmap_b200", "-Wl,-rpath,$ORIGIN"])


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
