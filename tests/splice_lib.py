"""Test helpers of spliced mapping: the cDNA chaining of the oracle (oracle/wm_oracle_cdna.c) and of the reference
(oracle/ref_harness_cdna.cpp, where the reference's sources and oracle/_ref are present), the cDNA emulations of the chaining kernels
(tests/hostsim/splice_emul.cpp, splice_cta_emul.cpp) and the oracle-backed spliced pipeline (tests/hostsim/splice_backend.cpp).
Every library is compiled once per process into a temporary directory."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
HOSTSIM = os.path.join(ROOT, "tests", "hostsim")
CSRC = os.path.join(ROOT, "winnowmap_b200", "csrc")
PKG = os.path.join(ROOT, "winnowmap_b200")
CUDA_INC = f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include"
GXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off"]
CHAIN_ARGTYPES = [C.c_int] * 8 + [C.c_float, C.c_long, ol._u64p, ol._u64p, ol._u64p, C.POINTER(C.c_long)]
SIG = [C.c_void_p, C.c_int] + [C.c_int] * 6 + [C.c_float]

_tmp = []
_libs = {}


def _dir():
    if not _tmp:
        _tmp.append(tempfile.mkdtemp(prefix="wm_splice_"))
    return _tmp[0]


def _once(name, make):
    if name not in _libs:
        _libs[name] = make(os.path.join(_dir(), name))
    return _libs[name]


def _hostsim():
    """libwm_hostsim.so (tests/hostsim/build.sh): the fiber runtime of the software warp."""
    so = os.path.join(HOSTSIM, "libwm_hostsim.so")
    if not os.path.exists(so):
        subprocess.check_call([os.path.join(HOSTSIM, "build.sh")], stderr=subprocess.DEVNULL)
    return ["-L" + HOSTSIM, "-l:libwm_hostsim.so", "-Wl,-rpath," + HOSTSIM]


def oracle():
    def make(so):
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", os.path.join(ORACLE, "wm_oracle.c"),
                               os.path.join(ORACLE, "wm_oracle_cdna.c"), "-o", so, "-lm"])
        L = C.CDLL(so)
        L.wmo_chain_dp_cdna.argtypes = CHAIN_ARGTYPES
        return L
    return _once("libwm_oracle_cdna.so", make)


def ref():
    """The reference's mm_chain_dp(is_cdna = 1), or None where its sources ($REF, default /root/reference) or oracle/_ref are absent."""
    def make(so):
        src = os.path.join(os.environ.get("REF", "/root/reference"), "src")
        lib_a = os.path.join(ORACLE, "_ref", "libwinnowmap.a")
        if not (os.path.isdir(src) and os.path.exists(lib_a)):
            return None
        subprocess.check_call(["/usr/bin/g++", "-O2", "-fopenmp", "-std=c++11", "-w", "-fPIC", "-shared", "-DHAVE_KALLOC", "-I" + src,
                               os.path.join(ORACLE, "ref_harness_cdna.cpp"), lib_a, "-o", so, "-lm", "-lz", "-lpthread"])
        L = C.CDLL(so)
        L.ref_chain_dp_cdna.argtypes = CHAIN_ARGTYPES
        return L
    return _once("libref_harness_cdna.so", make)


def oracle_chain_cdna(a_xy, *args, **kw):
    """oracle_lib.oracle_chain with is_cdna = 1: (u, chained anchors)."""
    return ol._chain(oracle().wmo_chain_dp_cdna, a_xy, *args, **kw)


def ref_chain_cdna(a_xy, *args, **kw):
    return ol._chain(ref().ref_chain_dp_cdna, a_xy, *args, **kw)


def emul():
    def make(so):
        subprocess.check_call(GXX + ["-fvisibility=hidden", CUDA_INC, os.path.join(HOSTSIM, "splice_emul.cpp"), "-o", so] + _hostsim())
        L = C.CDLL(so)
        L.wmt_emul_chain_fill_cdna.argtypes = SIG + [C.c_int, C.c_int] + [C.c_void_p] * 3
        L.wmt_chain_fill_scalar_gap.argtypes = SIG + [C.c_int] + [C.c_void_p] * 3
        return L
    return _once("libwm_splice_emul.so", make)


def cta():
    def make(so):
        subprocess.check_call(GXX + ["-fvisibility=hidden", "-I" + CSRC, "-I" + HOSTSIM, CUDA_INC, os.path.join(HOSTSIM, "splice_cta_emul.cpp"),
                               "-o", so] + _hostsim())
        L = C.CDLL(so)
        L.wmt_tile_cta_cdna.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int,
                                        C.c_uint64] + [C.c_void_p] * 4 + [C.c_char_p, C.c_int]
        L.wmt_tile_constants_cdna.argtypes = [C.c_void_p]
        return L
    return _once("libwm_splice_cta.so", make)


def pipeline(hpc=False):
    """wmt_map_file_splice over the oracle backend (hpc: with an HPC index)."""
    def make(so):
        host = sorted(glob.glob(os.path.join(CSRC, "host_*.cpp")))
        extra = ["-DWMT_SPLICE_HPC"] if hpc else []
        oc = [os.path.join(ORACLE, "wm_oracle.c"), os.path.join(ORACLE, "wm_oracle_cdna.c"),
              os.path.join(ORACLE, "wm_oracle_hpc.c" if hpc else "wm_oracle_occ.c")]
        subprocess.check_call(GXX + ["-fopenmp", CUDA_INC] + extra + [os.path.join(HOSTSIM, "splice_backend.cpp"), os.path.join(HOSTSIM, "kernel_emul.cpp")]
                              + host + [x for c in oc for x in ("-x", "c", c)] + ["-o", so, "-lz", "-lm", "-lpthread"], stderr=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmt_map_file_splice.argtypes = [C.c_char_p] * 3 + [C.c_int, C.c_int] + [C.c_char_p] * 2 + [C.c_int, C.c_uint64, C.c_int]
        return L
    return _once("libwm_splice_hpc.so" if hpc else "libwm_splice.so", make)


def tee():
    """wmt_tee_map_file_splice: the CUDA backend and the cDNA-aware oracle side by side, linked against the product library."""
    def make(so):
        subprocess.check_call(GXX + ["-fopenmp", "-DWMT_SPLICE_TEE", CUDA_INC, os.path.join(HOSTSIM, "splice_backend.cpp")] +
                              [x for c in ("wm_oracle.c", "wm_oracle_hpc.c", "wm_oracle_cdna.c") for x in ("-x", "c", os.path.join(ORACLE, c))] + ["-x", "none", f"-L{PKG}", "-lwinnowmap_b200", f"-Wl,-rpath,{PKG}", "-o", so, "-lz", "-lm", "-lpthread"])
        L = C.CDLL(so)
        L.wmt_tee_map_file_splice.argtypes = [C.c_char_p] * 3 + [C.c_int, C.c_int] + [C.c_char_p] * 2 + [C.c_int, C.c_int64, C.c_int, C.c_char_p]
        return L
    return _once("libwm_splice_tee.so", make)
