"""Test helpers of the command line: the product's parser and run (csrc/host_cli.cpp) over oracle-backed index parts
(tests/hostsim/cli_backend.cpp), compiled once per process into a temporary directory, and the reference's own main()
with its index and mapping entry points wrapped (oracle/_ref/winnowmap_cli_dump, built by oracle/build_cli_ref.sh) where
it exists."""
import ctypes as C
import glob
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DUMP = os.path.join(ROOT, "oracle", "_ref", "winnowmap_cli_dump")
N_CPU = 8  # the processor count both parsers derive the default thread count from
_lib = []


def lib():
    if not _lib:
        so = os.environ.get("WM_CLI_HOST_SO") or _build()
        L = C.CDLL(so)
        L.wmt_cli_main.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
        L.wmt_cli_parse.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int, C.c_char_p]
        _lib.append((L, so))
    return _lib[0][0]


def _build():
    d = tempfile.mkdtemp(prefix="wm_cli_")
    so = os.path.join(d, "libwm_cli_host.so")
    csrc = os.path.join(ROOT, "winnowmap_b200", "csrc")
    hs = os.path.join(ROOT, "tests", "hostsim")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
           f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include", os.path.join(hs, "cli_backend.cpp"), os.path.join(hs, "kernel_emul.cpp")]
    cmd += sorted(glob.glob(os.path.join(csrc, "host_*.cpp")))
    cmd += ["-x", "c", os.path.join(ROOT, "oracle", "wm_oracle.c"), "-x", "c", os.path.join(ROOT, "oracle", "wm_oracle_occ.c"),
            "-o", so, "-lz", "-lm", "-lpthread"]
    subprocess.check_call(cmd, stderr=subprocess.DEVNULL)
    return so


def argv_of(args):
    a = [b"winnowmap"] + [x.encode() for x in args]
    return len(a), (C.c_char_p * (len(a) + 1))(*a, None)


def cli_main_host(args, cwd):
    """`winnowmap args` through the product's command line on oracle backends, in a child process (the run redirects
    stdout and getopt keeps global state): its exit status and stdout."""
    script = ("import sys, os; sys.path.insert(0, %r); import cli_lib; n, v = cli_lib.argv_of(sys.argv[1:]); "
              "rc = cli_lib.lib().wmt_cli_main(n, v); sys.stdout.flush(); os._exit(rc)") % os.path.join(ROOT, "tests")
    lib()
    p = subprocess.run([sys.executable, "-c", script] + list(args), cwd=cwd, capture_output=True,
                       env=dict(os.environ, WM_CLI_HOST_SO=_lib[0][1]))
    return p.returncode, p.stdout, p.stderr


def parse_host(args, dump):
    """The product parser on `winnowmap args`: (status, dump text or None)"""
    if os.path.exists(dump):
        os.unlink(dump)
    n, v = argv_of(args)
    rc = lib().wmt_cli_parse(n, v, N_CPU, dump.encode())
    return rc, open(dump).read() if rc == 0 and os.path.exists(dump) else None


def parse_ref(args, dump, cwd):
    """The reference's main() on `winnowmap args`: (status, dump text or None), or None where it is not built"""
    if not os.path.exists(REF_DUMP):
        return None
    if os.path.exists(dump):
        os.unlink(dump)
    p = subprocess.run([REF_DUMP] + list(args), cwd=cwd, capture_output=True, env=dict(os.environ, WM_CLI_DUMP=dump))
    return p.returncode, open(dump).read() if os.path.exists(dump) else None
