"""Bindings and inputs of the junction-annotation tests (--junc-bed): the oracle's annotation (oracle/wm_oracle_junc.c), the
reference's own BED reader and annotation where built (oracle/_ref/libref_harness_junc.so), the device code on the software warp
(tests/hostsim/junc_emul.cpp) and the reference's interval records of the goldens' BEDs (tests/golden/splice_junc_ref_intervals.npz).
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MANIFEST = json.load(open(os.path.join(GOLDEN, "splice_junc_manifest.json")))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden  # noqa: E402

_libs = {}


def oracle():
    if "oracle" not in _libs:
        so = os.path.join(ROOT, "oracle", "libwm_oracle_junc.so")
        src = os.path.join(ROOT, "oracle", "wm_oracle_junc.c")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
            subprocess.check_call([os.path.join(ROOT, "oracle", "build_junc.sh")], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        for f in (L.wmo_bed_junc, L.wmo_bed_junc_rev):
            f.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.c_int32, C.c_void_p]
        _libs["oracle"] = L
    return _libs["oracle"]


def ref():
    """The reference's mm_idx_bed_read / mm_idx_bed_junc, or None where oracle/_ref was not built."""
    if "ref" not in _libs:
        so = os.path.join(ROOT, "oracle", "_ref", "libref_harness_junc.so")
        L = C.CDLL(so) if os.path.exists(so) else None
        if L is not None:
            L.ref_bed_read.argtypes = [C.c_int, C.c_void_p, C.c_char_p]
            L.ref_bed_intervals.argtypes = [C.c_int, C.c_void_p, C.c_int]
            L.ref_bed_junc.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
        _libs["ref"] = L
    return _libs["ref"]


def emul():
    if "emul" not in _libs:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_junc_emul_"), "lib.so")
        hs = os.path.join(ROOT, "tests", "hostsim")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                               os.path.join(hs, "junc_emul.cpp"), os.path.join(hs, "kernel_emul.cpp"), "-o", so])
        L = C.CDLL(so)
        L.wmt_bed_junc_dev.argtypes = [C.c_void_p] * 4 + [C.c_int] * 5 + [C.c_void_p]
        _libs["emul"] = L
    return _libs["emul"]


def pipeline(hpc=False):
    """wmt_map_file_junc_aln and wmt_bed_read over the oracle backend (tests/hostsim/junc_aln_backend.cpp; hpc: with an HPC
    index), compiled once per process."""
    key = "pipe_hpc" if hpc else "pipe"
    if key not in _libs:
        import glob
        so = os.path.join(tempfile.mkdtemp(prefix="wm_junc_aln_"), "lib.so")
        csrc, hs, orc = (os.path.join(ROOT, *p) for p in (("winnowmap_b200", "csrc"), ("tests", "hostsim"), ("oracle",)))
        oc = ["wm_oracle.c", "wm_oracle_cdna.c", "wm_oracle_hpc.c" if hpc else "wm_oracle_occ.c"]
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include"] + (["-DWMT_SPLICE_HPC"] if hpc else []) +
                              [os.path.join(hs, "junc_aln_backend.cpp"), os.path.join(hs, "kernel_emul.cpp")] +
                              sorted(glob.glob(os.path.join(csrc, "host_*.cpp"))) +
                              [x for c in oc for x in ("-x", "c", os.path.join(orc, c))] + ["-o", so, "-lz", "-lm", "-lpthread"],
                              stderr=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmt_map_file_junc_aln.argtypes = [C.c_char_p] * 3 + [C.c_int] * 3 + [C.c_int64] * 2 + [C.c_int, C.c_int64] + \
            [C.c_char_p] * 2 + [C.c_int, C.c_uint64, C.c_int, C.c_char_p]
        L.wmt_splice_aln_n_exts2.restype = C.c_int64
        L.wmt_bed_read.restype = C.c_int64
        L.wmt_bed_read.argtypes = [C.c_int, C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64]
        _libs[key] = L
    return _libs[key]


def names_arg(names):
    return (C.c_char_p * len(names))(*[n.encode() for n in names])


def records(per_seq):
    """(recs as an (n, 4) int32 array of mm_idx_intv1_t records, offsets) from per-sequence (st, en, strand) lists, sorted by st."""
    rows, off = [], [0]
    for ivs in per_seq:
        for st, en, sd in sorted(ivs, key=lambda v: v[0]):
            rows.append((st, en, -1, sd << 30))  # score 0, strand:2 in the top bits (-1 << 30 is 0b11 there)
        off.append(len(rows))
    return np.array(rows, np.int32).reshape(-1, 4), np.array(off, np.int64)


def strands(recs):
    return (recs[:, 3] >> 30).astype(np.int8)  # the int32 shift sign-extends strand:2


def scores(recs):
    return ((recs[:, 3] << 2) >> 2).astype(np.int32)


def oracle_junc(recs, off, rid, st, ln, reversed_):
    """wmo_bed_junc(_rev) of window [st, st + ln) of sequence rid."""
    s = np.zeros(max(ln, 1), np.uint8)
    r = np.ascontiguousarray(recs[off[rid]:off[rid + 1]], np.int32) if 0 <= rid < len(off) - 1 else np.zeros((0, 4), np.int32)
    f = oracle().wmo_bed_junc_rev if reversed_ else oracle().wmo_bed_junc
    f(r.ctypes.data if len(r) else None, len(r), st, st + ln, s.ctypes.data)
    return s[:ln]


def multiset(recs, off):
    """per sequence, the sorted (st, en, strand, score) tuples"""
    st, sd, sc = recs[:, 0], strands(recs), scores(recs)
    return [sorted(zip(st[a:b].tolist(), recs[a:b, 1].tolist(), sd[a:b].tolist(), sc[a:b].tolist())) for a, b in zip(off[:-1], off[1:])]


def ref_intervals(names, bed):
    """the reference's mm_idx_t::I after mm_idx_bed_read(bed) on an index of these names: (recs, off)"""
    L = ref()
    assert L.ref_bed_read(len(names), names_arg(names), bed.encode()) == 0
    rows, off = [], [0]
    for rid in range(len(names)):
        n = L.ref_bed_intervals(rid, None, 0)
        buf = np.zeros((n, 4), np.int32)
        L.ref_bed_intervals(rid, buf.ctypes.data, n)
        rows.append(buf)
        off.append(off[-1] + n)
    return np.concatenate(rows) if rows else np.zeros((0, 4), np.int32), np.array(off, np.int64)


def fixture():
    return np.load(os.path.join(GOLDEN, "splice_junc_ref_intervals.npz"))


def beds(tmp):
    """(full BED, mixed BED.gz) of the goldens, checked against the fixture's md5s"""
    fb, mb = make_golden.make_junc_beds(tmp)
    fx = fixture()
    assert make_golden.md5(fb) == str(fx["full_md5"]) and make_golden.md5(mb) == str(fx["mixed_md5"])
    return fb, mb


def inputs(name, tmp):
    m = MANIFEST[name]
    ref_, reads, wfile, bed = make_golden.make_junc_inputs(name, tmp)
    assert (make_golden.md5(ref_), make_golden.md5(reads), make_golden.md5(wfile), make_golden.md5(bed)) == \
        (m["ref_md5"], m["reads_md5"], m["w_md5"], m["bed_md5"])
    return ref_, reads, wfile, bed
