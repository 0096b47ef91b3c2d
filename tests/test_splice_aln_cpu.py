"""Spliced base-level alignment (-c / -a with -x splice / splice:hq / cdna or --splice) on the CPU: the product's host orchestration
(the two strand rounds of mm_align_skeleton, mm_fix_bad_ends_splice, the splice flags of every DP, ts:A) over the oracle backend,
whose DP is the oracle's ksw_exts2 when the orchestration's scoring asks for splice (tests/hostsim/splice_aln_backend.cpp), against
the reference's output in tests/golden/splice_aln_*; and the Python options of the opt-in."""
import ctypes as C
import glob
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MANIFEST = json.load(open(os.path.join(GOLDEN, "splice_aln_manifest.json")))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden  # noqa: E402

_libs = {}


def pipeline(hpc=False):
    """wmt_map_file_splice_aln over the oracle backend (hpc: with an HPC index), compiled once per process."""
    key = "hpc" if hpc else "plain"
    if key not in _libs:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_splice_aln_"), "lib.so")
        csrc, hs, orc = (os.path.join(ROOT, *p) for p in (("winnowmap_b200", "csrc"), ("tests", "hostsim"), ("oracle",)))
        oc = ["wm_oracle.c", "wm_oracle_cdna.c", "wm_oracle_hpc.c" if hpc else "wm_oracle_occ.c"]
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include"] + (["-DWMT_SPLICE_HPC"] if hpc else []) +
                              [os.path.join(hs, "splice_aln_backend.cpp"), os.path.join(hs, "kernel_emul.cpp")] +
                              sorted(glob.glob(os.path.join(csrc, "host_*.cpp"))) +
                              [x for c in oc for x in ("-x", "c", os.path.join(orc, c))] + ["-o", so, "-lz", "-lm", "-lpthread"],
                              stderr=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmt_map_file_splice_aln.argtypes = [C.c_char_p] * 3 + [C.c_int] * 3 + [C.c_int64] * 2 + [C.c_int, C.c_int64] + \
            [C.c_char_p] * 2 + [C.c_int, C.c_uint64, C.c_int]
        L.wmt_splice_aln_n_exts2.restype = C.c_int64
        _libs[key] = L
    return _libs[key]


def inputs(name, tmp):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_splice_inputs(m["reads"], tmp)
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"] and make_golden.md5(wfile) == m["w_md5"]
    return ref, reads, wfile


def check_output(name, out):
    """The output of a run equals the reference's (SAM: but for the @PG line)."""
    m = MANIFEST[name]
    got = open(out, "rb").read()
    if m["sam"]:
        got = make_golden.sam_without_pg(got)
    if hashlib.md5(got).hexdigest() == m["out_md5"]:
        return
    exp = gzip.open(os.path.join(GOLDEN, name + (".sam.stripped.gz" if m["sam"] else ".paf.gz"))).read().split(b"\n")
    gl = (make_golden.sam_strip_seq(got) if m["sam"] else got).split(b"\n")
    for i, (x, y) in enumerate(zip(exp, gl)):
        if x != y:
            raise AssertionError(f"{name} line {i}:\n{x[:300]}\n{y[:300]}")
    raise AssertionError(f"{name}: line count {len(exp)} vs {len(gl)} (or SEQ/QUAL text differs)")


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_oracle_backed_spliced_alignment_matches_reference(name, tmp_path):
    m, lo = MANIFEST[name], MANIFEST[name]["lib"]
    ref, reads, wfile = inputs(name, str(tmp_path))
    L = pipeline(lo.get("hpc", False))
    out = str(tmp_path / "o.out")
    n0 = L.wmt_splice_aln_n_exts2()
    rc = L.wmt_map_file_splice_aln(ref.encode(), wfile.encode(), lo["preset"].encode(), int(lo.get("splice", False)), int(lo.get("max_intron_len", 0)),
                                   int(lo.get("sam", False)), lo.get("set_flags", 0), lo.get("clear_flags", 0), lo.get("noncan", -1),
                                   lo.get("max_sw_mat", 0), reads.encode(), out.encode(), 8, lo.get("part_bases", 0), int(lo.get("split", False)))
    assert rc >= 1, rc
    assert L.wmt_splice_aln_n_exts2() > n0, "no DP went to ksw_exts2"
    check_output(name, out)


def test_goldens_cover_the_strand_rounds():
    """The -c golden has hits on both transcript strands and ties between the rounds (no ts:A); -u n gives ts:A:- throughout."""
    c = gzip.open(os.path.join(GOLDEN, "splice_aln_c.paf.gz")).read().decode().splitlines()
    ts = [next((f for f in ln.split("\t") if f.startswith("ts:A:")), None) for ln in c]
    assert ts.count("ts:A:+") > 0 and ts.count("ts:A:-") > 0 and ts.count(None) > 0
    assert any("N" in next(f for f in ln.split("\t") if f.startswith("cg:Z:")) for ln in c)
    un = gzip.open(os.path.join(GOLDEN, "splice_aln_un.paf.gz")).read().decode().splitlines()
    assert un and all("\tts:A:-" in ln for ln in un if "\tcg:Z:" in ln)


# ---------------------------------------------------------------------------------------------------------------- options

def test_make_options_spliced_alignment_opt_in():
    from winnowmap_b200 import mapper as M
    for preset in ("splice", "splice:hq", "cdna"):
        for cigar, sam in ((True, False), (False, True)):
            with pytest.raises(ValueError):
                M.make_options(preset, cigar=cigar, sam=sam)
            io, mo = M.make_options(preset, cigar=cigar, sam=sam, spliced_alignment=True)
            assert mo.flag & M.F_SPLICE and mo.flag & M.F_CIGAR
            assert bool(mo.flag & M.F_OUT_SAM) == sam
            assert M.lib().wm_check_opt(C.byref(io), C.byref(mo)) == -8  # the C check keeps its answer
    io, mo = M.make_options("map-ont", splice=True, max_intron_len=20000, spliced_alignment=True)
    assert mo.flag & M.F_SPLICE and mo.flag & M.F_CIGAR and mo.max_gap_ref == 20000
    # without spliced mapping the keyword changes nothing
    a, b = M.make_options("map-ont"), M.make_options("map-ont", spliced_alignment=True)
    assert bytes(a[1]) == bytes(b[1])
    io, mo = M.make_options("splice", cigar=False, spliced_alignment=True)
    assert not mo.flag & M.F_CIGAR


_JUNC_CHILD = r'''
import ctypes as C, sys
sys.path.insert(0, %r)
import test_splice_aln_cpu as T
ref, reads, wfile, out, sam = sys.argv[1:6]
L = T.pipeline()
L.wmt_splice_aln_set_junc(1)
sys.exit(L.wmt_map_file_splice_aln(ref.encode(), wfile.encode(), b"splice", 0, 0, 0, 0, 0, -1, 0, reads.encode(), out.encode(), 4, 0, 0) != 1)
'''


def test_spliced_alignment_refuses_an_index_with_junctions(tmp_path):
    """An index that carries junction intervals (--junc-bed, WM_IDX_JUNC at upload): spliced alignment exits with a message
    instead of aligning without them (junction annotation is not built)."""
    import subprocess
    ref, reads, wfile = inputs("splice_aln_c", str(tmp_path))
    r = subprocess.run([sys.executable, "-c", _JUNC_CHILD % os.path.dirname(os.path.abspath(__file__)), ref, reads, wfile,
                        str(tmp_path / "o.paf"), "0"], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 1 and b"--junc-bed" in r.stderr and b"not supported" in r.stderr, r.stderr[-500:]
