"""Self and all-vs-all mapping (-D, --dual=no, -X) and single-strand mapping (--for-only, --rev-only) without a GPU.

The product's host orchestration runs on the oracle backend with the seed filter restated from skip_seed
(tests/hostsim/overlap_backend.cpp) and must reproduce the reference's goldens (tests/golden/overlap_*, made by
tools/make_golden.py --overlap) byte for byte.  The name-rank reduction the device filter uses is checked against strcmp."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden  # noqa: E402

MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "overlap_manifest.json")))
F = dict(no_diag=0x001, no_dual=0x002, no_ljoin=0x400, for_only=0x100000, rev_only=0x200000, all_chains=0x800000)


def lib_flags(o):
    """The mapping flags Mapper sets for the library options of a manifest entry (winnowmap_b200/mapper.py make_options)."""
    f = 0
    if o.get("no_diag"):
        f |= F["no_diag"]
    if o.get("dual") is False:
        f |= F["no_dual"]
    if o.get("all_vs_all"):
        f |= F["all_chains"] | F["no_diag"] | F["no_dual"] | F["no_ljoin"]
    f |= {"for": F["for_only"], "rev": F["rev_only"]}.get(o.get("strand"), 0)
    return f


@pytest.fixture(scope="module")
def overlap_sim(tmp_path_factory):
    d = os.path.join(ROOT, "tests", "hostsim")
    cs = os.path.join(ROOT, "winnowmap_b200", "csrc")
    so = str(tmp_path_factory.mktemp("overlap_sim") / "libwm_overlap_sim.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", f"-I{cuda}/include",
                           os.path.join(d, "overlap_backend.cpp"), os.path.join(d, "kernel_emul.cpp")]
                          + [os.path.join(cs, f) for f in ("host_map.cpp", "host_align.cpp", "host_glue.cpp", "host_io.cpp", "host_format.cpp")]
                          + ["-x", "c", os.path.join(ROOT, "oracle", "wm_oracle.c"), "-o", so, "-lz", "-lm", "-lpthread"])
    L = C.CDLL(so)
    L.wmt_map_file_overlap.argtypes = [C.c_char_p] * 5 + [C.c_int, C.c_int, C.c_int64]
    L.wmt_name_filter.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_void_p]
    return L


def _first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
    return f"line count {len(la)} vs {len(lb)}"


@pytest.mark.parametrize("name", sorted(n for n in MANIFEST if not MANIFEST[n]["lib"].get("hpc")))
def test_host_overlap_matches_reference(overlap_sim, name, tmp_path):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_overlap_inputs(m["inputs"], str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    o = m["lib"]
    mode = 2 if o.get("sam") else (0 if o.get("cigar") is False else 1)
    out = str(tmp_path / "out")
    rc = overlap_sim.wmt_map_file_overlap(ref.encode(), wfile.encode() if wfile else None, o["preset"].encode(), reads.encode(), out.encode(),
                                          8, mode, lib_flags(o))
    assert rc == 0
    got = open(out, "rb").read()
    if mode == 2:
        got = make_golden.sam_without_pg(got)
        if hashlib.md5(got).hexdigest() != m["sam_md5"]:
            exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".sam.stripped.gz")).read()
            got = make_golden.sam_strip_seq(got)
            assert got == exp, _first_diff(exp, got)
            pytest.fail("SEQ/QUAL differ")
    else:
        exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".paf.gz")).read()
        assert got == exp, _first_diff(exp, got)


def _strcmp(a, b):
    return (a > b) - (a < b)  # bytes compare as unsigned char, as strcmp does


def test_name_rank_reduction_matches_strcmp(overlap_sim):
    """cmp > 0 <=> rank[rid] < lt and cmp == 0 <=> eq && rank[rid] == lt, over all pairs of a crafted name set: shared prefixes,
    duplicates, the empty name, bytes >= 0x80, query names absent from the index, and a read without a name."""
    names = [b"r1", b"r10", b"r1", b"r", b"", b"r1\x80", b"r1\xff", b"\xc3\xa9", b"chr1", b"chr10", b"chr2", b"chr1", b"a" * 300, b"Z", b"z"]
    queries = names + [b"r0", b"r11", b"r1\x7f", b"r1\x80\x00x", b"\xff", b"0", b"a" * 299, b"a" * 301, b"chr1_", b"q"]
    has = [1] * len(queries) + [0]
    queries = queries + [None]
    n, m = len(names), len(queries)
    out = (C.c_uint8 * (n * m))()
    overlap_sim.wmt_name_filter(n, (C.c_char_p * n)(*names), m, (C.c_char_p * m)(*queries), (C.c_int * m)(*has), out)
    for j, q in enumerate(queries):
        for i, s in enumerate(names):
            v = out[j * n + i]
            if q is None:
                assert v == 4
                continue
            c = _strcmp(q.split(b"\0")[0], s)
            assert v == (1 if c > 0 else 0) | (2 if c == 0 else 0), (q, s, v)
