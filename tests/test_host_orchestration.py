"""CPU-only end-to-end test of the product's HOST orchestration (wave scheduler, align state machines, glue, PAF
writer): the product's host sources are linked with a test-only Backend served by the CPU oracle
(tests/hostsim/cpu_backend.cpp) and the PAF must be byte-identical to the reference goldens.  This exercises every
host code path the GPU runs use, without a GPU; the device kernels themselves are covered by the -m gpu tests."""
import ctypes as C
import gzip
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden  # noqa: E402

MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "manifest.json")))


@pytest.fixture(scope="module")
def hostsim():
    d = os.path.join(ROOT, "tests", "hostsim")
    subprocess.check_call([os.path.join(d, "build.sh")], stderr=subprocess.DEVNULL)
    L = C.CDLL(os.path.join(d, "libwm_hostsim.so"))
    L.wmt_map_file.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    L.wmt_set_scoring.argtypes = [C.c_int] * 7
    return L


@pytest.mark.parametrize("name", ["ont_small", "hifi_small", "ont_sv", "ont_tandem", "asm20_small", "ont_single_gap", "asm5_small", "asm10_small",
                                  "ont_sv_long_inc"])
def test_host_pipeline_matches_reference_golden(hostsim, name, tmp_path):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_inputs(name, str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"]
    out = str(tmp_path / "o.paf")
    hostsim.wmt_set_scoring(*make_golden.scoring_override(m["params"]))  # -A / -B / --score-N / -O / -E of the case
    rc = hostsim.wmt_map_file(ref.encode(), wfile.encode() if wfile else None, m["params"]["preset"].encode(), reads.encode(), out.encode(), 8)
    assert rc == 0
    exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".paf.gz")).read()
    got = open(out, "rb").read()
    if got != exp:
        le, lg = exp.split(b"\n"), got.split(b"\n")
        for i, (x, y) in enumerate(zip(le, lg)):
            if x != y:
                fx, fy = x.split(b"\t"), y.split(b"\t")
                cols = [j for j, (p, q) in enumerate(zip(fx, fy)) if p != q]
                raise AssertionError(f"line {i} cols {cols}: {[fx[j][:50] for j in cols[:5]]} vs {[fy[j][:50] for j in cols[:5]]}")
        raise AssertionError(f"line count {len(le)} vs {len(lg)}")


@pytest.mark.parametrize("name", ["ont_small", "ont_sv"])
def test_host_sam_writer_matches_reference_golden(hostsim, name, tmp_path):
    """SAM output (-a) of the host writer, oracle-backed: byte-identical to the reference's SAM but for the @PG line."""
    import hashlib
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_inputs(name, str(tmp_path))
    out = str(tmp_path / "o.sam")
    hostsim.wmt_map_file_sam.argtypes = hostsim.wmt_map_file.argtypes
    rc = hostsim.wmt_map_file_sam(ref.encode(), wfile.encode() if wfile else None, m["params"]["preset"].encode(), reads.encode(), out.encode(), 8)
    assert rc == 0
    got = make_golden.sam_without_pg(open(out, "rb").read())
    if hashlib.md5(got).hexdigest() != m["sam_md5"]:
        exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".sam.stripped.gz")).read().split(b"\n")
        gl = make_golden.sam_strip_seq(got).split(b"\n")
        for i, (x, y) in enumerate(zip(exp, gl)):
            if x != y:
                fx, fy = x.split(b"\t"), y.split(b"\t")
                cols = [j for j, (p, q) in enumerate(zip(fx, fy)) if p != q]
                raise AssertionError(f"line {i} cols {cols}: {[fx[j][:60] for j in cols[:5]]} vs {[fy[j][:60] for j in cols[:5]]}")
        raise AssertionError(f"line count {len(exp)} vs {len(gl)} (or SEQ/QUAL text differs)")


@pytest.mark.parametrize("key,sam,flags", [("paf_cs", 0, 0x40), ("paf_cs_long", 0, 0x40 | 0x800), ("sam_md", 1, 0x1000000),
                                            ("paf_eqx", 0, 0x4000000), ("sam_softclip", 1, 0x80000),
                                            ("sam_no2nd_hitonly", 1, 0x4000 | 0x40000000), ("paf_no_hit", 0, 0x8000000),
                                            ("sam_fastq_comment", 1, 0x2000000), ("paf_edge", 0, 0), ("sam_edge", 1, 0),
                                            ("paf_edge_N0", 0, 0), ("paf_edge_N3", 0, 0)])
def test_host_output_options_match_reference(hostsim, key, sam, flags, tmp_path):
    """Output options against the reference run with the same switches: --cs / --cs=long / --MD difference strings
    (src/format.c:141-243), --eqx (=/X CIGAR, src/align.c:169-238), -Y, --secondary=no --sam-hit-only, --paf-no-hit, and
    gzipped FASTQ input with comments under -y (QUAL column, comment copied to the record), and the N-rich edge reads
    under --score-N 0 and 3."""
    import hashlib
    case = make_golden.TAG_CASES[key]
    name = case[0]
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_inputs(name, str(tmp_path))
    if len(case) > 2 and case[2] == "fastq":
        reads = make_golden.fastq_gz_of(reads, reads + ".fq.gz")
    if len(case) > 2 and case[2] == "edge":  # empty, tiny, N-rich, lower-case, chimeric, unmappable reads
        reads = make_golden.edge_reads_of(reads, reads + ".edge.fa")
    out = str(tmp_path / "o.txt")
    if len(case) > 3:  # --score-N
        hostsim.wmt_set_scoring(*make_golden.scoring_override(dict(scoring=case[3])))
    hostsim.wmt_map_file_flags.argtypes = [C.c_char_p] * 5 + [C.c_int, C.c_int, C.c_int64]
    rc = hostsim.wmt_map_file_flags(ref.encode(), wfile.encode() if wfile else None, m["params"]["preset"].encode(), reads.encode(), out.encode(), 8, sam, flags)
    assert rc == 0
    got = make_golden.sam_without_pg(open(out, "rb").read())
    if hashlib.md5(got).hexdigest() != m["tag_md5"][key]:
        if key == "paf_cs":
            exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".cs.paf.gz")).read().split(b"\n")
            for i, (x, y) in enumerate(zip(exp, got.split(b"\n"))):
                if x != y:
                    fx, fy = x.split(b"\t"), y.split(b"\t")
                    cols = [j for j, (p, q) in enumerate(zip(fx, fy)) if p != q]
                    raise AssertionError(f"line {i} cols {cols}: {[fx[j][:80] for j in cols[:3]]} vs {[fy[j][:80] for j in cols[:3]]}")
        raise AssertionError(f"{key}: output differs from the reference (md5)")


def test_index_pair_sort_is_the_sorted_order(hostsim):
    """wm_index_build orders the (minimizer, position) pairs of the reference by hash, then position (src/index.c:239)
    with a partitioned parallel sort (csrc/host_index.h): same result as a plain sort, for any thread count."""
    import numpy as np
    hostsim.wmt_sort_index_pairs.argtypes = [C.c_void_p, C.c_int64, C.c_int]
    rng = np.random.default_rng(5)
    for n, key_bits, threads in [(0, 30, 4), (1, 30, 4), (1000, 30, 8), (70000, 12, 3), (300000, 30, 8), (500000, 38, 16)]:
        x = (rng.integers(0, 1 << key_bits, size=n, dtype=np.uint64) << np.uint64(8)) | rng.integers(0, 256, size=n, dtype=np.uint64)
        y = rng.permutation(n).astype(np.uint64)
        a = np.stack([x, y], axis=1).copy()
        hostsim.wmt_sort_index_pairs(a.ctypes.data, n, threads)
        order = np.lexsort((y, x >> np.uint64(8)))
        assert np.array_equal(a, np.stack([x[order], y[order]], axis=1)), (n, key_bits, threads)


def test_reference_packing_matches_the_plain_loop(hostsim):
    """pack_seq4 (csrc/host_index.h: whole words in parallel, shared edge words serially) against mm_seq4_set applied base by base
    (src/mmpriv.h:29): several sequences back to back at odd offsets, lengths around the word size, IUPAC and lower case."""
    import numpy as np
    rng = np.random.default_rng(12)
    hostsim.wmt_pack_seq4.argtypes = [C.c_void_p, C.c_uint64, C.c_char_p, C.c_uint64]
    alphabet = np.frombuffer(b"ACGTacgtNnRYU", dtype=np.uint8)
    code = {ord("A"): 0, ord("a"): 0, ord("C"): 1, ord("c"): 1, ord("G"): 2, ord("g"): 2, ord("T"): 3, ord("t"): 3}
    lens = [0, 1, 3, 7, 8, 9, 15, 16, 17, 5, 64, 100, 40000, 2, 33000, 6]
    seqs = [alphabet[rng.integers(0, len(alphabet), size=n)].tobytes() for n in lens]
    total = sum(lens)
    S = np.zeros((total + 7) // 8 + 1, np.uint32); E = np.zeros_like(S)
    o = 0
    for sq in seqs:
        hostsim.wmt_pack_seq4(S.ctypes.data, o, sq, len(sq))
        for j, ch in enumerate(sq):
            E[(o + j) >> 3] |= np.uint32(code.get(ch, 4) << (((o + j) & 7) << 2))
        o += len(sq)
    assert np.array_equal(S, E)


def test_scorings_whose_int8_lanes_wrap_are_refused(hostsim, tmp_path):
    """check_opt (csrc/host_io.cpp) refuses two gap pairs with -A + q + 2e > 128 (return code -7): there the reference's ksw_extd2_sse wraps its int8 lanes and the device fill, which keeps them in 16 bits,
    would differ.  Every scoring of tee_lib.SCORINGS passes, and so do the limit itself and one gap pair (ksw_extz2 wraps
    as the reference does).  The oracle-backed run refuses the same options."""
    import ctypes as C
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import tee_lib as T
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import make_options

    def check(a, b, q, e, q2, e2, sc_ambi):
        io, mo = make_options("map-ont")
        mo.a, mo.b, mo.q, mo.e, mo.q2, mo.e2, mo.sc_ambi = a, b, q, e, q2, e2, sc_ambi
        return lib().wm_check_opt(C.byref(io), C.byref(mo))
    for name, s in T.SCORINGS.items():
        assert check(*s) == 0, name
    assert check(*T.REFUSED_SCORINGS["wrap_probe"]) == -7
    assert check(82, 4, 40, 3, 83, 1, 1) == 0 and check(83, 4, 40, 3, 83, 1, 1) == -7   # 82 + 40 + 6 = 128 / 129
    assert check(121, 4, 4, 2, 24, 1, 1) == -7 and check(120, 4, 4, 2, 24, 1, 1) == 0
    assert check(100, 4, 40, 3, 40, 3, 1) == 0                                           # one gap pair
    m = MANIFEST["ont_small"]
    ref, reads, wfile = make_golden.make_inputs("ont_small", str(tmp_path))
    hostsim.wmt_set_scoring(*make_golden.scoring_override(dict(scoring=T.REFUSED_SCORINGS["wrap_probe"])))
    assert hostsim.wmt_map_file(ref.encode(), None, m["params"]["preset"].encode(), reads.encode(), str(tmp_path / "o.paf").encode(), 8) != 0
