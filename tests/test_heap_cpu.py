"""--heap-sort=yes without a GPU: the oracle's restatement of collect_seed_hits_heap (oracle/wm_oracle_heap.c) against the
digests of the reference's own function (oracle/ref_harness_heap.cpp) on crafted match sets under every skip_seed flag, the
device's replay compiled for the host (csrc/seed_heap.cuh on tests/hostsim/heap_emul.cpp) against the oracle, and the product's
host orchestration on the oracle backend (tests/hostsim/heap_backend.cpp) against the heap_* goldens, byte for byte."""
import ctypes as C
import glob
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import heap_lib as H  # noqa: E402
import make_golden  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
MANIFEST = json.load(open(os.path.join(GOLDEN, "heap_manifest.json")))
_ix = None


def index():
    global _ix
    if _ix is None:
        _ix = H.Index()
    return _ix


def case_set():
    ix = index()
    c = H.cases(ix)
    c["self"] = H.self_query(ix)
    return c


CASE_NAMES = ["one_hash_many_copies", "duplicate_groups_interleaved", "lists_of_length_one", "max_occ_cut", "absent_hashes", "unique_lists",
              "read_0", "read_1", "read_2", "read_3", "read_4", "read_5", "self"]
FLAG_NAMES = [f[0] for f in H.FLAG_SETS]
_ref_ix = None


def ref_index():
    global _ref_ix
    if _ref_ix is None:
        _ref_ix = H.RefIndex(index().write_fasta(tempfile.mkdtemp(prefix="wm_heap_ref_")))
    return _ref_ix


def as_tuple(r):
    a, rep, mp = r
    return a, np.array([rep], np.int64), mp


@pytest.mark.parametrize("case", CASE_NAMES)
@pytest.mark.parametrize("flags", FLAG_NAMES)
def test_oracle_matches_reference(case, flags):
    mv, qlen, max_occ = case_set()[case]
    _, flag, qname = dict((f[0], f) for f in H.FLAG_SETS)[flags]
    got = as_tuple(H.oracle_heap(index(), mv, qlen, max_occ, flag, qname))
    H.assert_ref(f"heap_{case}_{flags}", got, lambda: as_tuple(ref_index().hits(mv, qlen, max_occ, flag, qname)))
    if H.have_ref():  # the reference itself, live
        exp = as_tuple(ref_index().hits(mv, qlen, max_occ, flag, qname))
        assert all(np.array_equal(x, y) for x, y in zip(got, exp))


@pytest.mark.parametrize("case", CASE_NAMES)
def test_sorted_path_matches_reference(case):
    """The default collection (radix_sort_128x's order) on the same sets: the tie orders the heap is compared with."""
    mv, qlen, max_occ = case_set()[case]
    got = H.oracle_sorted(index(), mv, qlen, max_occ)
    H.assert_ref(f"sorted_{case}", got, lambda: ref_index().hits(mv, qlen, max_occ, heap=False)[0])


def test_cases_reach_the_corners():
    """Ties that change the order against radix_sort_128x, a set without ties (same order), a max_occ cut (rep_len), MM_SEED_SELF
    and the -D diagonal, and every filter dropping something."""
    ix, cs = index(), case_set()
    n_diff = 0
    for name, (mv, qlen, mo) in cs.items():
        a = H.oracle_heap(ix, mv, qlen, mo)[0]
        s = H.oracle_sorted(ix, mv, qlen, mo)
        ties = len(a) > 1 and bool((a[1:, 0] == a[:-1, 0]).any())
        assert (a[1:, 0] >= a[:-1, 0]).all(), name  # ascending in x: forward anchors, then reverse ones
        if not ties:
            assert np.array_equal(a, s), name
        n_diff += not np.array_equal(a, s)
    assert n_diff >= 8
    u = H.oracle_heap(ix, *cs["unique_lists"])[0]
    assert len(u) > 100 and len(np.unique(u[:, 0])) == len(u)
    assert H.oracle_heap(ix, *cs["max_occ_cut"])[1] > 0
    mv, qlen, mo = cs["self"]
    plain = H.oracle_heap(ix, mv, qlen, mo)[0]
    d = H.oracle_heap(ix, mv, qlen, mo, H.F_NO_DIAG, b"qself")[0]
    assert len(d) < len(plain) and int((d[:, 1] >> np.uint64(43) & np.uint64(1)).sum()) > 0
    for _, flag, qname in H.FLAG_SETS[1:]:
        if qname is not None or flag & (H.F_FOR_ONLY | H.F_REV_ONLY):
            assert len(H.oracle_heap(ix, mv, qlen, mo, flag, qname)[0]) < len(plain) or flag == H.F_NO_DUAL


@pytest.mark.parametrize("case", CASE_NAMES)
@pytest.mark.parametrize("flags", FLAG_NAMES)
@pytest.mark.parametrize("stage", [True, False], ids=["staged", "global"])
def test_device_replay_on_the_host_matches_oracle(case, flags, stage):
    """wm_heap_replay_task on the software warp, over the task's anchors in ascending x with equal x in a scrambled order (as the
    tie-exact sort may leave them), with the occurrence lists staged or read where they lie."""
    mv, qlen, max_occ = case_set()[case]
    _, flag, qname = dict((f[0], f) for f in H.FLAG_SETS)[flags]
    exp = H.oracle_heap(index(), mv, qlen, max_occ, flag, qname)[0]
    rng = np.random.default_rng(len(exp))
    scrambled = exp[np.lexsort((rng.random(len(exp)), exp[:, 0]))] if len(exp) else exp
    r, got = H.emul_heap(index(), mv, qlen, max_occ, flag, qname, stage, scrambled)
    assert r == len(exp)
    assert np.array_equal(got, exp)


def test_device_replay_reports_a_foreign_slice():
    """A slice that is not the task's (one anchor too few) is reported, not silently overwritten."""
    mv, qlen, max_occ = case_set()["read_1"]
    exp = H.oracle_heap(index(), mv, qlen, max_occ)[0]
    r, _ = H.emul_heap(index(), mv, qlen, max_occ, 0, None, True, exp[:-1])
    assert r != len(exp) - 1


# ---- host orchestration on the oracle backend against the goldens ----
_lib = None


def pipeline():
    """wmt_map_file_heap over the oracle backend, compiled once per process."""
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_heap_host_"), "lib.so")
        csrc, hs, orc = (os.path.join(ROOT, *p) for p in (("winnowmap_b200", "csrc"), ("tests", "hostsim"), ("oracle",)))
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                               os.path.join(hs, "heap_backend.cpp"), os.path.join(hs, "kernel_emul.cpp")] +
                              sorted(glob.glob(os.path.join(csrc, "host_*.cpp"))) +
                              [x for c in ("wm_oracle.c", "wm_oracle_occ.c", "wm_oracle_heap.c") for x in ("-x", "c", os.path.join(orc, c))] +
                              ["-o", so, "-lz", "-lm", "-lpthread"], stderr=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmt_map_file_heap.argtypes = [C.c_char_p] * 4 + [C.c_int, C.c_int, C.c_uint64, C.c_int]
        _lib = L
    return _lib


def inputs(name, tmp):
    m = MANIFEST[name]
    ref, reads = make_golden.make_heap_inputs(m["inputs"], tmp)
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"]
    return ref, reads


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


# what this oracle backend serves: no homopolymer-compressed index, cDNA chaining or self-mapping seed filter
# (tests/test_gpu_heap.py runs those cases)
HOST_CASES = sorted(n for n, m in MANIFEST.items() if not (m["lib"].get("hpc") or m["lib"].get("all_vs_all") or m["lib"]["preset"] == "splice"))


@pytest.mark.parametrize("name", HOST_CASES)
def test_oracle_backed_heap_mapping_matches_reference(name, tmp_path):
    lo = MANIFEST[name]["lib"]
    ref, reads = inputs(name, str(tmp_path))
    out = str(tmp_path / "o.out")
    mode = 2 if lo.get("sam") else (0 if lo.get("cigar") is False else 1)
    rc = pipeline().wmt_map_file_heap(ref.encode(), lo["preset"].encode(), reads.encode(), out.encode(), 8, mode, lo.get("part_bases", 0),
                                      int(lo.get("split", False)))
    assert rc >= 1, rc
    check_output(name, out)


def test_manifest_cases_differ_where_ties_decide():
    """The all-vs-all golden and at least one mapping golden differ from the reference's run with --heap-sort=no (counted by
    make_golden.main_heap), and none is a command the command line would replay: it refuses --heap-sort=yes."""
    for m in MANIFEST.values():
        assert "cmd" not in m and "--heap-sort=yes" in m["ref_cmd"].split()
    assert MANIFEST["heap_tandem_X"]["n_lines_differing"] > 0
    assert any(m["n_lines_differing"] > 0 for n, m in MANIFEST.items() if not m["lib"].get("all_vs_all"))
    assert {"map-ont", "map-pb", "splice"} <= {m["lib"]["preset"] for m in MANIFEST.values()}


def test_heap_sort_option_sets_the_flag():
    from winnowmap_b200.mapper import F_HEAP_SORT, make_options
    assert make_options("map-ont", heap_sort=True)[1].flag & F_HEAP_SORT
    assert not make_options("map-ont")[1].flag & F_HEAP_SORT
