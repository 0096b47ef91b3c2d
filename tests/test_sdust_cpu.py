"""SDUST low-complexity masking (-T) without a GPU: the oracle's SDUST and minimizer squeeze (oracle/wm_oracle_sdust.c) against
the digests of the reference's own sdust() and mm_dust_minier (oracle/ref_harness_sdust.cpp), the device code compiled for the
host (csrc/sdust.cuh on tests/hostsim/sdust_emul.cpp) against the oracle, and the product's host orchestration on the oracle
backend (tests/hostsim/sdust_backend.cpp) against every sdust_* golden, byte for byte."""
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
import hpc_lib as H  # noqa: E402
import make_golden  # noqa: E402
import oracle_lib as ol  # noqa: E402
import sdust_lib as S  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
MANIFEST = json.load(open(os.path.join(GOLDEN, "sdust_manifest.json")))


@pytest.mark.parametrize("T", S.T_SET)
def test_oracle_sdust_matches_reference(T):
    seqs = S.case_set()
    got = tuple(S.oracle_sdust(s, T) for s in seqs)
    assert T > 40 or sum(len(g) for g in got) > 0
    S.assert_ref(f"sdust_T{T}", got, lambda: tuple(S.ref_sdust(s, T) for s in seqs))


@pytest.mark.parametrize("W", [3, 10, 63])
def test_oracle_sdust_other_windows_match_reference(W):
    seqs = S.crafted_sequences()
    got = tuple(S.oracle_sdust(s, 20, W) for s in seqs)
    S.assert_ref(f"sdust_T20_W{W}", got, lambda: tuple(S.ref_sdust(s, 20, W) for s in seqs))


def test_sdust_cases_reach_the_corners():
    """An N cut makes the perfect-interval list grow past C(62, 2) (what the device's capacity must cover), regions merge, and
    regions can end after the sequence (the window carries over an N)."""
    seqs = S.case_set()
    assert max(S.oracle_max_perfect(s, 1) for s in seqs) > 1891
    ends_past = any(len(r) and int(S.as_pairs(r)[:, 1].max()) > len(s) for s in seqs for r in [S.oracle_sdust(s, 1)])
    assert ends_past
    assert any(len(S.oracle_sdust(s, 20)) > 1 for s in seqs)


@pytest.mark.parametrize("T", S.T_SET)
def test_device_sdust_on_the_host_matches_oracle(T):
    for s in S.case_set():
        assert np.array_equal(S.emul_sdust(s, T), S.oracle_sdust(s, T)), (T, s[:40])


def test_device_sdust_small_list_gives_up_or_is_exact():
    """With the first pass's short perfect-interval list (WM_SDUST_PCAP_FAST) a sequence either comes out exact or is handed back
    for the second pass (-1): never a truncated region list.  The set holds sequences of both kinds."""
    n_back = 0
    for T in (1, 2, 20):
        for s in S.case_set():
            got = S.emul_sdust(s, T, pcap=S.PCAP_FAST)
            if got is None:
                n_back += 1
                assert S.oracle_max_perfect(s, T) > S.PCAP_FAST
            else:
                assert np.array_equal(got, S.oracle_sdust(s, T)), (T, s[:40])
    assert n_back > 0


def _minimizers(seqs, hpc):
    k, w = 15, 10
    ob = ol.OracleBloom(np.zeros(0, dtype=np.uint64))
    return [H.oracle_sketch_hpc(s, w, k) if hpc else ol.oracle_sketch(s, w, k, 0, ob) for s in seqs]


def _overlaps(m, reg):
    """Per minimizer: the bases of its span [pos - span + 1, pos] inside the regions, and its span."""
    pos = ((m[:, 1] & np.uint64(0xffffffff)) >> np.uint64(1)).astype(np.int64)
    span = (m[:, 0] & np.uint64(0xff)).astype(np.int64)
    s, e = pos - span + 1, pos + 1
    ov = np.zeros(len(m), dtype=np.int64)
    for rs, re in S.as_pairs(reg):
        ov += np.clip(np.minimum(e, re) - np.maximum(s, rs), 0, None)
    return ov, span


@pytest.mark.parametrize("hpc", [False, True])
@pytest.mark.parametrize("T", [2, 10, 20, 40])
def test_oracle_squeeze_matches_reference(T, hpc):
    seqs = [s for s in S.case_set() if len(s) >= 30]
    mzs = _minimizers(seqs, hpc)
    got = tuple(S.oracle_dust_minier(m, S.oracle_sdust(s, T)) for m, s in zip(mzs, seqs))
    n_all, n_kept = sum(len(m) for m in mzs), sum(len(g) for g in got)
    # T = 2 masks most of random sequence too (it keeps 6-9 %)
    assert (0.3 if T >= 10 else 0.02) * n_all < n_kept < n_all, (n_kept, n_all)
    # the set decides both ways on minimizers that lie partly in a region: some at most half in (kept), some more (dropped)
    ov = [_overlaps(m, S.oracle_sdust(s, T)) for m, s in zip(mzs, seqs)]
    part = np.concatenate([(o > 0) & (o < sp) for o, sp in ov])
    half = np.concatenate([o <= sp // 2 for o, sp in ov])
    assert (part & half).sum() > 0 and (part & ~half).sum() > 0
    S.assert_ref(f"dust_minier_T{T}_{'hpc' if hpc else 'k15'}", got,
                 lambda: tuple(S.ref_dust_minier(m, s, T) for m, s in zip(mzs, seqs)))


@pytest.mark.parametrize("hpc", [False, True])
def test_device_squeeze_on_the_host_matches_oracle(hpc):
    for T in (2, 10, 20, 40):
        seqs = [s for s in S.case_set() if len(s) >= 30]
        for m, s in zip(_minimizers(seqs, hpc), seqs):
            reg = S.oracle_sdust(s, T)
            assert np.array_equal(S.emul_dust_minier(m, reg), S.oracle_dust_minier(m, reg))


_lib = None


def pipeline():
    """wmt_map_file_sdust over the oracle backend, compiled once per process."""
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_sdust_host_"), "lib.so")
        csrc, hs, orc = (os.path.join(ROOT, *p) for p in (("winnowmap_b200", "csrc"), ("tests", "hostsim"), ("oracle",)))
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                               os.path.join(hs, "sdust_backend.cpp"), os.path.join(hs, "kernel_emul.cpp")] +
                              sorted(glob.glob(os.path.join(csrc, "host_*.cpp"))) +
                              [x for c in ("wm_oracle.c", "wm_oracle_occ.c", "wm_oracle_sdust.c") for x in ("-x", "c", os.path.join(orc, c))] +
                              ["-o", so, "-lz", "-lm", "-lpthread"], stderr=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmt_map_file_sdust.argtypes = [C.c_char_p] * 5 + [C.c_int, C.c_int, C.c_int64, C.c_int, C.c_uint64, C.c_int]
        _lib = L
    return _lib


def inputs(name, tmp):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_sdust_inputs(m["inputs"], tmp)
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"]
    assert (make_golden.md5(wfile) if wfile else None) == m["w_md5"]
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


# what this oracle backend serves: no homopolymer-compressed index, cDNA chaining or self-mapping seed filter
# (tests/test_gpu_sdust.py runs those cases)
HOST_CASES = sorted(n for n, m in MANIFEST.items() if not (m["lib"].get("hpc") or m["lib"].get("all_vs_all") or m["lib"]["preset"] == "splice"))


@pytest.mark.parametrize("name", HOST_CASES)
def test_oracle_backed_sdust_mapping_matches_reference(name, tmp_path):
    m, lo = MANIFEST[name], MANIFEST[name]["lib"]
    ref, reads, wfile = inputs(name, str(tmp_path))
    out = str(tmp_path / "o.out")
    mode = 2 if lo.get("sam") else (0 if lo.get("cigar") is False else 1)
    flags = 0
    rc = pipeline().wmt_map_file_sdust(ref.encode(), wfile.encode() if wfile else None, lo["preset"].encode(), reads.encode(), out.encode(), 8,
                                       mode, flags, lo["sdust_thres"], lo.get("part_bases", 0), int(lo.get("split", False)))
    assert rc >= 1, rc
    check_output(name, out)


def test_manifest_cases_all_mask():
    """Every golden differs from the reference's run without -T (asserted by make_golden.main_sdust) and none is a command the
    command line would replay: it refuses -T."""
    for m in MANIFEST.values():
        assert m["n_lines_differing"] > 0 and "cmd" not in m and "-T" in m["ref_cmd"].split()
    assert {"map-ont", "splice"} <= {m["lib"]["preset"] for m in MANIFEST.values()}


def test_mapper_refuses_out_of_range_threshold():
    from winnowmap_b200.mapper import SDUST_MAX_T, Mapper
    for bad in (-1, SDUST_MAX_T + 1):
        with pytest.raises(ValueError):
            Mapper("unused.fa", sdust_thres=bad)
