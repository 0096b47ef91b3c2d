"""Junction annotation (--junc-bed) on the CPU: the product's BED reader against the reference's interval records, the oracle's
annotation against the reference's mm_idx_bed_junc, the device code on the software warp against the oracle, and spliced
alignment through the product's host orchestration on the oracle backend (tests/hostsim/junc_aln_backend.cpp, each DP with the
oracle's annotation of its target window) against the reference's output in tests/golden/splice_junc_*."""
import gzip
import hashlib
import os

import numpy as np
import pytest

import junc_lib as jl
import test_splice_aln_cpu as sa

NAMES = ["chr1", "chr2"]


def product_intervals(names, bed):
    L = jl.pipeline()
    off = np.zeros(len(names) + 1, np.int64)
    n = L.wmt_bed_read(len(names), jl.names_arg(names), bed.encode(), None, off.ctypes.data, 0)
    assert n >= 0
    recs = np.zeros((max(n, 1), 4), np.int32)
    L.wmt_bed_read(len(names), jl.names_arg(names), bed.encode(), recs.ctypes.data, off.ctypes.data, n)
    return recs[:n], off


@pytest.mark.parametrize("kind", ["full", "mixed"])
def test_bed_reader_matches_reference_records(kind, tmp_path):
    fb, mb = jl.beds(str(tmp_path))
    fx = jl.fixture()
    names = [str(x) for x in fx["names"]]
    got = jl.multiset(*product_intervals(names, fb if kind == "full" else mb))
    exp = jl.multiset(fx[kind + "_recs"], fx[kind + "_off"])
    assert got == exp
    assert sum(map(len, exp)) > 100 and all(exp)
    for a, b in zip(fx[kind + "_off"][:-1], fx[kind + "_off"][1:]):  # sorted by start within each sequence
        assert np.all(np.diff(fx[kind + "_recs"][a:b, 0]) >= 0)


# one BED per kind of line the reader has to keep, drop or cut short (the lines of the "mixed" BED, and the edge cases around them)
LINE_KINDS = {
    "bed12": "chr1\t1000\t5000\ttx\t900\t+\t1000\t5000\t0\t3\t100,200,300,\t0,1500,3700,",
    "bed12_minus": "chr2\t100\t900\ttx\t5\t-\t100\t900\t0\t2\t50,60,\t0,740,",
    "bed12_touching_blocks": "chr1\t0\t300\ttx\t1\t+\t0\t300\t0\t3\t100,100,100,\t0,100,200,",
    "bed12_short_lists": "chr1\t0\t900\ttx\t1\t+\t0\t900\t0\t4\t100,100,\t0,400,\textra\t7,8",
    "bed6": "chr1\t200\t400\ti\t1000\t+",
    "no_strand": "chr1\t200\t400\ti\t3\t.",
    "bed3": "chr2\t10\t20",
    "bed4": "chr2\t10\t20\tname",
    "track": "track name=x",
    "comment": "#chr1\t1\t2",
    "unknown_contig": "chrX\t10\t20\tx\t0\t+",
    "st_eq_en": "chr1\t50\t50\tx\t0\t+",
    "st_gt_en": "chr1\t60\t50\tx\t0\t+",
    "negative_start": "chr1\t-5\t50\tx\t0\t+",
    "negative_end": "chr1\t5\t-50\tx\t0\t+",
    "eleven_columns": "chr1\t1000\t5000\ttx\t9\t-\t1000\t5000\t0\t2\t100,200,",
    "non_digit_block_count": "chr1\t1000\t5000\ttx\t9\t-\t1000\t5000\t0\tx2\t100,200,\t0,3800,",
    "crlf": "chr2\t300\t700\tcr\t12\t-\r",
    "big_score": "chr1\t5\t50\tx\t2000000000\t+",
    "empty": "",
}


@pytest.mark.parametrize("kind", sorted(LINE_KINDS))
def test_bed_reader_line_kind_matches_reference_live(kind, tmp_path):
    if jl.ref() is None:
        pytest.skip("oracle/_ref/libref_harness_junc.so not built (the reference's sources are absent)")
    bed = str(tmp_path / "k.bed")
    with open(bed, "w", newline="") as f:
        f.write("chr1\t7\t9\tanchor\t0\t+\n" + LINE_KINDS[kind] + "\n")
    assert jl.multiset(*product_intervals(NAMES, bed)) == jl.multiset(*jl.ref_intervals(NAMES, bed))


def test_bed_reader_missing_file_is_an_error(tmp_path):
    L = jl.pipeline()
    off = np.zeros(3, np.int64)
    assert L.wmt_bed_read(2, jl.names_arg(NAMES), str(tmp_path / "none.bed").encode(), None, off.ctypes.data, 0) == -1


def random_windows(rng, recs, off, n):
    """windows on both sequences of `off` plus one without intervals and one outside the table, biased to interval ends"""
    out = []
    n_seq = len(off) - 1
    for _ in range(n):
        rid = int(rng.integers(0, n_seq + 1))
        a, b = (off[rid], off[rid + 1]) if rid < n_seq else (0, 0)
        if b > a and rng.random() < 0.8:
            iv = recs[int(rng.integers(a, b))]
            mode = int(rng.integers(0, 4))
            st = int(iv[0]) if mode == 0 else int(iv[0]) - int(rng.integers(0, 300))
            en = int(iv[1]) if mode == 1 else int(iv[1]) - 1 if mode == 2 else int(iv[1]) + int(rng.integers(0, 300))
            st = max(st, 0)
        else:
            st = int(rng.integers(0, 200000))
            en = st + int(rng.integers(1, 3000))
        if en <= st:
            en = st + 1
        out.append((rid, st, en - st))
    return out


def test_oracle_annotation_matches_reference(tmp_path):
    if jl.ref() is None:
        pytest.skip("oracle/_ref/libref_harness_junc.so not built (the reference's sources are absent)")
    fb, mb = jl.beds(str(tmp_path))
    names = [str(x) for x in jl.fixture()["names"]] + ["empty_contig"]
    rng = np.random.default_rng(77)
    n_marked = 0
    for bed in (fb, mb):
        recs, off = jl.ref_intervals(names, bed)
        for rid, st, ln in random_windows(rng, recs, off, 1500):
            s = np.zeros(ln, np.uint8)
            jl.ref().ref_bed_junc(rid, st, st + ln, s.ctypes.data)
            got = jl.oracle_junc(recs, off, rid, st, ln, False)
            assert np.array_equal(got, s), (bed, rid, st, ln)
            n_marked += int(np.count_nonzero(s))
    assert n_marked > 1000


def test_device_annotation_on_the_software_warp_matches_oracle():
    fx = jl.fixture()
    rng = np.random.default_rng(78)
    for kind in ("full", "mixed"):
        recs, off = fx[kind + "_recs"], fx[kind + "_off"]
        keep = jl.strands(recs) != 0
        kst, ken, ksd = recs[keep, 0].copy(), recs[keep, 1].copy(), jl.strands(recs)[keep].copy()
        koff = np.array([0] + [int(np.count_nonzero(keep[:e])) for e in off[1:]], np.int64)
        for rid, st, ln in random_windows(rng, recs, off, 400):
            for rev in (0, 1):
                out = np.zeros(ln, np.uint8)
                jl.emul().wmt_bed_junc_dev(kst.ctypes.data, ken.ctypes.data, ksd.ctypes.data, koff.ctypes.data, len(off) - 1, rid, st, ln, rev,
                                           out.ctypes.data)
                assert np.array_equal(out, jl.oracle_junc(recs, off, rid, st, ln, rev)), (kind, rid, st, ln, rev)


def check_output(name, out):
    m = jl.MANIFEST[name]
    got = open(out, "rb").read()
    if m["sam"]:
        got = sa.make_golden.sam_without_pg(got)
    if hashlib.md5(got).hexdigest() == m["out_md5"]:
        return
    exp = gzip.open(os.path.join(jl.GOLDEN, name + (".sam.stripped.gz" if m["sam"] else ".paf.gz"))).read().split(b"\n")
    gl = (sa.make_golden.sam_strip_seq(got) if m["sam"] else got).split(b"\n")
    for i, (x, y) in enumerate(zip(exp, gl)):
        assert x == y, f"{name} line {i}:\n{x[:300]}\n{y[:300]}"
    raise AssertionError(f"{name}: line count {len(exp)} vs {len(gl)}")


def run_hostsim(lo, ref, reads, wfile, bed, out):
    L = jl.pipeline(lo.get("hpc", False))
    n0 = L.wmt_splice_aln_n_exts2()
    rc = L.wmt_map_file_junc_aln(ref.encode(), wfile.encode(), lo["preset"].encode(), int(lo.get("splice", False)),
                                 int(lo.get("max_intron_len", 0)), int(lo.get("sam", False)), lo.get("set_flags", 0),
                                 lo.get("clear_flags", 0), lo.get("noncan", -1), lo.get("max_sw_mat", 0), reads.encode(),
                                 out.encode(), 8, lo.get("part_bases", 0), int(lo.get("split", False)), bed.encode() if bed else None)
    assert L.wmt_splice_aln_n_exts2() > n0, "no DP went to ksw_exts2"
    return rc


@pytest.mark.parametrize("name", sorted(jl.MANIFEST))
def test_oracle_backed_junction_alignment_matches_reference(name, tmp_path):
    m = jl.MANIFEST[name]
    assert m["n_lines_differing"] > 0
    ref, reads, wfile, bed = jl.inputs(name, str(tmp_path))
    out = str(tmp_path / "o.out")
    assert run_hostsim(m["lib"], ref, reads, wfile, bed, out) >= 1
    check_output(name, out)


def test_bed_without_known_contigs_changes_nothing(tmp_path):
    """A BED whose lines name no sequence of the index: the output of the run without a BED (splice_aln_c)."""
    ref, reads, wfile = sa.inputs("splice_aln_c", str(tmp_path))
    bed = str(tmp_path / "other.bed")
    with open(bed, "w") as f:
        f.write("chrX\t100\t5000\ttx\t0\t+\t100\t5000\t0\t2\t100,100,\t0,4800,\nchrY\t10\t20\ti\t0\t-\n")
    out = str(tmp_path / "o.paf")
    assert run_hostsim(sa.MANIFEST["splice_aln_c"]["lib"], ref, reads, wfile, bed, out) == 1
    sa.check_output("splice_aln_c", out)


def test_junction_goldens_differ_from_runs_without_bed():
    for name, m in jl.MANIFEST.items():
        assert m["n_lines_differing"] > 0, name
    c = gzip.open(os.path.join(jl.GOLDEN, "splice_junc_c.paf.gz")).read()
    c0 = gzip.open(os.path.join(jl.GOLDEN, "splice_aln_c.paf.gz")).read()
    assert c != c0
