"""Junction annotation (--junc-bed) on the GPU: wm_bed_junc_batch against the oracle on crafted windows, every splice_junc_*
golden reproduced by Mapper(..., spliced_alignment=True, junc_bed=...), the reference's own interval records handed over with
wm_idx_set_junc, and runs that must not annotate (no splice DP, or no BED) unchanged and without an annotation launch."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

import junc_lib as jl
import test_splice_aln_cpu as sa
from test_junc_cpu import check_output, random_windows

pytestmark = pytest.mark.gpu


def junc_stats():
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import _setup
    L = _setup(lib())
    o = (C.c_double * 3)()
    L.wm_junc_stats(o, 1)
    return list(o)


def _check_batch(per_seq, windows):
    from winnowmap_b200 import kernels
    recs, off = jl.records(per_seq)
    got = kernels.bed_junc_batch(per_seq, windows)
    for (rid, st, ln, rev), g in zip(windows, got):
        assert np.array_equal(g, jl.oracle_junc(recs, off, rid, st, ln, rev)), (rid, st, ln, rev)
    return got


def test_bed_junc_batch_crafted_windows():
    # sequence 0: three isoforms sharing one donor, both strands, strand 0, intervals at the window's edges; sequence 1: none
    iso = [(100, 200, 1), (100, 300, 1), (100, 450, 1), (150, 160, -1), (150, 170, 0), (99, 101, -1), (200, 201, 1), (5, 6, -1)]
    per_seq = [iso, []]
    windows = []
    for st, en in ((100, 450), (100, 449), (99, 451), (100, 200), (101, 200), (150, 160), (0, 1000), (150, 171), (200, 201)):
        for rev in (0, 1):
            windows.append((0, st, en - st, rev))
    for ln in range(1, 18):  # lengths 1 to 17, on and around the shared donor
        for st in (99, 100, 150, 184, 199):
            windows.append((0, st, ln, ln & 1))
    windows += [(1, 0, 500, 0), (2, 0, 40, 1), (-1, 0, 16, 0)]  # the empty sequence and two outside the table
    got = _check_batch(per_seq, windows)
    assert got[0][0] == 1 and got[0][99] == 2 and got[0][349] == 2  # the shared donor carries one bit, the three acceptors theirs
    assert got[1][349] == 1 and got[1][0] == 2 and got[1][349 - 99] == 2  # the same window reversed: bytes reversed, bits not


def test_bed_junc_batch_dense_contig():
    """More than 10 000 intervals on one sequence, windows up to 200 kb (many passes of a warp), reversed and not."""
    rng = np.random.default_rng(91)
    st = np.sort(rng.integers(0, 300000, 12000))
    iv = [(int(s), int(s) + int(rng.integers(30, 20000)), int(rng.choice([1, -1, 0]))) for s in st]
    per_seq = [[], iv, [(10, 20, 1)]]
    recs, off = jl.records(per_seq)
    windows = [(rid, st0, ln, int(rng.integers(0, 2))) for rid, st0, ln in random_windows(rng, recs, off, 300)]
    windows += [(1, 0, 200000, 0), (1, 50000, 200000, 1), (0, 0, 1000, 0)]
    got = _check_batch(per_seq, windows)
    assert np.count_nonzero(got[-3]) > 5000


def _mapper(lo, ref, wfile, bed):
    from winnowmap_b200.mapper import Mapper
    mp = Mapper(ref, wfile, preset=lo["preset"], cigar=True, sam=lo.get("sam", False), hpc=lo.get("hpc", False), splice=lo.get("splice", False),
                max_intron_len=lo.get("max_intron_len"), part_bases=lo.get("part_bases"), split=lo.get("split", False), spliced_alignment=True,
                junc_bed=bed)
    mp.mo.flag = (mp.mo.flag | lo.get("set_flags", 0)) & ~lo.get("clear_flags", 0)
    return mp


@pytest.mark.parametrize("name", sorted(jl.MANIFEST))
def test_gpu_junction_alignment_matches_reference(name, tmp_path):
    ref, reads, wfile, bed = jl.inputs(name, str(tmp_path))
    mp = _mapper(jl.MANIFEST[name]["lib"], ref, wfile, bed)
    try:
        junc_stats()
        out = str(tmp_path / "o.out")
        mp.map_file(reads, out)
        n_launch, n_win, _ = junc_stats()
        assert n_launch > 0 and n_win > 0, "the annotation kernel did not run"
    finally:
        mp.close()
    check_output(name, out)


def test_set_junc_with_reference_records_then_map_batch(tmp_path):
    """The reference's own mm_idx_t::I records (the fixture) handed over with wm_idx_set_junc on an index uploaded with
    WM_IDX_JUNC (through the blob, which keeps the flag), then wm_gpu_map_batch + wm_format_batch: the records of splice_junc_c."""
    from winnowmap_b200 import kernels
    from winnowmap_b200.mapper import MapOpt, Mapper
    ref, reads, wfile, bed = jl.inputs("splice_junc_c", str(tmp_path))
    mp = Mapper(ref, wfile, preset="splice", cigar=True, spliced_alignment=True)
    L = mp.L
    try:
        fx = jl.fixture()
        recs, off = fx["full_recs"], fx["full_off"]
        per_seq = [[(int(r[0]), int(r[1]), int(s), int(c)) for r, s, c in zip(recs[a:b], jl.strands(recs[a:b]), jl.scores(recs[a:b]))]
                   for a, b in zip(off[:-1], off[1:])]
        I, keep = kernels.intv_records(per_seq)
        blob = mp.index_blob()
        words = blob.view(np.uint64)
        words[1] |= np.uint64(0x100 << 16)  # the index flag in the blob header: WM_IDX_JUNC
        L.wm_idx_blob_load.restype = C.c_void_p
        ctx = L.wm_idx_blob_load(blob.ctypes.data, blob.nbytes, 0)
        assert ctx
        assert L.wm_idx_set_junc(C.c_void_p(ctx), C.cast(I, C.c_void_p)) == 0
        recs_fa = sa.make_golden.read_fasta(reads)
        n = len(recs_fa)
        names = (C.c_char_p * n)(*[r[0].encode() for r in recs_fa])
        seqs = (C.c_char_p * n)(*[r[1].encode() for r in recs_fa])
        lens = (C.c_int32 * n)(*[len(r[1]) for r in recs_fa])
        n_reg, rep, fg = (C.c_int32 * n)(), (C.c_int32 * n)(), (C.c_int32 * n)()
        reg = (C.c_void_p * n)()
        L.wm_gpu_map_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int]
        assert L.wm_gpu_map_batch(ctx, C.byref(mp.mo), n, names, seqs, lens, n_reg, reg, rep, fg, 8) == 0
        out = str(tmp_path / "o.paf")
        L.wm_format_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_char_p]
        assert L.wm_format_batch(ctx, C.byref(mp.mo), n, names, seqs, lens, n_reg, reg, rep, out.encode()) == 0
        L.wm_free_regs.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        L.wm_free_regs(n, n_reg, reg)
        L.wm_gpu_destroy(C.c_void_p(ctx))
        del keep
    finally:
        mp.close()
    # wm_format_batch writes in input order, the reference a mini-batch by length (as wm_map_file does): the same records
    exp = gzip.open(os.path.join(jl.GOLDEN, "splice_junc_c.paf.gz")).read().split(b"\n")
    assert sorted(open(out, "rb").read().split(b"\n")) == sorted(exp)


def test_no_annotation_without_splice_dp_or_without_bed(tmp_path):
    """junc_bed on a run without spliced base alignment (-x splice without -c: splice_W) and spliced alignment without a BED
    (splice_aln_c): the existing goldens, and no annotation launch."""
    import json
    from winnowmap_b200.mapper import Mapper
    ref, reads, wfile, bed = jl.inputs("splice_junc_c", str(tmp_path))
    man = json.load(open(os.path.join(jl.GOLDEN, "splice_manifest.json")))
    assert man["splice_W"]["reads_md5"] == sa.make_golden.md5(reads)
    junc_stats()
    mp = Mapper(ref, wfile, preset="splice", cigar=False, junc_bed=bed)
    try:
        out = str(tmp_path / "w.paf")
        mp.map_file(reads, out)
    finally:
        mp.close()
    assert open(out, "rb").read() == gzip.open(os.path.join(jl.GOLDEN, "splice_W.paf.gz")).read()
    mp = Mapper(ref, wfile, preset="splice", cigar=True, spliced_alignment=True)
    try:
        out = str(tmp_path / "c.paf")
        mp.map_file(reads, out)
    finally:
        mp.close()
    sa.check_output("splice_aln_c", out)
    assert junc_stats()[0] == 0


def test_missing_bed_raises(tmp_path):
    from winnowmap_b200.mapper import Mapper
    ref, reads, wfile, bed = jl.inputs("splice_junc_c", str(tmp_path))
    with pytest.raises(RuntimeError):
        Mapper(ref, wfile, preset="splice", cigar=True, spliced_alignment=True, junc_bed=str(tmp_path / "none.bed"))
