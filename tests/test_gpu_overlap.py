"""Self and all-vs-all mapping (-D, --dual=no, -X) and single-strand mapping (--for-only, --rev-only) on the GPU: the seed
filter of the expand kernel and its stable compaction (csrc/seed.cu), end to end against the reference's goldens
(tests/golden/overlap_*, made by tools/make_golden.py --overlap)."""
import ctypes as C
import gzip
import hashlib
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import make_golden  # noqa: E402

pytestmark = pytest.mark.gpu
MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "overlap_manifest.json")))
PAF_CASES = sorted(n for n in MANIFEST if not MANIFEST[n]["lib"].get("sam"))


def _golden(name, suffix=".paf.gz"):
    return gzip.open(os.path.join(ROOT, "tests", "golden", name + suffix)).read()


def _first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
    return f"line count {len(la)} vs {len(lb)}"


def _inputs(name, tmp_path):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_overlap_inputs(m["inputs"], str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    return ref, reads, wfile


def _mapper(name, ref, wfile):
    from winnowmap_b200.mapper import Mapper
    return Mapper(ref, wfile, **MANIFEST[name]["lib"])


def _map(name, tmp_path, **kw):
    ref, reads, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile)
    out = str(tmp_path / "out")
    mp.map_file(reads, out, **kw)
    mp.close()
    return open(out, "rb").read()


@pytest.mark.parametrize("name", PAF_CASES)
def test_overlap_paf_matches_reference(name, tmp_path):
    got, exp = _map(name, tmp_path), _golden(name)
    assert got == exp, _first_diff(exp, got)


@pytest.mark.parametrize("name", sorted(n for n in MANIFEST if MANIFEST[n]["lib"].get("sam")))
def test_overlap_sam_matches_reference(name, tmp_path):
    got = make_golden.sam_without_pg(_map(name, tmp_path))
    if hashlib.md5(got).hexdigest() != MANIFEST[name]["sam_md5"]:
        exp = _golden(name, ".sam.stripped.gz")
        got = make_golden.sam_strip_seq(got)
        assert got == exp, _first_diff(exp, got)
        pytest.fail("SEQ/QUAL differ")


@pytest.mark.parametrize("name,chunk,lanes", [("overlap_ava_X_c", 150000, 4), ("overlap_ava_D_c", 60000, 3), ("overlap_tandem_rev_only", 100000, 2)])
def test_overlap_paf_independent_of_lane_chunking(name, chunk, lanes, tmp_path, monkeypatch):
    monkeypatch.setenv("WM_CHUNK_BASES", str(chunk))
    monkeypatch.setenv("WM_LANES", str(lanes))
    got, exp = _map(name, tmp_path), _golden(name)
    assert got == exp, _first_diff(exp, got)


def test_overlap_shards_merge_to_golden(tmp_path):
    """-X with world = 2: the filter depends on the read and the index only, so the tagged shards merge back to the golden."""
    name = "overlap_ava_X_c"
    ref, reads, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile)
    lines = []
    for rank in range(2):
        out = str(tmp_path / f"shard{rank}")
        mp.map_file(reads, out, rank=rank, world=2, tag_order=True)
        for ln in open(out, "rb").read().split(b"\n")[:-1]:
            b, p, rest = ln.split(b"\t", 2)
            lines.append((int(b), int(p), rest))
    mp.close()
    lines.sort(key=lambda t: (t[0], t[1]))  # stable: the records of one read keep their order
    got = b"".join(r + b"\n" for _, _, r in lines)
    exp = _golden(name)
    assert got == exp, _first_diff(exp, got)


def _lib():
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import MapOpt, _setup
    L = _setup(lib())
    L.wm_gpu_map_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    L.wm_format_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_int32),
                                  C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_char_p]
    L.wm_free_regs.argtypes = [C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]
    L.wm_map.restype = C.c_void_p
    L.wm_map.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(MapOpt), C.c_char_p]
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    return L


def _map_one(L, mp, mo, nm, s, qname, out):
    """wm_map of one read with name `qname` (None: NULL), formatted under the name nm."""
    n = C.c_int(0)
    reg = L.wm_map(mp.ctx, len(s), s, C.byref(n), None, C.byref(mo), qname)
    names = (C.c_char_p * 1)(nm); seqs = (C.c_char_p * 1)(s); lens = (C.c_int32 * 1)(len(s))
    n_reg = (C.c_int32 * 1)(n.value); regs = (C.c_void_p * 1)(reg); rl = (C.c_int32 * 1)(0)
    L.wm_format_batch(mp.ctx, C.byref(mo), 1, names, seqs, lens, n_reg, regs, rl, out.encode())
    L.wm_free_regs(1, n_reg, regs)
    return open(out, "rb").read()


def test_wm_map_without_name_applies_no_name_test(tmp_path):
    """wm_map(name = NULL) is mm_map with qname == 0: under -X the name tests are off, so the records are those of -P
    --no-long-join (-X without the seed filter), also without a name (the name seeds the tie-breaking hash); with the name,
    the self-hit goes."""
    from winnowmap_b200.mapper import F_ALL_CHAINS, F_NO_LJOIN, make_options
    L = _lib()
    name = "overlap_ava_X_c"
    ref, reads, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile)
    _, mo_plain = make_options("map-ont")
    mo_plain.flag |= F_ALL_CHAINS | F_NO_LJOIN
    recs = make_golden.read_fasta(reads)
    recs = [recs[i] for i in (0, 1, 2, 3)] + [max(recs, key=lambda r: len(r[1]))]
    n_self = 0
    for nm, s in recs:
        nm, s = nm.split()[0].encode(), s.encode()
        unnamed = _map_one(L, mp, mp.mo, nm, s, None, str(tmp_path / "a"))
        plain = _map_one(L, mp, mo_plain, nm, s, None, str(tmp_path / "b"))
        named = _map_one(L, mp, mp.mo, nm, s, nm, str(tmp_path / "c"))
        assert unnamed == plain, _first_diff(plain, unnamed)
        assert all(ln.split(b"\t")[5] != nm for ln in named.split(b"\n")[:-1])
        n_self += sum(ln.split(b"\t")[5] == nm for ln in unnamed.split(b"\n")[:-1])
    mp.close()
    assert n_self > 0  # without a name the reads find themselves


def _launches(L, mp, reads, out):
    L.wm_prof_reset()
    mp.map_file(reads, out)
    o = (C.c_double * 13)()
    L.wm_prof_get(o)
    return o[0]


def test_filter_launches_only_with_a_filter_option(tmp_path):
    """The filter's kernels (its expand instance, the scan and the compaction) run only with a filter option: the plain run
    still gives the reference's golden, and --for-only launches more kernels than it."""
    from winnowmap_b200.mapper import Mapper
    L = _lib()
    ref, reads, wfile = make_golden.make_inputs("ont_small", str(tmp_path))
    out = str(tmp_path / "o.paf")
    a = Mapper(ref, wfile, preset="map-ont")
    n_plain = _launches(L, a, reads, out)
    a.close()
    assert open(out, "rb").read() == gzip.open(os.path.join(ROOT, "tests", "golden", "ont_small.paf.gz")).read()
    c = Mapper(ref, wfile, preset="map-ont", strand="for")
    n_filter = _launches(L, c, reads, out)
    c.close()
    assert n_filter > n_plain > 0
