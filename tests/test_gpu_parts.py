"""Multi-part indexes (-I), --split-prefix merging and -f on the GPU: part-major and merged output byte-identical to the
reference's goldens (tests/golden/parts_*, made by tools/make_golden.py --parts), the per-part mid_occ the device selection
gives (csrc/occ_select.cu) against the reference's and the plain-C oracle's, and the borrowed per-part handles."""
import ctypes as C
import gzip
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]
import make_golden  # noqa: E402
from test_parts_host import cal_max_occ  # noqa: E402

pytestmark = pytest.mark.gpu
MAN = json.load(open(os.path.join(ROOT, "tests", "golden", "parts_manifest.json")))
CASES = MAN["cases"]


class IdxView(C.Structure):  # wm_idx_view_t
    _fields_ = [("k", C.c_int32), ("w", C.c_int32), ("n_seq", C.c_int32), ("seq_name", C.POINTER(C.c_char_p)), ("seq_len", C.c_void_p),
                ("seq_offset", C.c_void_p), ("S", C.c_void_p), ("S_words", C.c_uint64), ("n_keys", C.c_int64), ("keys", C.c_void_p),
                ("pos_off", C.c_void_p), ("pos", C.c_void_p), ("bloom_bits", C.c_uint64), ("bloom_table", C.c_void_p)]


def _lib():
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import MapOpt, _setup
    L = _setup(lib())
    L.wm_gpu_map_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]
    L.wm_format_batch.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_int32),
                                  C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_char_p]
    L.wm_free_regs.argtypes = [C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]
    L.wm_gpu_idx_upload.restype = C.c_void_p
    L.wm_gpu_idx_upload.argtypes = [C.POINTER(IdxView), C.c_int]
    L.wm_bloom_build.restype = C.c_void_p
    L.wm_bloom_build.argtypes = [C.c_void_p, C.c_int64]
    L.wm_bloom_bits.restype = C.c_uint64
    L.wm_bloom_bits.argtypes = [C.c_void_p]
    L.wm_bloom_table.restype = C.c_void_p
    L.wm_bloom_table.argtypes = [C.c_void_p]
    L.wm_bloom_destroy.argtypes = [C.c_void_p]
    L.wm_idx_n_seq.argtypes = [C.c_void_p]
    L.wm_idx_seq_name.restype = C.c_char_p
    L.wm_idx_seq_name.argtypes = [C.c_void_p, C.c_int]
    return L


def _golden(name, suffix=".paf.gz"):
    return gzip.open(os.path.join(ROOT, "tests", "golden", name + suffix)).read()


def _first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
    return f"line count {len(la)} vs {len(lb)}"


def _inputs(name, tmp_path):
    m = CASES[name]
    ref, reads, wfile = make_golden.make_parts_inputs(m["inputs"], str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    assert (make_golden.md5(wfile) if wfile else None) == m["w_md5"]
    return ref, reads, wfile


def _mapper(name, ref, wfile, **kw):
    from winnowmap_b200.mapper import Mapper
    return Mapper(ref, wfile, **dict(CASES[name]["lib"], **kw))


def _check(name, got):
    if CASES[name]["lib"].get("sam"):
        got = make_golden.sam_without_pg(got)
        if hashlib.md5(got).hexdigest() != CASES[name]["sam_md5"]:
            exp, got = _golden(name, ".sam.stripped.gz"), make_golden.sam_strip_seq(got)
            assert got == exp, _first_diff(exp, got)
            pytest.fail("SEQ/QUAL differ")
    else:
        exp = _golden(name)
        assert got == exp, _first_diff(exp, got)


def _map(name, tmp_path, mapper_kw=None, **kw):
    ref, reads, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile, **(mapper_kw or {}))
    assert mp.n_parts == len(CASES[name]["n_seq"])
    out = str(tmp_path / "out")
    mp.map_file(reads, out, **kw)
    mp.close()
    return open(out, "rb").read()


@pytest.mark.parametrize("name", sorted(CASES))
def test_parts_match_reference(name, tmp_path):
    """Part-major and merged output, SAM headers (@PG only; merged @SQ; a single part's @SQ twice), -X, -H and -f."""
    _check(name, _map(name, tmp_path))


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]["lib"].get("mid_occ_frac") is not None))
def test_mid_occ_per_part_matches_reference(name, tmp_path):
    """wm_mapopt_update on each part gives the mid_occ the reference printed for that part (src/main.c:403)."""
    from winnowmap_b200.mapper import make_options
    L = _lib()
    ref, _, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile)
    got = []
    for i in range(mp.n_parts):
        part = L.wm_idx_part(mp.ctx, i)
        _, mo = make_options("map-ont")
        mo.mid_occ_frac = CASES[name]["lib"]["mid_occ_frac"]
        assert L.wm_mapopt_update(C.byref(mo), part) == 0
        got.append(mo.mid_occ)
        assert L.wm_idx_cal_max_occ(part, mo.mid_occ_frac) == mo.mid_occ  # min_mid_occ does not bind here
    assert L.wm_idx_part(mp.ctx, mp.n_parts) is None
    mp.close()
    assert got == CASES[name]["mid_occ"]


def test_cal_max_occ_per_part_matches_reference(tmp_path):
    """Every part of every recorded parts input, every recorded f: the device selection equals the reference's function."""
    L = _lib()
    from winnowmap_b200.mapper import Mapper
    for key, rec in sorted(MAN["occ"].items()):
        ref, _, wfile = make_golden.make_parts_inputs(rec["inputs"], str(tmp_path))
        mp = Mapper(ref, wfile, preset="map-ont", part_bases=rec["I"], hpc=bool(rec["flag"]))
        assert [L.wm_idx_n_seq(L.wm_idx_part(mp.ctx, i)) for i in range(mp.n_parts)] == [p["n_seq"] for p in rec["parts"]]
        for i, p in enumerate(rec["parts"]):
            part = L.wm_idx_part(mp.ctx, i)
            for f, want in p["max_occ"].items():
                assert L.wm_idx_cal_max_occ(part, float(f)) == want, (key, i, f)
            assert L.wm_idx_cal_max_occ(part, 1e-30) == -1  # the rank reaches n: refused
        if mp.n_parts > 1:
            assert L.wm_idx_cal_max_occ(mp.ctx, 0.01) == -1  # one value per part
        mp.close()


def _upload_counts(L, counts):
    """A crafted index whose keys have the given occurrence counts."""
    counts = np.asarray(counts, np.uint64)
    n = len(counts)
    keys = np.arange(1, n + 1, dtype=np.uint64) * 7919
    pos_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    pos = np.zeros(int(pos_off[-1]), np.uint64)
    names = (C.c_char_p * 1)(b"s0")
    seq_len, seq_off, S = np.array([1000], np.uint32), np.array([0], np.uint64), np.zeros(125, np.uint32)
    b = L.wm_bloom_build(None, 0)
    v = IdxView(15, 10, 1, names, seq_len.ctypes.data, seq_off.ctypes.data, S.ctypes.data, len(S), n, keys.ctypes.data,
                pos_off.ctypes.data, pos.ctypes.data, L.wm_bloom_bits(b), L.wm_bloom_table(b))
    ctx = L.wm_gpu_idx_upload(C.byref(v), 0)
    L.wm_bloom_destroy(b)
    assert ctx
    return ctx


def test_device_selection_on_crafted_counts():
    """The radix selection against the oracle: all counts equal, heavy ties, counts >= 2^16 and >= 2^24 (every digit of the
    selection decides), n = 1, and ranks 0 and n - 1."""
    L = _lib()
    rng = np.random.default_rng(11)
    sets = {
        "all_equal": np.full(5000, 7),
        "heavy_ties": np.where(rng.random(20000) < 0.9, 3, rng.integers(1, 50, 20000)),
        "wide": np.concatenate([rng.integers(1, 5, 3000), [65536, 65537, 70000, 1 << 24, (1 << 24) + 3, 300, 255, 256]]),
        "single": np.array([42]),
        "two_bytes_tie": np.concatenate([np.full(100, 0x10203), np.full(100, 0x10204), np.full(50, 0x20203)]),
    }
    for name, cnt in sets.items():
        cnt = rng.permutation(cnt).astype(np.uint32)
        n = len(cnt)
        ctx = _upload_counts(L, cnt)
        fs = [0.0, 0.0002, 0.01, 0.1, 0.5, 0.9, 0.9999, 0.5 / n, 1e-30]  # 0.9999 and 0.5 / n: ranks 0 and n - 1
        for f in fs:
            want = cal_max_occ(cnt, f)
            assert L.wm_idx_cal_max_occ(ctx, f) == want, (name, f, want)
        assert cal_max_occ(cnt, 0.9999) == int(cnt.min()) + 1 and cal_max_occ(cnt, 0.5 / n) == int(cnt.max()) + 1
        L.wm_gpu_destroy(ctx)


def test_distinct_with_parts_equals_list_file(tmp_path):
    """distinct= counts the -W list over the whole reference once; the parts built from it map exactly as parts built from the
    file write_top_kmers writes."""
    from winnowmap_b200.mapper import Mapper, write_top_kmers
    ref, reads, _ = _inputs("parts_ont_c", tmp_path)
    lst = str(tmp_path / "list.txt")
    write_top_kmers(ref, lst, 15, 0.9998)
    outs = []
    for kw in (dict(distinct=0.9998), dict(kmer_freq=lst)):
        for split in (False, True):
            mp = Mapper(ref, preset="map-ont", part_bases=330000, split=split, **kw)
            assert mp.n_parts == 3
            out = str(tmp_path / "o")
            mp.map_file(reads, out)
            outs.append(open(out, "rb").read())
            mp.close()
    assert outs[0] == outs[2] and outs[1] == outs[3] and outs[0].count(b"\n") > 0


@pytest.mark.parametrize("chunk,lanes", [(60000, 3), (200000, 1)])
def test_merged_independent_of_lanes(chunk, lanes, tmp_path, monkeypatch):
    monkeypatch.setenv("WM_CHUNK_BASES", str(chunk))
    monkeypatch.setenv("WM_LANES", str(lanes))
    _check("parts_ont_c_split", _map("parts_ont_c_split", tmp_path))


def test_merged_shards_merge_to_golden(tmp_path):
    """world = 2 in merged mode: the merge is per read, so the tagged shards merge back to the golden."""
    name = "parts_ont_c_split"
    ref, reads, wfile = _inputs(name, tmp_path)
    mp = _mapper(name, ref, wfile)
    lines = []
    for rank in range(2):
        out = str(tmp_path / f"shard{rank}")
        mp.map_file(reads, out, rank=rank, world=2, tag_order=True)
        for ln in open(out, "rb").read().split(b"\n")[:-1]:
            b, p, rest = ln.split(b"\t", 2)
            lines.append((int(b), int(p), rest))
    with pytest.raises(RuntimeError):  # part-major output does not shard
        from winnowmap_b200.mapper import Mapper
        pm = Mapper(ref, wfile, preset="map-ont", part_bases=330000)
        try:
            pm.map_file(reads, str(tmp_path / "x"), rank=0, world=2)
        finally:
            pm.close()
    mp.close()
    lines.sort(key=lambda t: (t[0], t[1]))
    got = b"".join(r + b"\n" for _, _, r in lines)
    exp = _golden(name)
    assert got == exp, _first_diff(exp, got)


def _batch(L, ctx, mo, recs, out):
    n = len(recs)
    names = (C.c_char_p * n)(*[nm.encode() for nm, _ in recs])
    seqs = (C.c_char_p * n)(*[s for _, s in recs])
    lens = (C.c_int32 * n)(*[len(s) for _, s in recs])
    n_reg = (C.c_int32 * n)(); regs = (C.c_void_p * n)(); rl = (C.c_int32 * n)(); fg = (C.c_int32 * n)()
    rc = L.wm_gpu_map_batch(ctx, C.byref(mo), n, names, seqs, lens, n_reg, regs, rl, fg, 8)
    if rc != 0:
        return rc
    assert L.wm_format_batch(ctx, C.byref(mo), n, names, seqs, lens, n_reg, regs, rl, out.encode()) == 0
    L.wm_free_regs(n, n_reg, regs)
    return 0


def test_map_batch_per_part_and_merged(tmp_path):
    """wm_gpu_map_batch on wm_idx_part(ctx, i) gives part i's slice of the part-major golden; on the whole context it gives
    the merged golden under split_prefix and is refused without it."""
    L = _lib()
    ref, reads, wfile = _inputs("parts_ont_c", tmp_path)
    mp = _mapper("parts_ont_c", ref, wfile)
    recs = make_golden.read_fasta(reads)
    order = sorted(range(len(recs)), key=lambda i: (len(recs[i][1]), i), reverse=True)  # one mini-batch, longest first
    recs = [(recs[i][0].split()[0], recs[i][1].encode()) for i in order]
    exp = _golden("parts_ont_c").split(b"\n")[:-1]
    out = str(tmp_path / "b")
    start = 0
    for i in range(mp.n_parts):
        part = L.wm_idx_part(mp.ctx, i)
        assert _batch(L, part, mp.mo, recs, out) == 0
        got = open(out, "rb").read().split(b"\n")[:-1]
        names = {L.wm_idx_seq_name(part, j) for j in range(L.wm_idx_n_seq(part))}
        assert all(ln.split(b"\t")[5] in names for ln in got) and got
        assert got == exp[start:start + len(got)], (i, _first_diff(b"\n".join(exp[start:start + len(got)]), b"\n".join(got)))
        start += len(got)
    assert start == len(exp)
    assert _batch(L, mp.ctx, mp.mo, recs, out) == -1
    mo = mp.mo
    mo.split_prefix = b"x"
    assert _batch(L, mp.ctx, mo, recs, out) == 0
    assert open(out, "rb").read() == _golden("parts_ont_c_split")
    mp.close()


def test_reads_without_seed_hit(tmp_path):
    """A wave in which no read has a seed hit (here every chunk of a part-major pass under small chunks, and a file of random
    reads against one index) chains nothing and prints nothing."""
    import gen_data
    from winnowmap_b200.mapper import Mapper
    ref, _, wfile = make_golden.make_inputs("ont_small", str(tmp_path))
    reads = str(tmp_path / "random.fa")
    rng = np.random.default_rng(5)
    gen_data.write_fasta(reads, [(f"rnd{i}", gen_data.random_seq(rng, 3000 + 500 * i)) for i in range(6)])
    mp = Mapper(ref, wfile, preset="map-ont")
    out = str(tmp_path / "o")
    mp.map_file(reads, out)
    mp.close()
    assert open(out, "rb").read() == b""


@pytest.mark.parametrize("name", ["parts_ont_c", "parts_ont_a_split"])
def test_parts_small_chunks(name, tmp_path, monkeypatch):
    """Chunks of a few reads: in part-major and merged passes many chunks have no hit at all in a part."""
    monkeypatch.setenv("WM_CHUNK_BASES", "30000")
    monkeypatch.setenv("WM_LANES", "2")
    _check(name, _map(name, tmp_path))


def test_multi_part_refusals(tmp_path):
    from winnowmap_b200.mapper import Mapper
    ref, reads, wfile = _inputs("parts_ont_c", tmp_path)
    mp = Mapper(ref, wfile, preset="map-ont", part_bases=330000)
    with pytest.raises(RuntimeError):
        mp.index_blob()
    mp.close()
    one = Mapper(ref, wfile, preset="map-ont", part_bases=10 ** 9)  # -I above the reference: an ordinary index
    assert one.n_parts == 1 and len(one.index_blob()) > 0
    one.close()
