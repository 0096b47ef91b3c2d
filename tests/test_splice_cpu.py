"""Spliced mapping without base alignment (-x splice / splice:hq / cdna, --splice, -G) on the CPU: the cDNA gap cost of mm_chain_dp
(reference src/chain.c:69-77) in the oracle, in the CPU emulations of the chaining kernels and in the oracle-backed host pipeline,
and the options of the spliced presets.  The oracle's chaining is compared with the reference's own mm_chain_dp(is_cdna = 1) where
the reference's sources and oracle/_ref are present, else with the digests recorded from it in tests/golden/splice_ref_digests.json
(WM_RECORD_REF=1 records).  The harness libraries come from splice_lib.py."""
import ctypes as C
import gzip
import json
import os

import numpy as np
import pytest

import oracle_lib as ol
import splice_lib as S
from test_oracle_vs_ref import make_anchors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MANIFEST = json.load(open(os.path.join(GOLDEN, "splice_manifest.json")))
DIGESTS_FN = os.path.join(GOLDEN, "splice_ref_digests.json")
# chaining arguments of -x splice (src/options.c:116-129, src/map.c:374-389): max_gap_ref = bw = 200000, max_gap = 2000,
# min_gap_ref 1000; and the -G 20000 variant
SPLICE_CHAIN = [(200000, 1000, 2000, 200000, 25, 5000), (20000, 1000, 2000, 20000, 25, 5000), (200000, 1000, 2000, 200000, 3, 300)]

import sys  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden  # noqa: E402

_digests = None


def check_ref(key, got, ref_fn):
    """got (u, b) of the oracle's cDNA chaining equals the reference's mm_chain_dp(is_cdna = 1) on the same input."""
    global _digests
    if _digests is None:
        _digests = json.load(open(DIGESTS_FN)) if os.path.exists(DIGESTS_FN) else {}
    d = ol.digest(*got)
    have_ref = S.ref() is not None
    if have_ref and ol.recording():
        _digests[key] = ol.digest(*ref_fn())
        with open(DIGESTS_FN, "w") as f:
            json.dump(_digests, f, indent=0, sort_keys=True)
            f.write("\n")
    if have_ref:
        assert d == ol.digest(*ref_fn()), key
    assert key in _digests, f"no reference digest for {key} (record with WM_RECORD_REF=1)"
    assert _digests[key] == d, key


def spliced_anchors(rng, n_exons, intron_max=250000, span=15, noise=0):
    """Anchors of one spliced read: a diagonal per exon, the exons separated on the reference by introns (dr > dq: the gaps the cDNA
    cost makes cheap) and a few small indels inside exons; some paralogous copies of exons elsewhere, and `noise` random anchors."""
    xs, ys, q, r = [], [], 100, 100000
    for e in range(n_exons):
        L = int(rng.integers(60, 600))
        pos = np.sort(rng.choice(np.arange(L), size=max(2, L // 12), replace=False))
        shift = np.cumsum(rng.integers(-2, 3, size=len(pos)) * (rng.random(len(pos)) < 0.1))
        xs.append(r + pos + shift), ys.append(q + pos)
        if rng.random() < 0.3:  # a paralogous copy of this exon downstream
            xs.append(r + 400000 + pos), ys.append(q + pos)
        q += L
        r += L + int(np.exp(rng.uniform(np.log(60), np.log(intron_max))))
    if noise:
        xs.append(rng.integers(100000, r, size=noise)), ys.append(rng.integers(100, q, size=noise))
    x, y = np.concatenate(xs).astype(np.int64), np.concatenate(ys).astype(np.int64)
    a = np.stack([x.astype(np.uint64), np.uint64(span) << np.uint64(32) | y.astype(np.uint64)], axis=1)
    return ol.oracle_sort128(a)


def _corpus(seed):
    rng = np.random.default_rng(seed)
    out = [(f"rand{n}", make_anchors(rng, n, repeats=bool(n & 1))) for n in (0, 1, 3, 100, 700, 3000)]
    out += [(f"tx{k}", spliced_anchors(rng, int(rng.integers(2, 30)), noise=int(rng.integers(0, 200)))) for k in range(8)]
    return out


# ---------------------------------------------------------------------------------------------------------------- oracle

@pytest.mark.parametrize("seed", range(3))
def test_oracle_cdna_chain_matches_reference(seed):
    changed = 0
    for name, a in _corpus(5300 + seed):
        for pi, (mx, mn, my, bw, skip, it) in enumerate(SPLICE_CHAIN):
            got = S.oracle_chain_cdna(a, mx, mn, my, bw, max_skip=skip, max_iter=it)
            check_ref(f"cdna:{seed}:{name}:{pi}", got, lambda: S.ref_chain_cdna(a, mx, mn, my, bw, max_skip=skip, max_iter=it))
            plain = ol.oracle_chain(a, mx, mn, my, bw, max_skip=skip, max_iter=it)
            changed += ol.digest(*plain) != ol.digest(*got)
    assert changed > 0  # the cDNA gap cost changes chains on these inputs


# ------------------------------------------------------------------------------------------------------------ emulations

def _fpv(n):
    return [np.zeros(max(n, 1), np.int32) for _ in range(3)]


def _scalar(a, prm, cdna=True):
    out = _fpv(len(a))
    S.emul().wmt_chain_fill_scalar_gap(a.ctypes.data, len(a), *prm, 1.0, int(cdna), *(o.ctypes.data for o in out))
    return out


def _emulated(a, prm, mode, cap=48):
    got = _fpv(len(a))
    assert S.emul().wmt_emul_chain_fill_cdna(a.ctypes.data, len(a), *prm, 1.0, mode, cap, *(o.ctypes.data for o in got)) == 0
    return got


def test_emulated_forward_passes_match_scalar_cdna():
    """Plain warp loop, dense candidates, the rings (64 slots: the older-than-ring path; 1024) and the tile formulation (128-slot
    ring: the locked deep path), each in its cDNA instantiation, against the scalar restatement."""
    differs = 0
    for name, a in _corpus(5400):
        a = np.ascontiguousarray(a)
        for prm in SPLICE_CHAIN:
            exp = _scalar(a, prm)
            differs += any(not np.array_equal(x, y) for x, y in zip(exp, _scalar(a, prm, cdna=False)))
            for mode in range(5):
                for x, y, w in zip(exp, _emulated(a, prm, mode), "fpv"):
                    assert np.array_equal(x[:len(a)], y[:len(a)]), (name, prm, mode, w)
    assert differs > 0


def test_tile_list_cdna_matches_scalar():
    """The tile formulation with lists of 2 and 7 entries (refills, breaks inside and after the first list) and a 128-slot ring."""
    for name, a in _corpus(5500)[3:]:
        a = np.ascontiguousarray(a)
        for prm in SPLICE_CHAIN:
            exp = _scalar(a, prm)
            for cap in (2, 7):
                for x, y, w in zip(exp, _emulated(a, prm, 4, cap), "fpv"):
                    assert np.array_equal(x[:len(a)], y[:len(a)]), (name, prm, cap, w)


def giant_spliced(rng, n_exons=400):
    """A giant spliced task whose 200 kb windows hold more than 4096 anchors: a long read's exons, densely seeded, over a gene
    region shorter than max_dist_x, plus paralogous copies: many anchors have candidates below the tile kernel's ring."""
    return spliced_anchors(rng, n_exons, intron_max=400, noise=300)


@pytest.mark.parametrize("sched", [(0, 0, 0), (2, 31, 0)])
def test_tile_cta_cdna_matches_scalar(sched):
    """The giant-task kernel's CTA body in its cDNA instantiation on an emulated CTA at its real 4096-slot ring: parity, and the
    locked deep path is taken."""
    K = S.cta()
    k = np.zeros(3, np.int32)
    K.wmt_tile_constants_cdna(k.ctypes.data)
    assert tuple(k) == (4096, 48, 32)  # the emulated kernel runs at the product's constants
    a = np.ascontiguousarray(giant_spliced(np.random.default_rng(5600)))
    n = len(a)
    assert n > 6000
    x = a[:, 0].astype(np.int64)
    assert (np.searchsorted(x, x - 200000) < np.arange(n) - 4096).any()  # windows reach more than 4096 anchors back
    prm = np.array(SPLICE_CHAIN[0] + SPLICE_CHAIN[2], np.int32)
    off, order, set_id = np.array([0, n], np.int64), np.zeros(1, np.int32), np.zeros(1, np.uint8)
    got, stats, err = _fpv(n), np.zeros(10, np.int64), C.create_string_buffer(4096)
    rc = K.wmt_tile_cta_cdna(a.ctypes.data, off.ctypes.data, 1, order.ctypes.data, prm.ctypes.data, 1.0, set_id.ctypes.data, *sched,
                             *(o.ctypes.data for o in got), stats.ctypes.data, err, 4096)
    assert rc == 0, err.value
    for e, g, w in zip(_scalar(a, SPLICE_CHAIN[0]), got, "fpv"):
        assert np.array_equal(e[:n], g[:n]), w
    assert stats[0] > 0  # deep scans


# ----------------------------------------------------------------------------------------------------- host pipeline

def splice_inputs(name, tmp):
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_splice_inputs(m["reads"], str(tmp))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    return ref, reads, wfile if m["use_W"] else None


def check_golden(name, got):
    exp = gzip.open(os.path.join(GOLDEN, name + ".paf.gz")).read()
    if got != exp:
        for i, (x, y) in enumerate(zip(exp.split(b"\n"), got.split(b"\n"))):
            assert x == y, f"{name} line {i}: exp {x[:200]!r} got {y[:200]!r}"
        raise AssertionError(f"{name}: line count differs")


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_host_pipeline_matches_splice_golden(name, tmp_path):
    """The product's host orchestration (stage 1 under --splice, the fallback route, chain_post without the long join, the -I merge)
    on the oracle backends, chaining as the ChainParams of the orchestration ask, against the reference's PAF."""
    o = MANIFEST[name]["lib"]
    ref, reads, wfile = splice_inputs(name, tmp_path)
    out = str(tmp_path / "o.paf")
    L = S.pipeline(hpc=bool(o.get("hpc")))
    n = L.wmt_map_file_splice(ref.encode(), wfile.encode() if wfile else None, o["preset"].encode(), int(bool(o.get("splice"))),
                              o.get("max_intron_len", 0), reads.encode(), out.encode(), 8, o.get("part_bases", 0), int(bool(o.get("split"))))
    assert n > (1 if o.get("part_bases") else 0), n
    assert L.wmt_splice_cdna_mismatch() == 0  # both parameter sets of every call carry the same is_cdna
    check_golden(name, open(out, "rb").read())


# ------------------------------------------------------------------------------------------------------------ options

@pytest.fixture(scope="module")
def mapper():
    from winnowmap_b200 import mapper as M
    L = M._setup(M.lib())
    L.wm_mapopt_update.argtypes = [C.POINTER(M.MapOpt), C.c_void_p]
    return M


def _raw(io, mo):
    return bytes(io), bytes(mo)


def test_cdna_and_splice_suffix_equal_splice(mapper):
    """mm_set_opt: "cdna" and any "splice:..." but splice:hq give exactly the options of "splice"; splice:hq differs in its scoring."""
    M = mapper
    base = _raw(*M.make_options("splice", cigar=False))
    for p in ("cdna", "splice:xyz", "splice:"):
        assert _raw(*M.make_options(p, cigar=False)) == base, p
    io, mo = M.make_options("splice", cigar=False)
    assert (io.k, io.w, io.flag) == (15, 25, 0)
    assert mo.flag & (M.F_SPLICE | M.F_SPLICE_FOR | M.F_SPLICE_REV | M.F_SPLICE_FLANK) == M.F_SPLICE | M.F_SPLICE_FOR | M.F_SPLICE_REV | M.F_SPLICE_FLANK
    assert not mo.SVaware and (mo.max_gap, mo.max_gap_ref, mo.bw) == (2000, 200000, 200000)
    assert (mo.a, mo.b, mo.q, mo.e, mo.q2, mo.e2, mo.noncan, mo.junc_bonus, mo.zdrop, mo.zdrop_inv) == (1, 2, 2, 1, 32, 0, 9, 9, 200, 100)
    _, hq = M.make_options("splice:hq", cigar=False)
    assert (hq.junc_bonus, hq.b, hq.q, hq.q2) == (5, 4, 6, 24)
    assert M.make_options("splice:hq", cigar=False)[0].w == 25


def test_max_intron_len_and_mapopt_update_rules(mapper):
    M = mapper
    _, ont = M.make_options("map-ont", cigar=False)
    _, g = M.make_options("map-ont", cigar=False, max_intron_len=20000)  # -G without MM_F_SPLICE: nothing
    assert bytes(g) == bytes(ont)
    _, g = M.make_options("splice", cigar=False, max_intron_len=20000)
    assert (g.max_gap_ref, g.bw) == (20000, 20000)
    _, g = M.make_options("splice", cigar=False, max_intron_len=0)
    assert (g.max_gap_ref, g.bw) == (200000, 200000)
    _, g = M.make_options("map-ont", cigar=False, splice=True, max_intron_len=30000)  # --splice -G
    assert g.flag & M.F_SPLICE and (g.max_gap_ref, g.bw) == (30000, 30000) and g.SVaware
    for bit in (M.F_SPLICE_FOR, M.F_SPLICE_REV):  # mm_mapopt_update: a strand flag implies MM_F_SPLICE
        _, mo = M.make_options("map-ont", cigar=False)
        mo.flag |= bit
        assert M.lib().wm_mapopt_update(C.byref(mo), None) == 0
        assert mo.flag & M.F_SPLICE
    _, mo = M.make_options("map-ont", cigar=False)
    assert M.lib().wm_mapopt_update(C.byref(mo), None) == 0 and not mo.flag & M.F_SPLICE


def test_splice_with_alignment_is_refused(mapper, tmp_path):
    M = mapper
    for kw in (dict(preset="splice"), dict(preset="cdna", sam=True), dict(preset="map-ont", splice=True)):
        with pytest.raises(ValueError, match="alignment"):
            M.make_options(**kw)
        with pytest.raises(ValueError, match="alignment"):
            M.Mapper(str(tmp_path / "absent.fa"), **kw)
    io, mo = M.make_options("splice", cigar=False)
    assert M.lib().wm_check_opt(C.byref(io), C.byref(mo)) == 0
    for f in (M.F_CIGAR | M.F_OUT_CG, M.F_CIGAR | M.F_OUT_SAM):
        mo2 = M.MapOpt.from_buffer_copy(mo)
        mo2.flag |= f
        assert M.lib().wm_check_opt(C.byref(io), C.byref(mo2)) == -8
