"""Homopolymer-compressed minimizers (-H) on the GPU: the HPC sketch kernel against the oracle, the device-built -H
index against the reference's, and end-to-end PAF / SAM against the reference's -H goldens (tests/golden/hpc_*,
made by tools/make_golden.py --hpc)."""
import gzip
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hpc_lib as H  # noqa: E402
import make_golden  # noqa: E402

pytestmark = pytest.mark.gpu
MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "hpc_manifest.json")))


def _golden(name, suffix=".paf.gz"):
    return gzip.open(os.path.join(ROOT, "tests", "golden", name + suffix)).read()


def _first_diff(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
    return f"line count {len(la)} vs {len(lb)}"


def _map(name, tmp_path, **kw):
    from winnowmap_b200.mapper import Mapper
    m = MANIFEST[name]
    ref, reads, wfile = make_golden.make_hpc_inputs(name, str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"], "synthetic input generator drifted"
    mp = Mapper(ref, wfile, preset=m["params"]["preset"], hpc=True, **kw)
    out = str(tmp_path / "out")
    mp.map_file(reads, out)
    return mp, open(out, "rb").read()


@pytest.mark.parametrize("k,w", [(15, 10), (15, 50), (16, 10), (19, 25), (28, 5)])
def test_hpc_sketch_matches_oracle(k, w):
    from winnowmap_b200 import kernels
    seqs = H.crafted_sequences() + H.random_sequences(11 + k, 1200)  # about 2 Mbase of homopolymer-rich reads
    kmers = H.hpc_kmers(seqs, k, 300, seed=k)
    gb, ob = kernels.Bloom(kmers), H.HpcBloom(kmers)
    rids = np.arange(len(seqs), dtype=np.uint32)
    got = kernels.sketch_batch(gb, seqs, w, k, rids, hpc=True)
    n_long = 0
    for i, s in enumerate(seqs):
        exp = H.oracle_sketch_hpc(s, w, k, i, ob)
        assert np.array_equal(got[i], exp), (i, len(s), len(got[i]), len(exp))
        n_long += int((exp[:, 0] & np.uint64(0xff) > np.uint64(k)).sum())
    assert n_long > 0  # spans above k: the position map is exercised


def _blob_index(blob):
    """keys, pos_off, pos and the index flag from a context blob (layout: csrc/capi_map.cu wm_idx_blob_write)."""
    h = blob[:64].view(np.uint64)
    n_seq, names, s_words, n_keys, n_pos = (int(h[i]) for i in (2, 3, 4, 5, 6))
    pad8 = lambda x: (x + 7) & ~7  # noqa: E731
    o = 64 + pad8(n_seq * 4) + n_seq * 8 + pad8(names) + pad8(s_words * 4)
    keys = blob[o:o + 8 * n_keys].view(np.uint64)
    o += 8 * n_keys
    poff = blob[o:o + 8 * (n_keys + 1)].view(np.uint64)
    o += 8 * (n_keys + 1)
    pos = blob[o:o + 8 * n_pos].view(np.uint64)
    return keys.copy(), poff.copy(), pos.copy(), int(h[1]) >> 16 & 0xffff


@pytest.mark.parametrize("name", ["hpc_clr", "hpc_ont_small"])
def test_hpc_index_matches_reference(name, tmp_path):
    from winnowmap_b200.mapper import Mapper, make_options
    ref, _, _ = make_golden.make_hpc_inputs(name, str(tmp_path))
    io, _ = make_options(MANIFEST[name]["params"]["preset"])
    mp = Mapper(ref, None, preset=MANIFEST[name]["params"]["preset"], hpc=True)
    assert mp.hpc
    keys, poff, pos, flag = _blob_index(mp.index_blob())
    mp.close()
    assert flag == 1
    H.assert_ref(f"hpc_index_{name}", (keys, poff, pos), lambda: H.ref_index_hpc(ref, None, io.k, io.w))


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_hpc_paf_matches_reference(name, tmp_path):
    mp, got = _map(name, tmp_path)
    st = mp.stats()
    mp.close()
    assert st["n_dp_jobs"] > 0
    exp = _golden(name)
    assert got == exp, _first_diff(exp, got)


@pytest.mark.parametrize("name", [n for n in sorted(MANIFEST) if MANIFEST[n].get("sam_md5")])
def test_hpc_sam_matches_reference(name, tmp_path):
    mp, got = _map(name, tmp_path, sam=True)
    mp.close()
    got = make_golden.sam_without_pg(got)
    if hashlib.md5(got).hexdigest() != MANIFEST[name]["sam_md5"]:
        exp = _golden(name, ".sam.stripped.gz")
        got = make_golden.sam_strip_seq(got)
        assert got == exp, _first_diff(exp, got)
        pytest.fail("SEQ/QUAL differ")


@pytest.mark.parametrize("name,chunk,lanes", [("hpc_ont_small", 150000, 4), ("hpc_clr", 60000, 3)])
def test_hpc_paf_independent_of_lane_chunking(name, chunk, lanes, tmp_path, monkeypatch):
    monkeypatch.setenv("WM_CHUNK_BASES", str(chunk))
    monkeypatch.setenv("WM_LANES", str(lanes))
    mp, got = _map(name, tmp_path)
    mp.close()
    exp = _golden(name)
    assert got == exp, _first_diff(exp, got)


def test_hpc_blob_round_trip(tmp_path):
    """The flag travels in the blob: a context re-created from it maps with -H."""
    from winnowmap_b200.mapper import Mapper
    name = "hpc_clr"
    mp, _ = _map(name, tmp_path)
    blob = mp.index_blob()
    mp.close()
    _, reads, wfile = make_golden.make_hpc_inputs(name, str(tmp_path))
    mp2 = Mapper(None, None, preset=MANIFEST[name]["params"]["preset"], blob=blob)
    assert mp2.hpc
    out = str(tmp_path / "blob.paf")
    mp2.map_file(reads, out)
    mp2.close()
    got, exp = open(out, "rb").read(), _golden(name)
    assert got == exp, _first_diff(exp, got)


def test_plain_blob_unchanged(tmp_path):
    """Without -H the blob header keeps its old form: no flag bits in the second word."""
    from winnowmap_b200.mapper import Mapper
    ref, _, _ = make_golden.make_hpc_inputs("hpc_clr", str(tmp_path))
    mp = Mapper(ref, None, preset="map-pb-clr")
    assert not mp.hpc
    h = mp.index_blob()[:64].view(np.uint64)
    mp.close()
    assert int(h[1]) == (15 << 32 | 50)
