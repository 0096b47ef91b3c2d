"""The -W list counted on the GPU (csrc/topfreq.cu, wm_topfreq / wm_index_build_topfreq) against the plain-C oracle
(oracle/wm_oracle_topfreq.c) and the meryl stand-in, and whole runs through Mapper(distinct=...) against the reference
binary's goldens, which it made from the stand-in's list."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen_data  # noqa: E402
import make_golden  # noqa: E402
import topfreq_lib as T  # noqa: E402

pytestmark = pytest.mark.gpu
MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "manifest.json")))
LIST_CASES = sorted(n for n, c in make_golden.CASES.items() if c["use_W"])


def _inputs(tmp_path):
    """name -> (fasta, contigs, k, distinct) of every reference the list comparisons run on"""
    rng = np.random.default_rng(77)
    out = {}
    for k in (15, 16, 19, 21, 28):
        c = T.genome(200 + k, k)
        out[f"genome_k{k}"] = (c, k, 0.9998)
        out[f"genome_k{k}_d09"] = (c, k, 0.9)
    tandem = [(n, s.tobytes()) for n, s in gen_data.make_ref(rng, 3_000_000, 3, True)]
    out["tandem_k15"] = (tandem, 15, 0.9998)
    out["tandem_k24"] = (tandem, 24, 0.9998)
    # counts far above the small-count bins of the histogram: 3 Mbp of one 37-base unit, with random flanks; at 0.9998 the
    # threshold is one of the unit's counts, at 0.99 it is 1 and the unit's k-mers are listed
    unit = gen_data.random_seq(rng, 37).tobytes()
    one = [("u", gen_data.random_seq(rng, 5000).tobytes() + unit * 81000), ("r", gen_data.random_seq(rng, 20000).tobytes())]
    out["one_unit"] = (one, 17, 0.9998)
    out["one_unit_d099"] = (one, 17, 0.99)
    out["empty"] = ([], 15, 0.9998)
    out["all_n"] = ([("n1", b"N" * 5000), ("n2", b"n" * 40)], 15, 0.9998)
    return {name: (T.write_fasta(str(tmp_path / f"{name}.fa"), c), c, k, d) for name, (c, k, d) in out.items()}


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    return _inputs(tmp_path_factory.mktemp("topfreq"))


def _blob(mp):
    """The index blob with its padding bytes zeroed (Mapper.index_blob leaves them as the allocator found them)."""
    buf = np.zeros(mp.L.wm_idx_blob_size(mp.ctx), dtype=np.uint8)
    mp.L.wm_idx_blob_write(mp.ctx, buf.ctypes.data)
    return buf


def _check(name, got, contigs, k, distinct):
    kmers, counts, thr = got
    ek, ec, ethr, _ = T.oracle_top_kmers(contigs, k, distinct)
    assert thr == ethr, (name, thr, ethr)
    assert np.array_equal(kmers, ek) and np.array_equal(counts, ec), (name, len(kmers), len(ek))


def test_device_list_matches_oracle(cases):
    from winnowmap_b200.mapper import top_kmers
    for name, (fa, contigs, k, d) in cases.items():
        _check(name, top_kmers(fa, k, d), contigs, k, d)
    assert top_kmers(cases["one_unit"][0], 17, 0.99)[1].max() > 80000
    assert top_kmers(cases["empty"][0], 15)[0].size == 0 and top_kmers(cases["all_n"][0], 15)[0].size == 0


_CHILD = r'''
import sys, numpy as np
sys.path.insert(0, %r)
from winnowmap_b200.mapper import top_kmers
out = {}
for i, a in enumerate(sys.argv[2:]):
    fa, k, d = a.split(",")
    km, c, t = top_kmers(fa, int(k), float(d))
    out["k%%d" %% i], out["c%%d" %% i], out["t%%d" %% i] = km, c, np.array([t])
np.savez(sys.argv[1], **out)
''' % ROOT


@pytest.mark.parametrize("part_kmers", [5000, 150000])
def test_device_list_with_many_partitions(cases, part_kmers, tmp_path):
    """WM_TOPFREQ_PART_KMERS caps a partition at a few thousand k-mers: the small references split into hundreds of
    partitions (a bucket larger than the cap, e.g. the one unit's, makes a partition of its own), and the list is
    recounted partition by partition in the second sweep."""
    names = list(cases)
    dst = str(tmp_path / "o.npz")
    args = [f"{cases[n][0]},{cases[n][2]},{cases[n][3]}" for n in names]
    env = dict(os.environ, WM_TOPFREQ_PART_KMERS=str(part_kmers))
    subprocess.run([sys.executable, "-c", _CHILD, dst] + args, env=env, check=True, timeout=900)
    z = np.load(dst)
    for i, n in enumerate(names):
        fa, contigs, k, d = cases[n]
        _check(n, (z[f"k{i}"], z[f"c{i}"], int(z[f"t{i}"][0])), contigs, k, d)


def test_bad_arguments_are_refused(cases):
    from winnowmap_b200.mapper import Mapper, top_kmers
    fa = cases["genome_k15"][0]
    for k, d in ((0, 0.9998), (29, 0.9998), (15, 0.0), (15, 1.5)):
        with pytest.raises(ValueError):
            top_kmers(fa, k, d)
    with pytest.raises(ValueError):
        Mapper(fa, fa, distinct=0.9998)
    with pytest.raises(ValueError):
        Mapper(fa, distinct=2.0)


def test_empty_references_build_like_an_empty_list(cases):
    """No k-mer at all: the bloom filter is sized as for an empty -W file, so the blob equals the one built without a list."""
    from winnowmap_b200.mapper import Mapper
    for name in ("empty", "all_n"):
        fa = cases[name][0]
        a = Mapper(fa, distinct=0.9998)
        b = Mapper(fa)
        assert np.array_equal(_blob(a), _blob(b))
        assert a.stats()["n_topfreq"] == 0
        a.close(); b.close()


@pytest.mark.parametrize("name", LIST_CASES)
def test_golden_runs_through_distinct(name, tmp_path):
    """The golden case mapped with the list counted on the device: byte-identical to the reference binary fed the stand-in's
    list, after checking that both lists are the same.  The index blob equals the one built from the stand-in's file."""
    from winnowmap_b200.mapper import Mapper, top_kmers
    import ctypes as C
    m, c = MANIFEST[name], make_golden.CASES[name]
    d = c.get("w_distinct", 0.9998)
    ref, reads, wfile = make_golden.make_inputs(name, str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"]
    kmers, counts, _ = top_kmers(ref, c["k"], d)
    wk, wc = T.read_list(wfile)
    assert np.array_equal(kmers, wk) and np.array_equal(counts, wc)
    mp = Mapper(ref, preset=m["params"]["preset"], cigar=True, distinct=d)
    make_golden.apply_scoring(mp.mo, m["params"])
    assert mp.L.wm_check_opt(C.byref(mp.io), C.byref(mp.mo)) == 0
    st = mp.stats()
    assert st["n_topfreq"] == len(wk) and st["topfreq_threshold"] > 1
    out = str(tmp_path / "out.paf")
    mp.map_file(reads, out)
    blob = _blob(mp)
    mp.close()
    exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".paf.gz")).read()
    assert open(out, "rb").read() == exp
    fb = Mapper(ref, wfile, preset=m["params"]["preset"])
    assert np.array_equal(blob, _blob(fb))
    fb.close()


def test_hpc_index_counts_the_uncompressed_reference(tmp_path):
    """-H with distinct=: the list is the one meryl gives on ref.fa (uncompressed), the filter is probed with the compressed
    k-mers: the blob equals the -H blob built from the stand-in's file."""
    from winnowmap_b200.mapper import Mapper
    ref, _, wfile = make_golden.make_inputs("ont_tandem", str(tmp_path))
    a = Mapper(ref, preset="map-ont", hpc=True, distinct=0.9998)
    b = Mapper(ref, wfile, preset="map-ont", hpc=True)
    assert a.hpc and np.array_equal(_blob(a), _blob(b))
    a.close(); b.close()


def test_midsize_tandem_reference_matches_stand_in(tmp_path):
    """The 20 Mbp tandem-repeat reference of test_gpu_e2e.py: the device list is the stand-in's."""
    from winnowmap_b200.mapper import top_kmers
    contigs = gen_data.make_ref(np.random.default_rng(1005), 20_000_000, 2, True)
    fa = str(tmp_path / "mid.fa")
    gen_data.write_fasta(fa, contigs)
    kmers, counts, thr = top_kmers(fa, 15, 0.9998)
    sk, sc, sthr = gen_data.top_kmers(contigs, 15, 0.9998)
    assert thr == sthr and np.array_equal(kmers, sk) and np.array_equal(counts, sc) and len(kmers) > 1000
