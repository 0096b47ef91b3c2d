"""The -W list without a GPU: the plain-C oracle (oracle/wm_oracle_topfreq.c) against the meryl stand-in of tools/gen_data.py,
the library's threshold rule against the oracle at the rule's edges, and the device's k-mer walk (csrc/topfreq.cuh) compiled
for the host against a byte-per-base restatement."""
import ctypes as C
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

LIST_CASES = sorted(n for n, c in make_golden.CASES.items() if c["use_W"])


def _np(contigs):
    return [(n, np.frombuffer(s, dtype=np.uint8)) for n, s in contigs]


@pytest.mark.parametrize("distinct", [0.9998, 0.99, 0.9])
@pytest.mark.parametrize("k", [15, 16, 19])
def test_oracle_matches_stand_in(k, distinct):
    contigs = T.genome(100 + k, k)
    kmers, counts, thr, nd = T.oracle_top_kmers(contigs, k, distinct)
    sk, sc, sthr = gen_data.top_kmers(_np(contigs), k, distinct)
    assert thr == sthr and np.array_equal(kmers, sk) and np.array_equal(counts, sc)
    assert nd > 10000 and (thr > 1 if distinct == 0.9998 else thr == 1)
    if distinct <= 0.99:
        assert len(kmers) > 0
    if k % 2 == 0 and distinct == 0.9:  # the planted palindromes are counted once per occurrence and some are listed
        pal = {min(T.spell(v, k), T.revcomp(T.spell(v, k))) for v in kmers.tolist() if T.spell(v, k) == T.revcomp(T.spell(v, k))}
        assert pal


def test_genome_reaches_the_corners():
    contigs = T.genome(115, 16)
    cat = b"".join(s for _, s in contigs)
    assert b"N" in cat and any(ch in cat for ch in b"RYKMSWBDHV") and any(ch in cat for ch in b"acgt")
    assert any(len(s) == 0 for _, s in contigs) and any(0 < len(s) < 16 for _, s in contigs)


@pytest.mark.parametrize("name", LIST_CASES)
def test_oracle_matches_golden_lists(name, tmp_path):
    """Every golden case built with a -W list: the oracle's list is the stand-in's file the reference binary was fed."""
    c = make_golden.CASES[name]
    ref, _, wfile = make_golden.make_inputs(name, str(tmp_path))
    contigs = [(n, s.encode()) for n, s in make_golden.read_fasta(ref)]
    kmers, counts, thr, _ = T.oracle_top_kmers(contigs, c["k"], c.get("w_distinct", 0.9998))
    wk, wc = T.read_list(wfile)
    assert np.array_equal(kmers, wk) and np.array_equal(counts, wc)
    assert len(kmers) > 0 and thr > 1


# (counts of the distinct k-mers, D, meryl's threshold)
EDGES = [
    ([1, 1, 2, 3, 3], 0.5, 1),             # target 2 (the stand-in compares with 2.5 and takes 2)
    ([5, 7], 0.4, 5),                      # target (uint64)0.8 = 0: the first value
    ([1, 2, 2, 9], 1.0, 9),                # D = 1: the largest value, an empty list
    ([4], 0.9998, 4),                      # one distinct k-mer
    ([1, 1, 1, (1 << 20) + 3, (1 << 20) + 9], 0.8, (1 << 20) + 3),  # counts above 2^20
]


@pytest.mark.parametrize("counts,distinct,want", EDGES)
def test_library_threshold_matches_oracle_at_the_edges(counts, distinct, want):
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import _setup
    L = _setup(lib())
    vals, occ = np.unique(np.array(counts, dtype=np.uint64), return_counts=True)
    vals, occ = np.ascontiguousarray(vals, dtype=np.uint64), np.ascontiguousarray(occ, dtype=np.uint64)
    got = L.wm_topfreq_threshold(vals.ctypes.data, occ.ctypes.data, len(vals), distinct)
    kmers, kc, thr, nd = T.oracle_top_kmers(T.hist_contigs(counts), 11, distinct)
    assert nd == len(counts) and sorted(kc.tolist()) == sorted(c for c in counts if c > want)
    assert got == thr == want


def test_stand_in_differs_from_meryl_on_the_example():
    """Documented difference (DESIGN.md section 5): the stand-in compares with the untruncated product."""
    contigs = T.hist_contigs([1, 1, 2, 3, 3])
    _, sc, sthr = gen_data.top_kmers(_np(contigs), 11, 0.5)
    _, kc, thr, _ = T.oracle_top_kmers(contigs, 11, 0.5)
    assert (sthr, len(sc)) == (2, 2) and (thr, len(kc)) == (1, 3)


def test_library_threshold_of_an_empty_histogram():
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import _setup
    assert _setup(lib()).wm_topfreq_threshold(None, None, 0, 0.9998) == 0


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("topfreq") / "topfreq_emul.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                           os.path.join(ROOT, "tests", "hostsim", "topfreq_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.wmt_tf_codes.restype = C.c_long
    L.wmt_tf_codes.argtypes = [C.c_char_p, C.c_long, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return L


def _byte_codes(seqs, k):
    """Byte-per-base restatement: (pool position, canonical code) of every k-mer of ACGTacgt inside one sequence."""
    pos, codes, o = [], [], 0
    for s in seqs:
        for i in range(len(s) - k + 1):
            w = s[i:i + k]
            if all(ch in b"ACGTacgt" for ch in w):
                f = w.upper().decode()
                codes.append(min(int(f.translate(str.maketrans("ACGT", "0123")), 4), int(T.revcomp(f).translate(str.maketrans("ACGT", "0123")), 4)))
                pos.append(o + i)
        o += len(s)
    return np.array(pos, dtype=np.int64), np.array(codes, dtype=np.uint64)


@pytest.mark.parametrize("k", [1, 2, 7, 15, 16, 19, 27, 28])
def test_kmer_walk_matches_byte_restatement(emul, k):
    """Sequences of every length around the 32-base groups, N and IUPAC codes at group edges, sequences shorter than k."""
    rng = np.random.default_rng(k)
    seqs = []
    for _ in range(120):
        n = int(rng.integers(1, 140))
        s = bytearray(rng.choice(list(b"ACGTacgt"), n).tolist())
        for _ in range(int(rng.integers(0, 3))):
            s[int(rng.integers(0, n))] = int(rng.choice(list(b"NRY")))
        seqs.append(bytes(s))
    pool = b"".join(seqs)
    off = np.cumsum([0] + [len(s) for s in seqs]).astype(np.int64)
    pos, codes = np.zeros(len(pool) + 1, dtype=np.int64), np.zeros(len(pool) + 1, dtype=np.uint64)
    n = emul.wmt_tf_codes(pool, len(pool), off.ctypes.data, len(seqs), k, pos.ctypes.data, codes.ctypes.data)
    ep, ec = _byte_codes(seqs, k)
    assert n == len(ep) and np.array_equal(pos[:n], ep) and np.array_equal(codes[:n], ec)
