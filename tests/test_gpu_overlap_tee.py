"""The seed filter of -D / --dual=no / -X / --for-only / --rev-only, call by call: crafted seed_chain calls go to the CUDA
backend and to the filtering oracle backend (tests/hostsim/overlap_tee.cpp, overlap_oracle.h), and every field of every
task must agree, the chained anchors with their MM_SEED_SELF bits included.  The end-to-end goldens cannot see that bit
(every self-hit they hold is a full-length diagonal hit), so this is where it is checked.

The crafted batch:
  * a reference sequence named like a 20 kb read and equal to its first 2000 bases (a stage-1 window length of map-ont),
    with a repeat inside: the windows of length 2000 trip the NO_DIAG length test, drop the diagonal (window-relative
    positions, as the reference compares them) and flag the off-diagonal forward anchors MM_SEED_SELF;
  * two reference sequences with the same name, and reads named like them, before and after them in strcmp order;
  * a read whose every occurrence is skipped (its name sorts after every reference name under --dual=no);
  * a read without a name (the name tests are off);
  * --for-only on a reverse-strand read (every occurrence skipped) and --rev-only on the same reads."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tee_lib as T  # noqa: E402

F_NO_DIAG, F_NO_DUAL, F_FOR_ONLY, F_REV_ONLY = 0x001, 0x002, 0x100000, 0x200000
K, W = 15, 10


@pytest.fixture(scope="module")
def tee(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("overlap_tee") / "libwm_overlap_tee.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", f"-I{cuda}/include",
                           os.path.join(T.HOSTSIM, "overlap_tee.cpp"), "-x", "c", os.path.join(ROOT, "oracle", "wm_oracle.c"),
                           os.path.join(ROOT, "oracle", "wm_oracle_hpc.c"), "-x", "none", f"-L{T.PKG}", "-lwinnowmap_b200",
                           f"-Wl,-rpath,{T.PKG}", "-o", so, "-lz", "-lm", "-lpthread"])
    L = C.CDLL(so)
    s, i, i64, p = C.c_char_p, C.c_int, C.c_int64, C.c_void_p
    L.wmt_tee_overlap_seed_chain.argtypes = [s, i, i, i, i64, i, p, s, p, i, p, p, p, i, s]
    return L


def _batch(tmp):
    """(reference FASTA, read names, read sequences, windows)."""
    rng = np.random.default_rng(11)
    rand = lambda n: T._rand(rng, n)  # noqa: E731
    unit = rand(400)
    prefix = rand(200) + unit + rand(600) + unit + rand(400)   # 2000 bases, the unit at 200 and 1200
    read_l = prefix + rand(18000)
    s1, s2, chr1 = rand(6000), rand(6000), rand(60000)
    refs = [("chr1", chr1), ("dup", s1), ("rL", prefix), ("dup", s2), ("a", rand(3000))]
    ref = os.path.join(str(tmp), "ref.fa")
    with open(ref, "w") as f:
        for nm, sq in refs:
            f.write(f">{nm}\n{sq.decode()}\n")
    noisy = lambda sq: T._noisy(rng, sq, 0.03)[0]  # noqa: E731
    reads = [("rL", read_l), ("dup", s1), ("dupA", noisy(s2)), ("du", noisy(s2)), ("zz", noisy(chr1[20000:32000])),
             (None, read_l), ("fw", noisy(chr1[5000:15000])), ("rv", T.revcomp(noisy(chr1[30000:40000]))), ("rL", prefix + unit + prefix)]
    wins = []
    for i, (_, sq) in enumerate(reads):
        wins.append((i, 0, len(sq)))
    for wb, wl in ((0, 2000), (500, 2000), (1, 2000), (0, 5656), (1200, 2000)):
        wins.append((0, wb, wl))   # the rL read: windows as long as the rL sequence trip the length test
        wins.append((5, wb, wl))   # the same bases without a name
    wins += [(8, 0, 2000), (8, 2400, 2000), (1, 0, 2000), (1, 1000, 5000)]
    return ref, [nm for nm, _ in reads], [sq for _, sq in reads], wins


def _run(L, tmp, flag, dev):
    ref, names, seqs, wins = _batch(tmp)
    seq, off = T._pool(seqs)
    nm = (C.c_char_p * len(names))(*[n.encode() if n is not None else None for n in names])
    r1 = np.ascontiguousarray(np.asarray(wins, dtype=np.int32).reshape(-1, 3))
    keys = ("max_dist_x", "min_dist_x", "max_dist_y", "bw", "max_skip", "max_iter", "min_cnt", "min_sc")
    ci = np.array([[c[k] for k in keys] for c in T.CHAIN_SETS], dtype=np.int32)
    cf = np.array([c["gap_scale"] for c in T.CHAIN_SETS], dtype=np.float32)
    rep = str(tmp / f"report_{flag:x}_{dev}.txt")
    rc = L.wmt_tee_overlap_seed_chain(ref.encode(), K, W, dev, flag, len(seqs), nm, seq, off.ctypes.data, len(r1), r1.ctypes.data,
                                      ci.ctypes.data, cf.ctypes.data, 1 << 20, rep.encode())
    assert rc == 0, rc
    return T.Report(rep)


# what each flag set must reach in the crafted batch: chained MM_SEED_SELF anchors, windows left empty
REACH = {
    F_NO_DIAG: dict(self=True, empty=True),    # the exact copy of a "dup" sequence: all diagonal
    F_NO_DIAG | F_NO_DUAL: dict(self=True, empty=True),   # -X
    F_NO_DUAL: dict(self=False, empty=True),
    F_FOR_ONLY: dict(self=False, empty=True),
    F_REV_ONLY: dict(self=False, empty=True),
}


@pytest.mark.parametrize("flag", sorted(REACH))
def test_crafted_batch_reaches_its_cases(tee, flag, tmp_path):
    """Without a device: two filtering oracle backends agree, and the batch holds what the GPU test relies on."""
    r = _run(tee, tmp_path, flag, T.DEV_ORACLE)
    assert r.n_mismatch == 0, r.text()
    assert (r["overlap.self_anchors"] > 0) == REACH[flag]["self"], r.text()
    assert (r["overlap.empty_tasks"] > 0) == REACH[flag]["empty"], r.text()
    assert r["overlap.tasks_filtered"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("flag", sorted(REACH))
def test_seed_filter_matches_oracle_call_by_call(tee, flag, tmp_path):
    r = _run(tee, tmp_path, flag, T.DEV_GPU)
    assert r.n_mismatch == 0, r.text()
    assert (r["overlap.self_anchors"] > 0) == REACH[flag]["self"], r.text()
