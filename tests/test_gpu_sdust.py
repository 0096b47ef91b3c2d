"""SDUST (-T) on the H100: wm_sdust_batch against the oracle (the CPU test set, and one launch over several hundred 10-30 kb
tandem-rich reads), Mapper(..., sdust_thres=T) against every sdust_* golden, and sdust_thres=0 against the path without it."""
import ctypes as C
import gzip
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen_data  # noqa: E402
import make_golden  # noqa: E402
import sdust_lib as S  # noqa: E402
from test_sdust_cpu import MANIFEST, check_output, inputs  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("T", S.T_SET)
def test_sdust_batch_matches_oracle(T):
    from winnowmap_b200 import kernels
    seqs = S.case_set()
    got = kernels.sdust_batch(seqs, T)
    for s, g in zip(seqs, got):
        assert np.array_equal(g, S.as_pairs(S.oracle_sdust(s, T))), (T, s[:40])


def test_sdust_batch_other_windows():
    from winnowmap_b200 import kernels
    seqs = S.crafted_sequences()
    for W in (3, 10, 63):
        for s, g in zip(seqs, kernels.sdust_batch(seqs, 20, W)):
            assert np.array_equal(g, S.as_pairs(S.oracle_sdust(s, 20, W))), (W, s[:40])


def tandem_reads(n, seed=7):
    """n reads of 10-30 kb with microsatellites and tandem arrays, 5 % errors, a few N runs."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        L = int(rng.integers(10000, 30001))
        s = bytearray(gen_data.random_seq(rng, L).tobytes())
        for _ in range(int(rng.integers(5, 30))):
            u = int(rng.integers(1, 40))
            unit = S.acgt(rng, u)
            span = int(rng.integers(30, 1500))
            at = int(rng.integers(0, L - span))
            s[at:at + span] = (unit * (span // u + 1))[:span]
        for i in np.nonzero(rng.random(L) < 0.05)[0]:
            s[i] = b"ACGT"[int(rng.integers(0, 4))]
        if rng.random() < 0.2:
            at = int(rng.integers(0, L - 10))
            s[at:at + 5] = b"NNNNN"
        out.append(bytes(s))
    return out


def test_sdust_batch_long_tandem_reads_one_launch():
    from winnowmap_b200 import kernels
    seqs = tandem_reads(400)
    got = kernels.sdust_batch(seqs, 20)
    n_reg = 0
    for s, g in zip(seqs, got):
        assert np.array_equal(g, S.as_pairs(S.oracle_sdust(s, 20)))
        n_reg += len(g)
    assert n_reg > 400


def test_sdust_batch_refuses_bad_arguments():
    from winnowmap_b200 import kernels
    for T, W in ((0, 64), ((1 << 20) + 1, 64), (20, 65), (20, 2)):
        with pytest.raises(ValueError):
            kernels.sdust_batch([b"ACGT"], T, W)


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_mapper_sdust_matches_reference(name, tmp_path):
    from winnowmap_b200.mapper import Mapper
    lo = dict(MANIFEST[name]["lib"])
    ref, reads, wfile = inputs(name, str(tmp_path))
    mp = Mapper(ref, wfile, **lo)
    out = str(tmp_path / "o.out")
    mp.map_file(reads, out)
    mp.close()
    check_output(name, out)


def _launches(L):
    o = (C.c_double * 13)()
    L.wm_prof_get(o)
    return int(o[0])


def test_sdust_off_is_the_path_without_it(tmp_path):
    """sdust_thres=0 maps the ont_tandem golden as before, with the same number of kernel launches as a Mapper without the
    argument; -T 20 on the same input launches more."""
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import Mapper
    L = lib()
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    ref, reads, wfile = make_golden.make_inputs("ont_tandem", str(tmp_path))
    exp = gzip.open(os.path.join(ROOT, "tests", "golden", "ont_tandem.paf.gz")).read()
    counts = []
    for kw in ({}, dict(sdust_thres=0), dict(sdust_thres=20)):
        mp = Mapper(ref, wfile, preset="map-ont", **kw)
        out = str(tmp_path / "o.paf")
        L.wm_prof_reset()
        mp.map_file(reads, out)
        counts.append(_launches(L))
        mp.close()
        if kw.get("sdust_thres", 0) == 0:
            assert open(out, "rb").read() == exp
    assert counts[0] == counts[1] and counts[2] > counts[1], counts
