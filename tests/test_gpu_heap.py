"""--heap-sort=yes on the H100: the seed stage alone (wm_seed_batch) against the oracle's collect_seed_hits_heap on the crafted
sets under every skip_seed flag, with tasks that take the small and the large shared-memory launch, the global-memory heap and
one task of more than 10^5 anchors; only tasks with ties are replayed; Mapper(..., heap_sort=True) against every heap_* golden;
and heap_sort=False is the path without it."""
import ctypes as C
import gzip
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import heap_lib as H  # noqa: E402
import make_golden  # noqa: E402
from test_heap_cpu import CASE_NAMES, MANIFEST, case_set, check_output, index, inputs  # noqa: E402

pytestmark = pytest.mark.gpu


def run_batch(tasks, max_occ, heap=True):
    """tasks: list of (mv, qlen, flag, qname) -> kernels.seed_batch results"""
    from winnowmap_b200 import kernels
    ix = index()
    skip = [H.skip_bits(ix, flag, qname) for _, _, flag, qname in tasks]
    return kernels.seed_batch(ix.keys, ix.pos_off, ix.pos, [(mv, qlen) for mv, qlen, _, _ in tasks], max_occ, heap=heap,
                              seq_len=ix.seq_len, name_rank=ix.name_rank, skip=skip if any(s != (0, 0) for s in skip) else None)


def check_task(res, mv, qlen, max_occ, flag, qname):
    a, rep, nmp, mpos = res
    exp, rep0, mp0 = H.oracle_heap(index(), mv, qlen, max_occ, flag, qname)
    assert np.array_equal(a, exp)
    assert rep == rep0 and nmp == len(mp0)
    kept = mpos[mpos >> np.uint32(31) == 1] & np.uint32(0x7fffffff)
    assert np.array_equal(kept.astype(np.uint64), mp0 & np.uint64(0xffffffff))


@pytest.mark.parametrize("case", CASE_NAMES)
def test_seed_batch_heap_matches_oracle(case):
    """One batch per set: one task per skip_seed flag set."""
    mv, qlen, max_occ = case_set()[case]
    tasks = [(mv, qlen, flag, qname) for _, flag, qname in H.FLAG_SETS]
    for res, (_, _, flag, qname) in zip(run_batch(tasks, max_occ), tasks):
        check_task(res, mv, qlen, max_occ, flag, qname)


@pytest.mark.parametrize("case", CASE_NAMES)
def test_seed_batch_without_heap_is_the_sorted_path(case):
    mv, qlen, max_occ = case_set()[case]
    a = run_batch([(mv, qlen, 0, None)], max_occ, heap=False)[0][0]
    assert np.array_equal(a, H.oracle_sorted(index(), mv, qlen, max_occ))


def _big_tasks():
    """(name, mv, qlen): a task in the large launch with its lists staged, one with its heap in shared memory and its lists in
    global memory (more than 10^5 anchors), and one whose heap lies in global memory"""
    ix = index()
    rng = np.random.default_rng(3)
    cnt = np.diff(ix.pos_off.astype(np.int64))
    big = ix.keys[np.argmax(cnt)]
    mid = ix.keys[(cnt >= 2) & (cnt < 8)]
    single = ix.keys[cnt == 1]

    def mk(hashes):
        qlen = 4 * len(hashes) + 100
        qp = np.sort(rng.choice(np.arange(H.K, qlen), size=len(hashes), replace=False))
        return H._mv([(int(h), int(p), int(rng.integers(0, 2))) for h, p in zip(hashes, qp)]), qlen

    out = []
    out.append(("staged_large", *mk(list(rng.choice(mid, 900)) + list(rng.choice(single, 100)))))
    hashes = [big] * 2600 + list(rng.choice(single, 300))
    out.append(("giant", *mk([hashes[i] for i in rng.permutation(len(hashes))])))
    out.append(("global_heap", *mk(list(rng.choice(mid, 5000)) + list(rng.choice(single, 1500)))))
    return out


def test_seed_batch_heap_every_memory_tier():
    from winnowmap_b200 import kernels
    ix = index()
    big = _big_tasks()
    small = [(case_set()[c][0], case_set()[c][1]) for c in ("duplicate_groups_interleaved", "read_1", "read_5")]
    tasks = [(mv, qlen, 0, None) for mv, qlen in small] + [(mv, qlen, 0, None) for _, mv, qlen in big]
    need = [len(mv) * 48 + sum(ix.count(int(x) >> 8) for x in mv[:, 0]) * 8 for mv, _, _, _ in tasks]
    assert need[0] <= 24 << 10 and need[-3] > 24 << 10 and need[-3] <= 200 << 10
    assert len(big[-1][1]) * 48 > 200 << 10
    kernels.seed_heap_stats(reset=True)
    res = run_batch(tasks, 5000)
    st = kernels.seed_heap_stats()
    for r, (mv, qlen, flag, qname) in zip(res, tasks):
        check_task(r, mv, qlen, 5000, flag, qname)
    assert len(res[-2][0]) >= 100000
    assert st["tasks"] == len(tasks) and st["global_heaps"] == 1 and st["mismatches"] == 0, st
    print(f"\n[heap-tiers] {st}")


def test_tasks_without_ties_are_not_replayed():
    from winnowmap_b200 import kernels
    cs = case_set()
    tasks = [(cs["unique_lists"][0], cs["unique_lists"][1], 0, None), (cs["one_hash_many_copies"][0], cs["one_hash_many_copies"][1], 0, None)]
    kernels.seed_heap_stats(reset=True)
    res = run_batch(tasks, 5000)
    st = kernels.seed_heap_stats()
    for r, t in zip(res, tasks):
        check_task(r, *t[:2], 5000, *t[2:])
    assert st["tasks"] == 1 and st["anchors"] == len(res[1][0]), st


def _mapper(ref, lo):
    from winnowmap_b200.mapper import Mapper
    lo = dict(lo)
    return Mapper(ref, None, heap_sort=True, **lo)


@pytest.mark.parametrize("name", sorted(MANIFEST))
def test_mapper_heap_sort_matches_reference(name, tmp_path):
    from winnowmap_b200 import kernels
    ref, reads = inputs(name, str(tmp_path))
    mp = _mapper(ref, MANIFEST[name]["lib"])
    out = str(tmp_path / "o.out")
    kernels.seed_heap_stats(reset=True)
    mp.map_file(reads, out)
    mp.close()
    st = kernels.seed_heap_stats()
    check_output(name, out)
    assert st["mismatches"] == 0, st
    if MANIFEST[name]["n_lines_differing"]:  # the ties that changed the reference's output were replayed here
        assert st["tasks"] > 0, st


def _launches(L):
    o = (C.c_double * 13)()
    L.wm_prof_get(o)
    return int(o[0])


def test_heap_sort_off_is_the_path_without_it(tmp_path):
    """heap_sort=False maps the ont_tandem golden as before, with the same number of kernel launches as a Mapper without the
    argument; heap_sort=True on the same input launches more (tie scan and replay per seed pass)."""
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import Mapper
    L = lib()
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    ref, reads, wfile = make_golden.make_inputs("ont_tandem", str(tmp_path))
    exp = gzip.open(os.path.join(ROOT, "tests", "golden", "ont_tandem.paf.gz")).read()
    counts = []
    for kw in ({}, dict(heap_sort=False), dict(heap_sort=True)):
        mp = Mapper(ref, wfile, preset="map-ont", **kw)
        out = str(tmp_path / "o.paf")
        L.wm_prof_reset()
        mp.map_file(reads, out)
        counts.append(_launches(L))
        mp.close()
        assert open(out, "rb").read() == exp  # (this input has no tie that changes its output)
    assert counts[0] == counts[1] and counts[2] > counts[1], counts
