"""CPU check of the giant-task chaining kernel as a whole CTA (csrc/chain.cu: wm_chain_fill_tile_kernel, whose body is
wm_chain_fill_tile_cta of csrc/chain_tile.cuh): its 32 warps run on an emulated CTA (tests/hostsim, cuda_emul.h: run_cta) at the
kernel's own ring (4096 slots) and list (48 entries), under schedules chosen here, against the scalar restatement of src/chain.c:45-90.

The warps share no barrier inside a task: a warp enters tile T only once tile T - 2 is complete (done-masks), reads coordinates of
tiles three back and older from the ring before it waits, waits for the anchors of tiles T - 1 and T it depends on, and redoes a scan
that needs anchors below the ring under a CTA lock with the global t[] marks.  A GPU run cannot choose its schedule; here the
schedules drive the protocol to its limits: a laggard warp that runs only when every other warp is blocked, a leader that runs
whenever it can, round robin at every warp-wide sync and a seeded random choice.  Each run reports, from the emulated atomics, the
deep scans (lock acquisitions), the failed lock attempts and the most tiles that were partly published at once.

The emulation is sequentially consistent: a missing __threadfence_block, volatile or __ldcg is invisible to it (those stay checked on
the device only)."""
import ctypes as C
import os
import shutil
import subprocess
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_chain_tile_list import PARAMS, _tandem
from test_oracle_vs_ref import make_anchors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.path.join(ROOT, "tests", "hostsim")
CSRC = os.path.join(ROOT, "winnowmap_b200", "csrc")
SIG = [C.c_void_p, C.c_int] + [C.c_int] * 6 + [C.c_float]
RING, LIST, WARPS = 4096, 48, 32
# the parameter sets of test_chain_tile_list.py, and one whose max_skip lets scans run through their windows
PARAMS_ALL = PARAMS + [(5000, 1000, 5000, 500, 1000, 5000)]
PAIRS = [(0, 5), (1, 2), (3, 4)]  # two parameter sets per CTA (per-task set ids)
# (kind, warp, seed) of cuda_emul.h: round robin, random, laggard (runs only when every other warp is blocked), leader
SCHEDULES = {"round_robin": (0, 0, 0), "random": (1, 0, 7), "laggard31": (2, 31, 0), "laggard0": (2, 0, 0), "leader0": (3, 0, 0)}
# Tiles partly published at once, at most: anchors publish after the wait, which lets warps into tile T only once tile T - 2 is
# complete; so when tile T holds a published anchor, every tile below T - 1 is complete, and only T - 1 and T can be partial.
IN_FLIGHT_BOUND = 2
NPROC = os.cpu_count() or 1


def _build(csrc=CSRC, out=None):
    cmd = [os.path.join(HOSTSIM, "build_tile_cta.sh"), csrc] + ([out] if out else [])
    subprocess.check_call(cmd, stderr=subprocess.DEVNULL)
    return _load(out or os.path.join(HOSTSIM, "libwm_tilecta.so"))


def _load(path):
    L = C.CDLL(path)
    L.wmt_tile_cta.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_uint64] + \
        [C.c_void_p] * 4 + [C.c_char_p, C.c_int]
    L.wmt_tile_scan_paths.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_void_p]
    L.wmt_tile_constants.argtypes = [C.c_void_p]
    return L


@pytest.fixture(scope="module")
def libs():
    subprocess.check_call([os.path.join(HOSTSIM, "build.sh")], stderr=subprocess.DEVNULL)
    H = C.CDLL(os.path.join(HOSTSIM, "libwm_hostsim.so"))
    H.wmt_chain_fill_scalar.argtypes = SIG + [C.c_void_p] * 3
    L = _build()
    k = np.zeros(3, np.int32)
    L.wmt_tile_constants(k.ctypes.data)
    assert tuple(k) == (RING, LIST, WARPS)  # the emulated kernel runs at the product's constants
    return H, L


# ---------------------------------------------------------------------------------------------------------------- inputs

def _xy(x, y, span=15):
    x, y = np.asarray(x, np.int64), np.asarray(y, np.int64)
    o = np.lexsort((y, x))
    return np.ascontiguousarray(np.stack([x[o].astype(np.uint64), np.uint64(span) << np.uint64(32) | y[o].astype(np.uint64)], axis=1))


def deep_array(n_fill=4200):
    """Candidates below the ring, by construction.  Two chains on diagonals 600 apart (never candidates of each other): C2, 100 anchors
    (high f), then C1, 30 anchors (low f); then n_fill anchors at one x with y far above everything (no candidate has them, they have
    none); then G, 64 anchors at one x (not candidates of each other) between the two diagonals, whose candidates are C1 and C2, more
    than WM_CT_RING - 64 anchors back: two whole tiles of scans that need the locked deep path.  With max_skip 25 the reference breaks
    inside C1 (each C1 anchor carries the mark of the one after it), before C2, which would score higher: a lost global mark changes
    f.  Last, T, 30 anchors on G's diagonal out of reach of C1 / C2, whose candidates are G: in the ring, with p[j] below it."""
    d2, d1, s, e = np.arange(100), np.arange(30), np.arange(64), np.arange(30)
    x = [100000 + 10 * d2, 101000 + 10 * d1, np.full(n_fill, 101500), np.full(64, 101600), 106300 + 10 * e]
    y = [x[0] - 99000, x[1] - 99600, 10 ** 7 + np.arange(n_fill), 2300 + s, x[4] - 99300]
    return _xy(np.concatenate(x), np.concatenate(y))


def zone_array():
    """A chain D of 32 anchors, 4032 anchors that are nobody's candidates, then a tile G of 32 anchors at one x whose candidates are D:
    D lies in [i0 + 32 - WM_CT_RING, i0 + 64 - WM_CT_RING) for G's tile i0 = 4064, the ring slots that the next tile (anchors 4096 ..,
    64 more that are nobody's candidates) overwrites.  The kernel takes D from global memory (deep path)."""
    d, s, g = np.arange(32), np.arange(32), np.arange(64)
    x = [100000 + 10 * d, np.full(4032, 100400), np.full(32, 100500), 200000 + g]
    y = [x[0] - 99000, 10 ** 7 + np.arange(4032), 1300 + s, 5 * 10 ** 6 - g]
    return _xy(np.concatenate(x), np.concatenate(y))


def diagonal(n, step=10):
    """One chain: anchor i's window holds i candidates (as long as they are within max_dist): with a max_skip above n, anchor 48 ends
    its window at exactly 48 candidates, and later ones overflow the list."""
    x = 100000 + step * np.arange(n)
    return _xy(x, x - 99000)


def _corpora():
    rng = np.random.default_rng(4711)
    deep = [deep_array(), diagonal(120), make_anchors(rng, 2049, repeats=False), make_anchors(rng, 50, repeats=True),
            make_anchors(rng, 0), make_anchors(rng, 33, repeats=True), zone_array()]
    tandem = [_tandem(rng, 150, 70, 171), _tandem(rng, 60, 40, 64), make_anchors(rng, 3000, repeats=True)]
    return {"deep": [np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 2) for a in deep],
            "tandem": [np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 2) for a in tandem]}


# ---------------------------------------------------------------------------------------------------------------- runs

def run_cta(L, arrays, set_id, prm_pair, sched):
    """The tasks in the given order on one emulated CTA; (rc, f, p, v, stats, err)."""
    off = np.cumsum([0] + [len(a) for a in arrays]).astype(np.int64)
    a = np.ascontiguousarray(np.concatenate(arrays)).astype(np.uint64)
    prm = np.ascontiguousarray(np.array(prm_pair, np.int32).reshape(-1))
    sid = np.asarray(set_id, np.uint8)
    order = np.arange(len(arrays), dtype=np.int32)
    f, p, v = (np.full(max(int(off[-1]), 1), -7, np.int32) for _ in range(3))
    st = np.zeros(10, np.int64)
    err = C.create_string_buffer(8192)
    kind, warp, seed = SCHEDULES[sched]
    rc = L.wmt_tile_cta(a.ctypes.data, off.ctypes.data, len(arrays), order.ctypes.data, prm.ctypes.data, 1.0, sid.ctypes.data, kind, warp, seed,
                        f.ctypes.data, p.ctypes.data, v.ctypes.data, st.ctypes.data, err, len(err))
    stats = dict(zip(["deep", "lock_fail", "polls", "in_flight", "published", "syncs", "switches", "retries", "events", "deadlock"], st.tolist()))
    return rc, [x[off[k]:off[k + 1]] for x in (f, p, v) for k in range(len(arrays))], stats, err.value.decode()


def scalar(H, a, prm):
    out = [np.full(len(a), -7, np.int32) for _ in range(3)]
    H.wmt_chain_fill_scalar(a.ctypes.data, len(a), *prm, 1.0, *(x.ctypes.data for x in out))
    return out


def scan_paths(L, a, prm):
    """Per anchor at the kernel's constants: deep (bit 0: a candidate the resolve examines lies below the ring, bit 1: one in the ring
    has its p[j] below it), candidates in the window, candidates consumed, whether the window ran out (1) or the loop broke (0)."""
    out = np.zeros((max(len(a), 1), 5), np.int32)
    pr = np.array(prm, np.int32)
    L.wmt_tile_scan_paths(a.ctypes.data, len(a), pr.ctypes.data, 1.0, out.ctypes.data)
    return out[:len(a)]


def tile_kernel_reach(arrays, prms):
    """On the CPU, at the tile kernel's constants, over the arrays and parameter sets: scans that need the locked deep path, the most
    such scans in one tile, and scans that consume more than WM_CT_LIST candidates (the list is refilled)."""
    if "reach" not in _LIBS:  # built once per process
        subprocess.check_call([os.path.join(HOSTSIM, "build.sh")], stderr=subprocess.DEVNULL)
        _LIBS["reach"] = _build()
    L = _LIBS["reach"]
    n_deep = per_tile = n_refill = 0
    for a in arrays:
        a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 2)
        for prm in prms:
            p = scan_paths(L, a, prm)
            d = np.flatnonzero(p[:, 0] > 0)
            n_deep += len(d)
            per_tile = max(per_tile, int(np.bincount(d // 32).max()) if len(d) else 0)
            n_refill += int((p[:, 2] > LIST).sum())
    return n_deep, per_tile, n_refill


_LIBS = {}


def _set_ids(n):
    return [k & 1 for k in range(n)]


def _mismatch(H, arrays, set_id, pair, got):
    n = len(arrays)
    for k, a in enumerate(arrays):
        want = scalar(H, a, PARAMS_ALL[pair[set_id[k]]])
        for m, nm in enumerate("fpv"):
            g = got[m * n + k]
            if not np.array_equal(want[m], g):
                i = int(np.argmax(want[m] != g))
                return f"task {k} (n {len(a)}) {nm}[{i}]: want {want[m][i]} got {g[i]}"
    return None


@pytest.fixture(scope="module")
def parity_runs(libs):
    """Every (corpus, parameter pair, schedule), in parallel threads (the emulation releases the GIL)."""
    H, L = libs
    corpora = _corpora()
    jobs = [(c, pair, s) for c in corpora for pair in PAIRS for s in SCHEDULES]
    t0 = time.time()

    def one(job):
        c, pair, s = job
        arrays = corpora[c]
        sid = _set_ids(len(arrays))
        rc, got, stats, err = run_cta(L, arrays, sid, [PARAMS_ALL[pair[0]], PARAMS_ALL[pair[1]]], s)
        return job, (rc, err, stats, _mismatch(H, arrays, sid, pair, got) if rc == 0 else None)

    with ThreadPoolExecutor(NPROC) as ex:
        res = dict(ex.map(one, jobs))
    print(f"\nparity: {len(jobs)} CTA runs of {sum(len(a) for c in corpora.values() for a in c)} anchors per corpus set, {time.time() - t0:.0f} s")
    return corpora, res


def test_tile_cta_matches_scalar(parity_runs):
    """f / p / v of every task equal the scalar restatement, for every input, parameter set and schedule, and no schedule deadlocks
    or takes more tiles in flight than the wait rule allows."""
    _, res = parity_runs
    bad = [(job, r[1] or r[3]) for job, r in res.items() if r[0] != 0 or r[3]]
    assert not bad, bad[:5]
    for job, (rc, err, stats, mm) in res.items():
        assert 1 <= stats["in_flight"] <= IN_FLIGHT_BOUND, (job, stats)


def test_tile_cta_inputs_reach_the_paths(libs, parity_runs):
    """The inputs and schedules reach what they are there for: deep scans and contention for the lock, scans that need a mark below the
    ring only, whole tiles of deep scans, list refills, a window of exactly WM_CT_LIST candidates, windows across the ring boundary,
    and, under the laggard schedule, as many tiles in flight as the protocol allows."""
    H, L = libs
    corpora, res = parity_runs
    paths = {}
    for c, arrays in corpora.items():
        for k, a in enumerate(arrays):
            for pair in PAIRS:
                prm = PARAMS_ALL[pair[_set_ids(len(arrays))[k]]]
                paths[c, k, prm] = scan_paths(L, a, prm)
    allp = np.concatenate([p for p in paths.values() if len(p)])
    deep, n_cand, used, ended = allp[:, 0], allp[:, 1], allp[:, 2], allp[:, 3] == 1
    assert (deep & 1).sum() > 0 and (deep == 2).sum() > 0, "deep scans for a candidate below the ring, and for a mark only"
    assert (used > LIST).sum() > 0, "list refills"
    assert ((n_cand == LIST) & ended).sum() > 0, "a window of exactly WM_CT_LIST candidates"
    whole = [max(np.bincount(np.flatnonzero(p[:, 0] > 0) // 32, minlength=1)) for p in paths.values() if len(p)]
    assert max(whole) == 32, "a whole tile of deep scans"
    # the scans that take the deep path are those the lock serves (per task: the first attempt fails exactly then)
    for c in corpora:
        arrays = corpora[c]
        for pair in PAIRS:
            sid = _set_ids(len(arrays))
            want = sum(int((paths[c, k, PARAMS_ALL[pair[sid[k]]]][:, 0] > 0).sum()) for k in range(len(arrays)))
            for s in SCHEDULES:
                assert res[c, pair, s][2]["deep"] == want, (c, pair, s, res[c, pair, s][2], want)
    stats = [r[2] for r in res.values()]
    assert max(s["lock_fail"] for s in stats) > 0, "contention for the lock"
    assert max(s["switches"] for s in stats) > 0
    # the laggard drives the others to the wait rule's limit; the leader and round robin interleave too
    for c in corpora:
        for pair in PAIRS:
            assert res[c, pair, "laggard31"][2]["in_flight"] == IN_FLIGHT_BOUND, (c, pair)
    # windows that cross the ring boundary and slots that wrap: a tandem task over twice the ring, windows longer than RING - 64
    assert len(corpora["tandem"][0]) > 2 * RING and window_span(corpora["tandem"][0], PARAMS_ALL[0]) > RING - 64


def window_span(a, prm):
    """max over i of i - st[i], st[i] of src/chain.c:49-55 in closed form: max(lb(max_dist_x), min(i - max_iter, lb(min_dist_x)))."""
    x = a[:, 0]
    lb = lambda d: np.searchsorted(x, np.where(x > np.uint64(d), x - np.uint64(d), np.uint64(0)), side="left")
    i = np.arange(len(x))
    st = lb(prm[0])
    st = np.where(i - st > prm[5], np.maximum(st, np.minimum(i - prm[5], lb(prm[1]))), st)
    return int((i - st).max())


# ---------------------------------------------------------------------------------------------------------------- mutations

WAIT = "\t\t\t\t\tif (Cp) { while ((done[(T - 1) & 7] & Cp) != Cp) __nanosleep(32); }\n"
MUTATIONS = {
    "no_Cp_wait": (WAIT, ""),
    "wait_T_minus_3": ("if (T >= 2) { while (done[(T - 2) & 7] != FULL)", "if (T >= 2) { while (done[(T - 3) & 7] != FULL)"),
    "phase_A_ring_to_i0_minus_32": ("if (j >= ring_lo && j < i0 - 64) {", "if (j >= ring_lo && j < i0 - 32) {"),
    "ring_lo_plus_32": ("const int ring_lo = i0 + 64 - WM_CT_RING;", "const int ring_lo = i0 + 32 - WM_CT_RING;"),
    "reset_done_T_plus_1": ("if (lane == 0) done[(T + 4) & 7] = 0;", "if (lane == 0) done[(T + 1) & 7] = 0;"),
    "deep_without_lock": ("if (lane == 0) { while (atomicCAS(&S->lock, 0, 1) != 0) __nanosleep(64); }", ""),
}
MUTATED_HEADERS = ["chain_tile.cuh", "chain_dev.cuh"]
MUTATION_TRIES = [("deep", (0, 5), "laggard31"), ("deep", (0, 5), "round_robin"), ("deep", (0, 5), "random"), ("deep", (0, 5), "laggard0"),
                  ("tandem", (0, 5), "laggard31"), ("tandem", (0, 5), "random"), ("deep", (0, 5), "leader0")]


@pytest.fixture(scope="module")
def mutants(libs, tmp_path_factory):
    """One library per mutation, built from a copy of the product headers with that one change (in the CTA body, chain_tile.cuh, or
    the scan it calls, chain_dev.cuh)."""
    src = {h: open(os.path.join(CSRC, h)).read() for h in MUTATED_HEADERS}
    d = tmp_path_factory.mktemp("mutants")
    jobs = {}
    for name, (old, new) in MUTATIONS.items():
        where = [h for h in MUTATED_HEADERS if old in src[h]]
        assert sum(src[h].count(old) for h in MUTATED_HEADERS) == 1, (name, "the text to replace must occur exactly once in", MUTATED_HEADERS)
        m = d / name
        shutil.copytree(CSRC, m, ignore=shutil.ignore_patterns("*.cu", "*.cpp"))
        (m / where[0]).write_text(src[where[0]].replace(old, new))
        jobs[name] = (str(m), str(d / f"lib_{name}.so"))
    with ThreadPoolExecutor(NPROC) as ex:
        list(ex.map(lambda j: subprocess.check_call([os.path.join(HOSTSIM, "build_tile_cta.sh"), *j], stderr=subprocess.DEVNULL), jobs.values()))
    return {name: _load(out) for name, (_, out) in jobs.items()}


def test_tile_cta_catches_protocol_mutations(libs, mutants):
    """Each change to the protocol, made to a copy of the product headers, makes some schedule give a wrong f / p / v or a deadlock."""
    H, _ = libs
    corpora = _corpora()
    t0 = time.time()

    def hunt(name):
        L = mutants[name]
        for c, pair, s in MUTATION_TRIES:
            arrays = corpora[c]
            sid = _set_ids(len(arrays))
            rc, got, stats, err = run_cta(L, arrays, sid, [PARAMS_ALL[pair[0]], PARAMS_ALL[pair[1]]], s)
            if rc != 0:
                assert stats["deadlock"] == 1 and "tile" in err, (name, err)
                return name, (c, s, "deadlock")
            mm = _mismatch(H, arrays, sid, pair, got)
            if mm:
                return name, (c, s, mm)
        return name, None

    with ThreadPoolExecutor(NPROC) as ex:
        caught = dict(ex.map(hunt, MUTATIONS))
    print(f"\nmutations ({time.time() - t0:.0f} s):", caught)
    assert all(caught.values()), {k: v for k, v in caught.items() if not v}
