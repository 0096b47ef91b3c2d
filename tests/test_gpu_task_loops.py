"""The task loops of the CTA-level kernels and the switch-selected variants, against the oracle, bit for bit.

Most device time goes to kernels whose fixed grid keeps taking the next array or chaining task until none are left: the
giant anchor sort (csrc/seed.cu, wm_anchor_sort_giant_kernel, grid-stride), the chaining tile kernel and the ring and
backtrack kernels (csrc/chain.cu, counter-dispatched).  State that a worker carries from one task to the next (mbarrier
phases, work lists, walk state, done masks, rings, warp workspaces) is only used from a worker's second task on.  The
batches here are sized from the SM count so that workers take several tasks, and the CTA counts are capped by the
switches so that a single CTA takes all of them.

Every configuration runs in a child process with a timeout: the switches are read once per process, and some kernels spin
on shared-memory flags.  The child only runs the device; the oracle results are computed once, here."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as ol
from test_chain_tile_cta import deep_array, tile_kernel_reach, zone_array
from test_gpu_stages import _span_tandem, _tandem_anchors
from test_oracle_vs_ref import FLAGS, make_anchors, make_span_anchors, rand_pair

pytestmark = pytest.mark.gpu
TESTS_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT_DIR = os.path.dirname(TESTS_DIR)

_CHILD = r'''
import sys
sys.path.insert(0, %r)
import numpy as np
from winnowmap_b200 import kernels
kind, src, dst = sys.argv[1:4]
z = np.load(src)

def unpack(p):
    cat, off = z[p], z[p + "_off"]
    return [cat[off[i]:off[i + 1]] for i in range(len(off) - 1)]

def pack(out, p, lst):
    out[p] = np.concatenate([np.asarray(x).reshape(-1) for x in lst])
    out[p + "_off"] = np.cumsum([0] + [np.asarray(x).size for x in lst])

out = {}
if kind == "sort":
    pack(out, "a", kernels.radix_sort_128x_batch([x.reshape(-1, 2) for x in unpack("a")]))
elif kind == "chain":
    arrays = [x.reshape(-1, 2) for x in unpack("a")]
    for k, (mx, mn, my, bw, skip, it) in enumerate(z["prm"].tolist()):
        got = kernels.chain_dp_batch(arrays, mx, mn, my, bw, max_skip=skip, max_iter=it)
        pack(out, "u%%d" %% k, [u for u, _ in got]); pack(out, "b%%d" %% k, [b for _, b in got])
else:
    for k in range(int(z["n_batches"])):
        p = "%%d_" %% k
        ez, cig = kernels.ksw_extd2_batch(unpack(p + "q"), unpack(p + "t"), z[p + "mat"], *z[p + "gaps"].tolist(), z[p + "w"], z[p + "zdrop"],
                                          z[p + "eb"], z[p + "flag"])
        out[p + "ez"] = ez; pack(out, p + "cig", cig)
np.savez(dst, **out)
print("child ok")
''' % ROOT_DIR


def _pack(out, p, lst):
    out[p] = np.concatenate([np.asarray(x).reshape(-1) for x in lst])
    out[p + "_off"] = np.cumsum([0] + [np.asarray(x).size for x in lst])


def _unpack(z, p):
    cat, off = z[p], z[p + "_off"]
    return [cat[off[i]:off[i + 1]] for i in range(len(off) - 1)]


def _cfg_id(env):
    return " ".join(f"{k}={v}" for k, v in env.items()) or "defaults"


def _device(kind, src, env, tmp_path, timeout=600):
    dst = str(tmp_path / f"{kind}_out.npz")
    out = subprocess.run([sys.executable, "-c", _CHILD, kind, src, dst], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, timeout=timeout)
    assert out.returncode == 0 and b"child ok" in out.stdout, out.stdout[-3000:].decode(errors="replace")
    return np.load(dst)


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------- sort

def _sort_corpus(rng):
    """Arrays for the CTA sorts, largest first as wm_anchor_sort_run orders them (equal sizes keep their order).  Each
    state-carrying case follows a larger array: on one CTA directly, on three CTAs three places later."""
    def arr(x):
        return np.stack([np.asarray(x, dtype=np.uint64), np.arange(len(x), dtype=np.uint64)], axis=1)

    def rand64(n):
        return rng.integers(0, (1 << 64) - 1, size=n, dtype=np.uint64, endpoint=True)

    def by_top_byte(counts, digits, low_range):
        """Elements whose top byte is digits[j] for counts[j] of them: the first pass's sub-buckets have exactly these sizes."""
        d = np.repeat(np.asarray(digits, dtype=np.uint64), counts)
        x = d << np.uint64(56) | rng.integers(0, low_range, size=len(d), dtype=np.uint64)
        return x[rng.permutation(len(x))]

    def strand(n, frac):  # anchor-like: positions with ties, the strand bit on a fraction (one two-bucket pass)
        pos = (123456789 + rng.integers(0, max(2, n // 3), size=n) * 7).astype(np.uint64)
        return pos | ((rng.random(n) < frac).astype(np.uint64) << np.uint64(63))

    arrays = []
    # FIFO-fed walks: more misplaced slots than the resident list holds (32768 for <512>, 131072 for <2048>)
    arrays += [arr(rand64(150000)), arr(rand64(140000))]
    arrays += [arr(strand(60000, 0.5)), arr(strand(40000, 0.03))]  # two-bucket strand splits (the closed form)
    arrays += [arr(x) for x in (rand64(n) for n in rng.integers(25000, 100000, size=4))]
    arrays += [arr(rand64(20001)), arr(rand64(13313)), arr(rand64(13312))]  # resident walk; both sides of 13312
    # tandem-like fillers with heavy ties, between 13312 and the cases below
    for n in rng.integers(6000, 12000, size=14):
        arrays.append(arr((1000 + (rng.integers(0, n // 30, size=n) * 171) % 40000).astype(np.uint64)))
    # sub-buckets of exactly 64 / 65 and the stage sizes 512 / 513 and 2048 / 2049, with and without ties below the top byte
    arrays.append(arr(by_top_byte([64, 65, 512, 513, 2048, 2049, 3, 1], [1, 2, 3, 5, 8, 13, 21, 34], 1 << 56)))
    arrays.append(arr(by_top_byte([2049, 2048, 513, 512, 65, 64, 300, 2], [200, 201, 202, 250, 251, 252, 254, 255], 40)))
    arrays += [arr(np.zeros(5000, np.uint64)), arr(np.full(5000, 0x8000000012345678, np.uint64))]  # all equal: no phase-2 range
    # every sub-bucket <= 64 (the warps' mbarrier phases do not flip), then an odd and an even number of phase-2 ranges
    for _ in range(3):
        arrays.append(arr(by_top_byte([16] * 256, list(range(256)), 1 << 56)))
    for n_mid, n_rest in [(3, 40), (4, 30)]:
        for _ in range(3):
            rest = 2100 - 10 * (n_mid - 3) - 300 * n_mid
            counts = [300] * n_mid + [rest // n_rest + (j < rest % n_rest) for j in range(n_rest)]
            arrays.append(arr(by_top_byte(counts, list(range(100, 100 + n_mid + n_rest)), 1 << 56)))
    arrays += [arr(rand64(2049)), arr(rand64(2049)), arr(rand64(2048)), arr(rand64(65)), arr(rand64(1)), arr(rand64(0))]
    return sorted(arrays, key=len, reverse=True)  # (stable)


@pytest.fixture(scope="module")
def sort_case(tmp_path_factory):
    arrays = _sort_corpus(np.random.default_rng(41))
    sizes = [len(a) for a in arrays]
    assert sum(n > 2048 for n in sizes) >= 40
    # the state-carrying cases: 4096 (no phase-2 range), then 3 and 4 phase-2 ranges of 300
    assert sizes[sizes.index(4096):sizes.index(2049)] == [4096] * 3 + [2100] * 3 + [2090] * 3
    src = str(tmp_path_factory.mktemp("sort") / "in.npz")
    inp = {}
    _pack(inp, "a", arrays)
    np.savez(src, **inp)
    return src, arrays, [ol.oracle_sort128(a) for a in arrays]


SORT_CONFIGS = [{}, {"WM_SORT_MEDIUM_CTAS": "1"}, {"WM_SORT_MEDIUM_CTAS": "3"}, {"WM_SORT_GIANT_MIN": "2048", "WM_SORT_GIANT_CTAS": "1"},
                {"WM_SORT_GIANT_MIN": "20000", "WM_SORT_GIANT_CTAS": "2", "WM_SORT_MEDIUM_CTAS": "2"}, {"WM_SORT_TWO_MIN": "0"},
                {"WM_SORT_MEDIUM": "0"}, {"WM_SORT_GIANT": "0", "WM_SORT_MEDIUM": "0"}]


@pytest.mark.parametrize("env", SORT_CONFIGS, ids=_cfg_id)
def test_sort_task_loop_matches_oracle(sort_case, env, tmp_path):
    """radix_sort_128x on 40 arrays above 2048 in one call: both words of every element, so the tie order is checked."""
    src, arrays, exp = sort_case
    got = _unpack(_device("sort", src, env, tmp_path), "a")
    for i, (a, e, g) in enumerate(zip(arrays, exp, got)):
        g = g.reshape(-1, 2)
        if not np.array_equal(e, g):
            bad = np.flatnonzero((e != g).any(axis=1))
            raise AssertionError(f"array {i} (n {len(a)}): {len(bad)} elements differ, first at {bad[0]}: exp {e[bad[0]]} got {g[bad[0]]}")


# ---------------------------------------------------------------------------------------------------------------- chain

CHAIN_PRM = [(5000, 1000, 5000, 500, 25, 5000), (16000, 1000, 16000, 2000, 25, 5000), (5000, 50, 5000, 500, 3, 20)]


@pytest.fixture(scope="module")
def chain_case(tmp_path_factory, n_sm):
    rng = np.random.default_rng(79)
    giant = [_tandem_anchors(rng, 300, 200, 340), _tandem_anchors(rng, 120, 100, 171), make_anchors(rng, 9000, repeats=True),
             make_span_anchors(rng, 9000, repeats=True), _span_tandem(rng), make_anchors(rng, 5000, repeats=False),
             make_span_anchors(rng, 5000, repeats=False), make_span_anchors(rng, 4097, repeats=True), _tandem_anchors(rng, 80, 50, 200),
             make_anchors(rng, 3000, repeats=True), _tandem_anchors(rng, 60, 40, 64), make_anchors(rng, 2049, repeats=False)]
    giant += [deep_array(), zone_array()]  # candidates below the tile kernel's ring, by construction (test_chain_tile_cta.py)
    assert len(giant) >= 14 and min(len(a) for a in giant) == 2049
    # checked on the CPU at the tile kernel's constants before anything runs on the device: scans that need the locked deep path,
    # whole groups of them in one tile (warps contend for the lock), and scans that refill the candidate list
    n_deep, per_tile, n_refill = tile_kernel_reach(giant, CHAIN_PRM)
    assert n_deep > 0 and per_tile >= 8 and n_refill > 0, (n_deep, per_tile, n_refill)
    # medium tasks (129-2048 anchors): more than the ring kernel's warps at any ring size (3 CTAs of 4 warps per SM at 512)
    medium = [(make_span_anchors if j % 3 == 0 else make_anchors)(rng, int(n), repeats=bool(j & 1))
              for j, n in enumerate(rng.integers(129, 2049, size=3 * n_sm * 4 + 40))]
    # small tasks (<= 128 anchors): more than the small ring kernel's 6 CTAs of 8 warps per SM
    small = [(make_span_anchors if j % 4 == 0 else make_anchors)(rng, int(n), repeats=bool(j & 1))
             for j, n in enumerate(rng.integers(2, 129, size=6 * n_sm * 8 + 100))]
    edge = [make_anchors(rng, 0), make_anchors(rng, 1), make_anchors(rng, 1, repeats=True), make_anchors(rng, 0)]
    arrays = giant + medium + small + edge
    order = rng.permutation(len(arrays))  # tasks arrive in any order; the launcher sorts them by size
    arrays = [arrays[i] for i in order]
    assert sum(len(a) > 64 for a in arrays) > 2 * n_sm  # WM_CHAIN_BT_CTA_MIN=64: more CTA-backtrack tasks than its 2 CTAs per SM
    src = str(tmp_path_factory.mktemp("chain") / "in.npz")
    inp = {"prm": np.array(CHAIN_PRM, dtype=np.int64)}
    _pack(inp, "a", arrays)
    np.savez(src, **inp)
    exp = [[ol.oracle_chain(a, mx, mn, my, bw, max_skip=skip, max_iter=it) for a in arrays] for mx, mn, my, bw, skip, it in CHAIN_PRM]
    return src, arrays, exp


CHAIN_CONFIGS = [{}, {"WM_CHAIN_TILE_CTAS": "1"}, {"WM_CHAIN_TILE_CTAS": "1", "WM_CHAIN_TILE_MIN": "1"}, {"WM_CHAIN_BT_CTA_MIN": "64"},
                 {"WM_CHAIN_RING": "512"}, {"WM_CHAIN_RING": "2048"}, {"WM_CHAIN_MODE": "0"}]


@pytest.mark.parametrize("env", CHAIN_CONFIGS, ids=_cfg_id)
def test_chain_task_loop_matches_oracle(chain_case, env, tmp_path):
    """mm_chain_dp on thousands of tasks of every class in one call, for the three parameter sets of test_chain_matches_oracle:
    the chain list u and the chained anchors."""
    src, arrays, exp = chain_case
    z = _device("chain", src, env, tmp_path, timeout=900)
    for k, prm in enumerate(CHAIN_PRM):
        us, bs = _unpack(z, f"u{k}"), _unpack(z, f"b{k}")
        for i, a in enumerate(arrays):
            ue, be = exp[k][i]
            assert np.array_equal(np.asarray(ue).reshape(-1), us[i]), (prm, i, len(a), "u", len(ue), len(us[i]))
            assert np.array_equal(np.asarray(be).reshape(-1), bs[i]), (prm, i, len(a), "b")


# ---------------------------------------------------------------------------------------------------------------- DP

def _dp_batches():
    """(name, queries, targets, mat, gaps, w, zdrop, end_bonus, flag) of the DP corpora."""
    out = []
    rng = np.random.default_rng(900)  # test_extd2_random_batch, seed 0
    Q, T, W, Z, E, F = [], [], [], [], [], []
    for _ in range(400):
        tlen = int(rng.choice([1, 5, 16, 17, 33, 100, 250, 300, 700, 1100, 2500]))
        q, t = rand_pair(rng, tlen, err=float(rng.choice([0.02, 0.1, 0.3])), drift=int(rng.choice([0, 0, 30, 120, 400])),
                         n_runs=int(rng.integers(0, 3)))
        Q.append(q); T.append(t)
        W.append(int(rng.choice([5, 20, 50, 100, 751, 3001]))); Z.append(int(rng.choice([400, 200, 50, -1])))
        E.append(int(rng.choice([-1, 0, 10]))); F.append(FLAGS[int(rng.integers(0, len(FLAGS)))])
    out.append(("random", Q, T, ol.simple_mat(), (4, 2, 24, 1), W, Z, E, F))
    rng = np.random.default_rng(5)  # test_extd2_long_end_extension_and_empty
    q, t = rand_pair(rng, 9000, err=0.08, drift=300)
    out.append(("long_and_empty", [q, q[:1], np.zeros(0, np.uint8), q[:300]], [t, t[:1], t[:10], np.zeros(0, np.uint8)], ol.simple_mat(),
                (4, 2, 24, 1), [3001, 751, 751, 751], [400] * 4, [-1] * 4, [0x40, 0x40, 0, 0]))
    rng = np.random.default_rng(77)  # test_extd2_asm_scoring_and_swapped_gaps
    for a, b, go, ge, go2, ge2 in [(1, 4, 6, 2, 26, 1), (2, 4, 24, 1, 4, 2)]:
        Q, T = zip(*[rand_pair(rng, int(rng.integers(20, 900)), err=0.05, drift=int(rng.choice([0, 50]))) for _ in range(64)])
        out.append((f"asm{a},{b},{go},{ge},{go2},{ge2}", list(Q), list(T), ol.simple_mat(a, b, 1), (go, ge, go2, ge2), [200] * 64, [200] * 64,
                    [-1] * 64, [FLAGS[i % 4] for i in range(64)]))
    # early out: a mismatch above 2(q + e) makes the reference return before the sweep; with jobs above the cooperative
    # threshold (>= 300 000 band cells: tlen 2500 at w 3001), whose state slices live in global memory
    rng = np.random.default_rng(13)
    Q, T, W, F = [], [], [], []
    for i in range(48):
        q, t = rand_pair(rng, int(rng.choice([2500, 2500, 4000, 300, 40, 1])), err=0.05, drift=int(rng.choice([0, 50])))
        Q.append(q); T.append(t); W.append([3001, 751, 3001, -1][i % 4]); F.append(FLAGS[i % 4] | (0x10 if i % 3 == 0 else 0))
    Q += [np.zeros(0, np.uint8), Q[0][:10]]; T += [T[0][:10], np.zeros(0, np.uint8)]; W += [751, 751]; F += [0, 0]
    n = len(Q)
    for gaps in [(4, 2, 24, 1), (4, 2, 4, 2)]:
        out.append((f"early_out{gaps}", Q, T, ol.simple_mat(1, 13), gaps, W, [400] * n, [-1] * n, F))
    return out


def _coop(qlen, tlen, w):
    """The extd2 jobs the cooperative sweep takes at the defaults: those with a global state slice (wm_extd2_plan: more than
    512 target or 640 query cells) that wm_dp_is_coop (wm_common.cuh) selects."""
    if w < 0:
        w = max(qlen, tlen)
    fits = (tlen + 15) // 16 * 16 <= 512 and qlen <= 640
    return not fits and min(qlen, tlen, w + 1) >= 384 and tlen * min(qlen, 2 * w + 1) >= 300000


@pytest.fixture(scope="module")
def dp_case(tmp_path_factory):
    batches = _dp_batches()
    inp = {"n_batches": np.array(len(batches))}
    exp = []
    for k, (name, Q, T, mat, gaps, W, Z, E, F) in enumerate(batches):
        p = f"{k}_"
        _pack(inp, p + "q", Q); _pack(inp, p + "t", T)
        inp[p + "mat"], inp[p + "gaps"] = mat, np.array(gaps)
        for f, v in (("w", W), ("zdrop", Z), ("eb", E), ("flag", F)):
            inp[p + f] = np.array(v, dtype=np.int64)
        single = gaps[:2] == gaps[2:]
        exp.append([ol.oracle_extz2(Q[i], T[i], mat, *gaps[:2], W[i], Z[i], E[i], F[i]) if single else
                    ol.oracle_extd2(Q[i], T[i], mat, *gaps, W[i], Z[i], E[i], F[i]) for i in range(len(Q))])
    name, Q, T, _, _, W, _, _, _ = batches[-2]
    assert name.startswith("early_out") and sum(_coop(len(q), len(t), w) for q, t, w in zip(Q, T, W)) >= 8
    src = str(tmp_path_factory.mktemp("dp") / "in.npz")
    np.savez(src, **inp)
    return src, batches, exp


@pytest.mark.parametrize("env", [{}, {"WM_DP_V1": "1"}, {"WM_DP_COOP": "0"}], ids=_cfg_id)
def test_dp_variants_match_oracle(dp_case, env, tmp_path):
    """ksw_extd2 / ksw_extz2 under the default fill (v2 sweep, big jobs on a whole CTA), the v1 fill and big jobs on one warp
    with a global state slice: all eleven ksw_extz_t fields and the CIGAR.  Includes a scoring on which the reference
    returns before the sweep, with jobs the cooperative sweep takes."""
    src, batches, exp = dp_case
    z = _device("dp", src, env, tmp_path)
    bad = []
    for k, (name, Q, T, mat, gaps, W, Z, E, F) in enumerate(batches):
        ez, cig = z[f"{k}_ez"], _unpack(z, f"{k}_cig")
        for i in range(len(Q)):
            e0, c0 = exp[k][i]
            if not (np.array_equal(e0, ez[i]) and np.array_equal(c0, cig[i])):
                bad.append(f"{name} job {i}: qlen {len(Q[i])} tlen {len(T[i])} w {W[i]} flag {hex(F[i])} coop {_coop(len(Q[i]), len(T[i]), W[i])}: "
                           f"exp {list(e0)} got {list(ez[i])}")
    assert not bad, f"{len(bad)} jobs differ:\n" + "\n".join(bad[:20])
