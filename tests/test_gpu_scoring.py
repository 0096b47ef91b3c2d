"""The device DP kernels at every scoring the mapper accepts (tee_lib.SCORINGS): ksw_extd2 (ksw_extz2 for one gap pair) and
ksw_ll against the oracle, bit for bit.  The oracle is pinned to the reference's functions at the same scorings by
tests/test_oracle_vs_ref.py (test_every_scoring_matches_reference).

Each scoring's batch holds jobs of every class of the fill: state in the warp's shared-memory slice (tlen16 <= 512 and
qlen <= 640), state in a global slice, and jobs the cooperative sweep takes (two gap pairs only: the single-affine sweep
has no cooperative form); for two gap pairs, alignments with a gap longer than long_thres, and alignments that start with
a gap of about long_thres, so that the first row and column (-e below long_thres, long_diff at it, -e2 beyond) decide the
score; N runs in both sequences.  The batches run under the default fill, the v1 fill and without the cooperative sweep,
each in a child process (the switches are read once per process)."""
import numpy as np
import pytest

import oracle_lib as ol
import tee_lib as T
from test_gpu_task_loops import _cfg_id, _coop, _device, _pack, _unpack
from test_oracle_vs_ref import FLAGS, rand_pair

pytestmark = pytest.mark.gpu
NAMES = sorted(T.SCORINGS)


def _long_thres(q, e, q2, e2):
    """src/ksw2_extd2_sse.c:94-96, after the swap that puts the smaller q + e first."""
    if q2 + e2 < q + e:
        q, e, q2, e2 = q2, e2, q, e
    t = (q2 - q) // (e - e2) - 1
    return t + (q2 + e2 + t * e2 > q + e + t * e)


def _fits(qlen, tlen):
    return (tlen + 15) // 16 * 16 <= 512 and qlen <= 640


def _mutate(rng, s, err):
    """Substitutions only, at rate err."""
    s = s.copy()
    k = rng.random(len(s)) < err
    s[k] = (s[k] + rng.integers(1, 4, size=int(k.sum()))) & 3
    return s


def _batch(rng, scoring):
    """(Q, T, W, Z, E, F) of one scoring's batch."""
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[scoring]
    lt = _long_thres(q, e, q2, e2) if (q, e) != (q2, e2) else 20
    err = 0.01 if b >= 19 else 0.04  # the asm5-like scorings Z-drop noisier pairs early
    jobs = []

    def add(qs, ts, w, flag, zdrop=400, eb=-1):
        jobs.append((np.ascontiguousarray(qs, np.uint8), np.ascontiguousarray(ts, np.uint8), w, zdrop, eb, flag))

    for i in range(24):  # shared-memory slice
        qs, ts = rand_pair(rng, int(rng.choice([1, 5, 16, 17, 33, 100, 250, 480])), err=err, drift=int(rng.choice([0, 0, 30, 60])),
                           n_runs=int(rng.integers(0, 3)))
        add(qs[:640], ts, int(rng.choice([5, 50, 200, 751])), FLAGS[i % 4] | (0x10 if i % 5 == 0 else 0), int(rng.choice([400, 200, 50, -1])),
            int(rng.choice([-1, 0, 10, 1000])))
    for i in range(8):  # global state slice, band too narrow for the cooperative sweep
        qs, ts = rand_pair(rng, int(rng.choice([600, 900, 1300])), err=err, drift=int(rng.choice([0, 40])), n_runs=int(rng.integers(0, 2)))
        add(qs, ts, int(rng.choice([20, 100])), FLAGS[i % 4])
    for i in range(6):  # the cooperative sweep: >= 300 000 band cells, every dimension >= 384
        qs, ts = rand_pair(rng, int(rng.choice([1700, 2500])), err=err, drift=int(rng.choice([0, 60])), n_runs=1)
        add(qs, ts, [751, 3001][i & 1], FLAGS[i % 4])
    for tl, w in [(300, 751), (900, 100), (2000, 3001)]:  # one size per class
        # gaps of lt - 1 .. lt + 2 and a longer one at the start of the alignment, where the first row or column gives
        # their cost (a gap of lt bases ends on the boundary cell long_thres - 1, one of lt + 1 on long_thres), and in
        # the middle of the alignment
        for j, g in enumerate([lt - 1, lt, lt + 1, lt + 2, lt + int(rng.integers(3, 40))]):
            ts = rng.integers(0, 4, size=tl, dtype=np.uint8)
            body = _mutate(rng, ts, err / 2)
            ins = rng.integers(0, 4, size=g, dtype=np.uint8)
            # no match at the start of the other placements of the leading gap: the gap is the first CIGAR operation
            if j & 1:
                ts[:6] = (body[g:g + 6] + rng.integers(1, 4, size=6)) & 3
            else:
                ins[:6] = (ts[:6] + rng.integers(1, 4, size=6)) & 3
            lead = body[g:] if j & 1 else np.concatenate([ins, body])
            mid = np.concatenate([body[:tl // 2], body[tl // 2 + g:]]) if j & 1 else np.concatenate([body[:tl // 2], ins, body[tl // 2:]])
            for flag in (0, 0x08):
                add(lead, ts, w, flag)
            add(mid, ts, w, 0x40)
    if sc_ambi != 1:  # N runs of both sequences in every class
        for tl, w in [(200, 751), (700, 100), (2000, 3001)]:
            ts = rng.integers(0, 4, size=tl, dtype=np.uint8)
            qs = _mutate(rng, ts, err / 2)
            for p in rng.integers(0, tl - 30, size=4):
                qs[p:p + int(rng.integers(1, 20))] = 4
            for p in rng.integers(0, tl - 30, size=3):
                ts[p:p + int(rng.integers(1, 10))] = 4
            for flag in (0, 0x08, 0x40):
                add(qs, ts, w, flag)
    order = rng.permutation(len(jobs))
    return [list(x) for x in zip(*[jobs[i] for i in order])]


def _expected(scoring, Q, Tg, W, Z, E, F):
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[scoring]
    mat = ol.simple_mat(a, b, sc_ambi)
    if (q, e) == (q2, e2):
        return [ol.oracle_extz2(Q[i], Tg[i], mat, q, e, W[i], Z[i], E[i], F[i]) for i in range(len(Q))]
    return [ol.oracle_extd2(Q[i], Tg[i], mat, q, e, q2, e2, W[i], Z[i], E[i], F[i]) for i in range(len(Q))]


@pytest.fixture(scope="module")
def scoring_case(tmp_path_factory):
    inp = {"n_batches": np.array(len(NAMES))}
    batches, exp = [], []
    for k, name in enumerate(NAMES):
        a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[name]
        Q, Tg, W, Z, E, F = _batch(np.random.default_rng(5000 + k), name)
        p = f"{k}_"
        _pack(inp, p + "q", Q); _pack(inp, p + "t", Tg)
        inp[p + "mat"], inp[p + "gaps"] = ol.simple_mat(a, b, sc_ambi), np.array([q, e, q2, e2])
        for f, v in (("w", W), ("zdrop", Z), ("eb", E), ("flag", F)):
            inp[p + f] = np.array(v, dtype=np.int64)
        batches.append((name, Q, Tg, W, Z, E, F))
        exp.append(_expected(name, Q, Tg, W, Z, E, F))
    src = str(tmp_path_factory.mktemp("scoring") / "in.npz")
    np.savez(src, **inp)
    return src, batches, exp


def test_batches_hold_every_job_class(scoring_case):
    """Host-side: the classes the module docstring promises are in every scoring's batch, and the inputs reach them."""
    _, batches, exp = scoring_case
    for (name, Q, Tg, W, Z, E, F), ex in zip(batches, exp):
        a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[name]
        dims = [(len(qs), len(ts), w) for qs, ts, w in zip(Q, Tg, W)]
        assert sum(_fits(ql, tl) for ql, tl, w in dims) >= 20, name
        assert sum(not _fits(ql, tl) and not _coop(ql, tl, w) for ql, tl, w in dims) >= 8, name
        assert sum(_coop(ql, tl, w) for ql, tl, w in dims) >= 6, name
        early_out = max(b, sc_ambi) > 2 * (q + e)
        if early_out:  # no job is swept
            assert all(len(c) == 0 and ez[0] == 0 for ez, c in ex), name
            continue
        if (q, e) != (q2, e2):
            lt = _long_thres(q, e, q2, e2)
            long_gaps = sum(any((c & 0xf) in (1, 2) and (c >> 4) > lt for c in cig) for _, cig in ex)
            assert long_gaps >= 6, (name, long_gaps)
            # gap fills that open with a gap of lt and of lt + 1 bases, in each class (not under match_hi: with -A far
            # above -B, random bases align at a profit and the gap moves away from the start)
            for ln in (lt, lt + 1) if a < b else ():
                lead = [(len(qs), len(ts), w) for qs, ts, w, f, (_, cig) in zip(Q, Tg, W, F, ex)
                        if not f & 0x40 and len(cig) and (cig[0] & 0xf) in (1, 2) and (cig[0] >> 4) == ln]
                assert any(_fits(ql, tl) for ql, tl, w in lead) and any(_coop(ql, tl, w) for ql, tl, w in lead), (name, ln, lead)
                assert any(not _fits(ql, tl) and not _coop(ql, tl, w) for ql, tl, w in lead), (name, ln, lead)
        if sc_ambi != 1:
            n_jobs = sum(((qs == 4).any() or (ts == 4).any()) and len(cig) > 0 for qs, ts, (_, cig) in zip(Q, Tg, ex))
            assert n_jobs >= 6, (name, n_jobs)


@pytest.mark.parametrize("env", [{}, {"WM_DP_V1": "1"}, {"WM_DP_COOP": "0"}], ids=_cfg_id)
def test_dp_matches_oracle_at_every_scoring(scoring_case, env, tmp_path):
    """All eleven ksw_extz_t fields and the CIGAR of every job, at every scoring, under each fill variant."""
    src, batches, exp = scoring_case
    z = _device("dp", src, env, tmp_path)
    bad = []
    for k, (name, Q, Tg, W, Z, E, F) in enumerate(batches):
        ez, cig = z[f"{k}_ez"], _unpack(z, f"{k}_cig")
        for i in range(len(Q)):
            e0, c0 = exp[k][i]
            if not (np.array_equal(e0, ez[i]) and np.array_equal(c0, cig[i])):
                bad.append(f"{name} job {i}: qlen {len(Q[i])} tlen {len(Tg[i])} w {W[i]} flag {hex(F[i])} coop {_coop(len(Q[i]), len(Tg[i]), W[i])}: "
                           f"exp {list(e0)} got {list(ez[i])}")
    assert not bad, f"{len(bad)} jobs differ:\n" + "\n".join(bad[:20])


@pytest.mark.parametrize("name", NAMES)
def test_ll_matches_oracle_at_every_scoring(name):
    """ksw_ll_i16 (mm_align1_inv, src/align.c:72-87, calls it with the options' q and e and matrix) at each scoring."""
    from winnowmap_b200 import kernels
    a, b, q, e, q2, e2, sc_ambi = T.SCORINGS[name]
    mat = ol.simple_mat(a, b, sc_ambi)
    rng = np.random.default_rng(6000 + NAMES.index(name))
    Q, Tg = [], []
    for i in range(120):
        tl = int(rng.choice([1, 7, 8, 9, 40, 200, 600]))
        if i % 2:
            qs, ts = rand_pair(rng, tl, err=0.1, drift=int(rng.choice([0, 30])), n_runs=int(rng.integers(0, 3)))
        else:
            ts, qs = rng.integers(0, 5, size=tl, dtype=np.uint8), rng.integers(0, 5, size=int(rng.integers(1, 300)), dtype=np.uint8)
        Q.append(qs); Tg.append(ts)
    got = kernels.ksw_ll_batch(Q, Tg, mat, q, e)
    exp = np.array([ol.oracle_ll(qs, ts, mat, q, e) for qs, ts in zip(Q, Tg)], dtype=np.int32)
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert len(bad) == 0, f"{len(bad)} jobs differ, first {bad[0]}: exp {exp[bad[0]]} got {got[bad[0]]}"
