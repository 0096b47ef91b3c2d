"""GPU parity for the sketch / sort / chain kernels (through the C ABI) against the CPU oracle."""
import os

import numpy as np
import pytest

import oracle_lib as ol
from test_oracle_vs_ref import make_anchors, make_span_anchors

pytestmark = pytest.mark.gpu
TESTS_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT_DIR = os.path.dirname(TESTS_DIR)


def _rand_seq(rng, n):
    return bytes(b"ACGT"[c] for c in rng.integers(0, 4, size=n, dtype=np.uint8))


def _seq_set(rng, kmers, k):
    base = _rand_seq(rng, 40000)
    seqs = [base, base[:2000], base[5000:5130], base[:14], b"ACGTACGTAC", b""]
    s2 = bytearray(base[:9000])
    for p in range(500, 8000, 900):
        L = int(rng.integers(1, 80))
        s2[p:p + L] = b"N" * L
    seqs.append(bytes(s2))
    unit = _rand_seq(rng, 7)
    seqs.append(base[:300] + unit * 60 + base[300:900] + b"A" * 120 + base[900:1500] + (b"AC" * 70) + base[1500:2000] + b"acgtn" * 30 + base[2000:2500])
    if len(kmers):
        planted = bytearray(base[:6000])
        for j in range(min(40, len(kmers))):
            km = int(kmers[j])
            st = "".join("ACGT"[(km >> (2 * (k - 1 - i))) & 3] for i in range(k)).encode()
            planted[100 + j * 110: 100 + j * 110 + k] = st
        seqs.append(bytes(planted))
    # many windows of one read, as in stage 1
    seqs += [base[i:i + 2000] for i in range(0, 20000, 2000)]
    seqs += [base[:1023], base[1:1025], base[2:1027]]  # around the 1024-base sketch tile
    return seqs


# k = 27 / 28: the largest k of the parallel order kernel and of the sequential one, at the smallest and largest w
@pytest.mark.parametrize("n_k,k,w", [(0, 15, 50), (255, 15, 50), (5000, 15, 50), (300, 19, 50), (255, 15, 10), (0, 16, 20), (0, 6, 20),
                                     (0, 27, 1), (255, 27, 255), (0, 28, 1), (255, 28, 255)])
def test_sketch_matches_oracle(n_k, k, w):
    from winnowmap_b200 import kernels
    rng = np.random.default_rng(1000 + n_k + k + w)
    kmers = rng.integers(0, 1 << (2 * k), size=n_k, dtype=np.uint64)
    ob = ol.OracleBloom(kmers)
    gb = kernels.Bloom(kmers)
    assert gb.bits() == ob.bits()
    assert np.array_equal(gb.table(), ob.table())
    seqs = _seq_set(rng, kmers, k)
    if k % 2 == 0:
        seqs.append(seqs[0][:1000] + b"ACGTACGTACGTACGTAATT" * 5 + seqs[0][1000:3000])
    rids = np.arange(len(seqs)) % 3
    got = kernels.sketch_batch(gb, seqs, w, k, rids)
    for i, s in enumerate(seqs):
        exp = ol.oracle_sketch(s, w, k, int(rids[i]), ob) if len(s) else np.zeros((0, 2), np.uint64)
        assert np.array_equal(exp, got[i]), (i, len(s), len(exp), len(got[i]))


def test_sort_matches_oracle_with_ties():
    from winnowmap_b200 import kernels
    rng = np.random.default_rng(3)
    arrays = []
    for n in [0, 1, 2, 63, 64, 65, 200, 1000, 5000, 70000]:
        for key_bits in [3, 12, 28, 64]:
            hi = (1 << key_bits) - 1
            x = rng.integers(0, hi, size=n, dtype=np.uint64, endpoint=True)
            if key_bits == 64 and n:
                x[::3] = x[0]
            arrays.append(np.stack([x, np.arange(n, dtype=np.uint64)], axis=1))
    got = kernels.radix_sort_128x_batch(arrays)
    for a, g in zip(arrays, got):
        assert np.array_equal(ol.oracle_sort128(a), g), len(a)


def test_sort_two_bucket_passes_match_oracle():
    """Passes with exactly two non-empty buckets take a closed form in the walker kernels (csrc/seed.cu: wm_gs_two_bucket_pass)
    instead of the serial walk of src/ksort.h:126-138: anchor-like arrays with a strand bit (from one stray element to an even
    split), positions that straddle a 64 kb / 16 Mb boundary, heavy ties, sizes on both sides of the kernel's size classes."""
    from winnowmap_b200 import kernels
    rng = np.random.default_rng(31)
    arrays = []
    for n in [600, 2049, 2500, 9000, 40000, 150000]:
        for frac in [0.0, 0.0005, 0.03, 0.5, 0.97]:
            base = int(rng.choice([(1 << 16) * 37 - 700, (1 << 24) * 3 - 5000, 123456789]))
            span = int(rng.choice([1500, 40000, 140000]))
            pos = base + rng.integers(0, span, size=n)
            if rng.random() < 0.5:  # tandem-like: few distinct positions, many ties
                pos = base + (rng.integers(0, max(2, n // 40), size=n) * 171) % span
            x = pos.astype(np.uint64) | (np.uint64(rng.integers(0, 3)) << np.uint64(32))
            x = x | ((rng.random(n) < frac).astype(np.uint64) << np.uint64(63))
            arrays.append(np.stack([x, np.arange(n, dtype=np.uint64)], axis=1))
    got = kernels.radix_sort_128x_batch(arrays)
    for a, g in zip(arrays, got):
        assert np.array_equal(ol.oracle_sort128(a), g), len(a)


@pytest.mark.parametrize("seed", range(3))
def test_chain_matches_oracle(seed):
    from winnowmap_b200 import kernels
    rng = np.random.default_rng(500 + seed)
    arrays = [make_anchors(rng, n, repeats=bool((seed + i) & 1)) for i, n in enumerate([0, 1, 3, 10, 40, 100, 100, 700, 3000, 9000] * 3)]
    arrays += [make_span_anchors(rng, n, repeats=bool((seed + i) & 1)) for i, n in enumerate([1, 10, 100, 700, 3000, 9000])]
    for prm in [dict(max_dist_x=5000, min_dist_x=1000, max_dist_y=5000, bw=500), dict(max_dist_x=16000, min_dist_x=1000, max_dist_y=16000, bw=2000),
                dict(max_dist_x=5000, min_dist_x=50, max_dist_y=5000, bw=500, max_iter=20, max_skip=3)]:
        got = kernels.chain_dp_batch(arrays, **prm)
        for a, (u, b) in zip(arrays, got):
            ue, be = ol.oracle_chain(a, prm["max_dist_x"], prm["min_dist_x"], prm["max_dist_y"], prm["bw"],
                                     max_skip=prm.get("max_skip", 25), max_iter=prm.get("max_iter", 5000))
            assert np.array_equal(ue, u), (len(a), len(ue), len(u))
            assert np.array_equal(be, b), len(a)


def _tandem_anchors(rng, n_q, n_copies, unit, span=15):
    """Anchors of a read crossing a tandem array: every query minimizer hits every copy of the unit (many ties in x)."""
    q0 = np.sort(rng.choice(np.arange(50, 50 + n_q * 11), size=n_q, replace=False)).astype(np.int64)
    x, y = [], []
    for c in range(n_copies):
        x.append(1000 + c * unit + (q0 % unit))
        y.append(q0)
    x = np.concatenate(x).astype(np.uint64); y = np.concatenate(y).astype(np.uint64)
    xy = np.stack([x, np.uint64(span) << np.uint64(32) | y], axis=1)
    return ol.ref_sort128(xy) if ol.have_ref() else ol.oracle_sort128(xy)


def _span_tandem(rng):
    """A tandem lattice whose anchors carry spans from 1 to 255 and, on some, the tandem flag (bit 42 of y)."""
    a = _tandem_anchors(rng, 150, 60, 171)
    span = rng.integers(1, 256, size=len(a)).astype(np.uint64)
    tandem = (rng.random(len(a)) < 0.3).astype(np.uint64) << np.uint64(42)
    a[:, 1] = (a[:, 1] & np.uint64(0xffffffff)) | span << np.uint64(32) | tandem
    return ol.oracle_sort128(a)  # ties in x are ordered by y, flags included


def _giant_chain_arrays():
    from test_chain_tile_cta import deep_array, zone_array
    rng = np.random.default_rng(78)
    return [_tandem_anchors(rng, 120, 100, 171), _tandem_anchors(rng, 300, 200, 340), _tandem_anchors(rng, 60, 40, 64), make_anchors(rng, 9000, repeats=True),
            make_anchors(rng, 5000, repeats=False), make_anchors(rng, 33, repeats=True), make_anchors(rng, 1, repeats=False),
            make_span_anchors(rng, 9000, repeats=True), make_span_anchors(rng, 5000, repeats=False), _span_tandem(rng), deep_array(), zone_array()]


@pytest.mark.parametrize("tile_min", [None, 1])
def test_chain_giant_tasks_match_oracle(tile_min, tmp_path):
    """Giant tasks go through the tile kernel (one CTA per task, one warp per anchor of a 32-anchor tile, csrc/chain.cu): tandem
    lattices of up to 60 000 anchors, dense repeats and arrays crafted so that scans need the anchors below the kernel's ring (the
    locked deep path), against the oracle.  tile_min = 1 sends every task through that kernel.  In a child process: the kernel spins
    on shared-memory flags, a bug there must not hang the session."""
    import subprocess
    import sys
    from test_chain_tile_cta import tile_kernel_reach
    # on the CPU at the kernel's constants, before the device runs: deep scans, a tile of them, list refills
    n_deep, per_tile, n_refill = tile_kernel_reach(_giant_chain_arrays(), [(5000, 1000, 5000, 500, 25, 5000)])
    assert n_deep > 0 and per_tile >= 8 and n_refill > 0, (n_deep, per_tile, n_refill)
    code = r'''
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np
import oracle_lib as ol
from winnowmap_b200 import kernels
from test_oracle_vs_ref import make_anchors, make_span_anchors
from test_gpu_stages import _giant_chain_arrays
arrays = _giant_chain_arrays()
for prm in [dict(max_dist_x=5000, min_dist_x=1000, max_dist_y=5000, bw=500), dict(max_dist_x=16000, min_dist_x=1000, max_dist_y=16000, bw=2000),
            dict(max_dist_x=5000, min_dist_x=50, max_dist_y=5000, bw=500, max_iter=20, max_skip=3)]:
    got = kernels.chain_dp_batch(arrays, **prm)
    for a, (u, b) in zip(arrays, got):
        ue, be = ol.oracle_chain(a, prm["max_dist_x"], prm["min_dist_x"], prm["max_dist_y"], prm["bw"], max_skip=prm.get("max_skip", 25), max_iter=prm.get("max_iter", 5000))
        assert np.array_equal(ue, u) and np.array_equal(be, b), (len(a), prm)
print("giant ok")
''' % (ROOT_DIR, TESTS_DIR)
    env = dict(os.environ)
    if tile_min is not None:
        env["WM_CHAIN_TILE_MIN"] = str(tile_min)
    out = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    assert out.returncode == 0 and b"giant ok" in out.stdout, out.stdout[-2000:]


def test_ksw_ll_matches_oracle():
    """wm_ksw_ll_batch (ksw_ll_qinit + ksw_ll_i16, src/ksw2_ll_sse.c:32,80): score and the tie rules of the two end
    coordinates, against the oracle (itself pinned to the reference's function by tests/test_oracle_vs_ref.py)."""
    from winnowmap_b200 import kernels
    rng = np.random.default_rng(91)
    mat = ol.simple_mat()
    qs, ts = [], []
    for i in range(300):
        tl = int(rng.integers(1, 600)); ql = int(rng.integers(1, 400))
        t = rng.integers(0, 4, size=tl, dtype=np.uint8)
        if i % 3 == 0 and tl > ql + 5:  # the query is a noisy piece of the target (the inversion-rescue case, src/align.c:72-87)
            s0 = int(rng.integers(0, tl - ql))
            q = t[s0:s0 + ql].copy()
            m = rng.random(ql) < 0.1
            q[m] = (q[m] + 1) & 3
        elif i % 3 == 1:
            q = np.tile(t[:max(1, min(7, tl))], ql // max(1, min(7, tl)) + 1)[:ql].copy()  # periodic: many equal maxima
        else:
            q = rng.integers(0, 5, size=ql, dtype=np.uint8)
        qs.append(q); ts.append(t)
    for gapo, gape in [(4, 2), (6, 1)]:
        got = kernels.ksw_ll_batch(qs, ts, mat, gapo, gape)
        for i, (q, t) in enumerate(zip(qs, ts)):
            assert tuple(got[i]) == tuple(ol.oracle_ll(q, t, mat, gapo, gape)), (i, len(q), len(t))


def test_chain_dense_formulation_matches_oracle(tmp_path):
    """The dense-candidate forward pass (csrc/chain_dev.cuh) through the C ABI, in a child process: the switch is read
    once per process, and a CUDA fault must not take the test session with it."""
    import subprocess
    import sys
    code = r'''
import sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np
import oracle_lib as ol
from winnowmap_b200 import kernels
from test_oracle_vs_ref import make_anchors
rng = np.random.default_rng(77)
arrays = [make_anchors(rng, n, repeats=bool(i & 1)) for i, n in enumerate([0, 5, 100, 1500, 3000, 9000, 9000])]
for prm in [dict(max_dist_x=5000, min_dist_x=1000, max_dist_y=5000, bw=500), dict(max_dist_x=5000, min_dist_x=50, max_dist_y=5000, bw=500, max_iter=20, max_skip=3)]:
    got = kernels.chain_dp_batch(arrays, **prm)
    for a, (u, b) in zip(arrays, got):
        ue, be = ol.oracle_chain(a, prm["max_dist_x"], prm["min_dist_x"], prm["max_dist_y"], prm["bw"], max_skip=prm.get("max_skip", 25), max_iter=prm.get("max_iter", 5000))
        assert np.array_equal(ue, u) and np.array_equal(be, b), len(a)
print("dense ok")
''' % (ROOT_DIR, TESTS_DIR)
    env = dict(os.environ, WM_CHAIN_DENSE="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    assert out.returncode == 0 and b"dense ok" in out.stdout, out.stdout[-2000:]
