"""ctypes bindings and inputs of the --heap-sort=yes checks: the oracle's restatement of collect_seed_hits_heap
(oracle/libwm_oracle_heap.so), the reference's own collect_seed_hits_heap / collect_seed_hits (oracle/_ref/libref_harness_heap.so),
the device code of the replay compiled for the host (tests/hostsim/heap_emul.cpp) and the crafted match sets they run on.
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol  # noqa: E402

_u64p = C.POINTER(C.c_uint64)
_u32p = C.POINTER(C.c_uint32)
_i32p = C.POINTER(C.c_int32)
_u8p = C.POINTER(C.c_uint8)
_libs = {}

F_NO_DIAG, F_NO_DUAL, F_FOR_ONLY, F_REV_ONLY = 0x001, 0x002, 0x100000, 0x200000
SKIP_NO_DIAG, SKIP_NO_DUAL, SKIP_FOR_ONLY, SKIP_REV_ONLY, SKIP_NAME_EQ = 1, 2, 4, 8, 16
K, W = 15, 5

# WM_RECORD_REF=1 (with oracle/_ref built) recomputes every digest a test run reaches from the reference and rewrites the file.
HEAP_DIGESTS = os.path.join(ROOT, "tests", "golden", "heap_ref_digests.json")
_digests = None


def have_ref():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_harness_heap.so"))


def assert_ref(key, got, ref_fn):
    """got equals what the reference computes: against the recorded digest, and live where the reference harness is built."""
    global _digests
    if _digests is None:
        _digests = json.load(open(HEAP_DIGESTS)) if os.path.exists(HEAP_DIGESTS) else {}
    if ol.recording():
        out = ref_fn()
        _digests[key] = ol.digest(*(out if isinstance(out, tuple) else (out,)))
        with open(HEAP_DIGESTS, "w") as f:
            json.dump(_digests, f, indent=0, sort_keys=True)
            f.write("\n")
    assert key in _digests, f"no reference digest for {key} (record with WM_RECORD_REF=1)"
    assert ol.digest(*(got if isinstance(got, tuple) else (got,))) == _digests[key], key


def oracle():
    if "oracle" not in _libs:
        so = os.path.join(ROOT, "oracle", "libwm_oracle_heap.so")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(os.path.join(ROOT, "oracle", "wm_oracle_heap.c")):
            subprocess.check_call([os.path.join(ROOT, "oracle", "build_heap.sh")], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmo_idx_build.restype = C.c_void_p
        L.wmo_idx_build.argtypes = [_u64p, C.c_long]
        L.wmo_idx_free.argtypes = [C.c_void_p]
        L.wmo_collect_seed_hits_heap.restype = C.c_long
        L.wmo_collect_seed_hits_heap.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_char_p, C.POINTER(C.c_char_p), _u32p, _u64p, C.c_long,
                                                 C.c_int, _u64p, C.c_long, _i32p, _u64p, _i32p]
        L.wmo_collect_seed_hits.restype = C.c_long
        L.wmo_collect_seed_hits.argtypes = [C.c_void_p, C.c_int, _u64p, C.c_long, C.c_int, _u64p, C.c_long, _i32p, _u64p, _i32p]
        _libs["oracle"] = L
    return _libs["oracle"]


def ref():
    if "ref" not in _libs:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_harness_heap.so"))
        L.ref_heap_idx.restype = C.c_void_p
        L.ref_heap_idx.argtypes = [C.c_char_p, C.c_int, C.c_int]
        L.ref_heap_idx_free.argtypes = [C.c_void_p]
        L.ref_heap_seed_hits.restype = C.c_long
        L.ref_heap_seed_hits.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_char_p, _u64p, C.c_long, C.c_int, _u64p, C.c_long,
                                         _i32p, _u64p, _i32p]
        _libs["ref"] = L
    return _libs["ref"]


def emul():
    if "emul" not in _libs:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_heap_emul_"), "lib.so")
        hs = os.path.join(ROOT, "tests", "hostsim")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                               os.path.join(hs, "heap_emul.cpp"), os.path.join(hs, "kernel_emul.cpp"), "-o", so])
        L = C.CDLL(so)
        L.wmt_heap_replay_dev.restype = C.c_long
        L.wmt_heap_replay_dev.argtypes = [_u64p, C.c_int, _i32p, _u64p, _u8p, _u64p, _u32p, _u32p, C.c_int, C.c_uint32, C.c_uint32, C.c_int,
                                          C.c_int, _u64p, C.c_long]
        _libs["emul"] = L
    return _libs["emul"]


def _p(a, t):
    return a.ctypes.data_as(t)


# ---- the index the crafted match sets look up ----
def _revcomp(s: bytes):
    return s.translate(bytes.maketrans(b"ACGT", b"TGCA"))[::-1]


def index_sequences():
    """(names, sequences): random sequence with tandem arrays of short units (copies of one k-mer in one list), reverse-complement
    copies (both strands in one list) and a sequence named like the reads of the self-mapping cases."""
    rng = np.random.default_rng(20261019)

    def rs(n):
        return bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)])

    def arr(unit, copies, div):
        out = bytearray()
        for _ in range(copies):
            u = bytearray(unit)
            for i in np.nonzero(rng.random(len(u)) < div)[0]:
                u[i] = b"ACGT"[int(rng.integers(0, 4))]
            out += u
        return bytes(out)

    a = rs(3000) + arr(rs(23), 60, 0.01) + rs(2000) + arr(rs(41), 25, 0.02) + rs(2500)
    b = rs(1500) + _revcomp(a[2000:7000]) + rs(1000) + arr(rs(17), 80, 0.0) + rs(1500)
    c = rs(2000) + a[4000:6000] + arr(rs(60), 12, 0.01) + rs(1200)
    d = rs(2500) + arr(rs(31), 30, 0.01) + rs(900)
    return [b"qself", b"m2", b"a1", b"z9"], [a, b, c, d]


class Index:
    """The oracle's index of index_sequences (every minimizer, no -W list), as the oracle's lookup and as CSR arrays."""

    def __init__(self):
        self.names, self.seqs = index_sequences()
        mz = np.concatenate([ol.oracle_sketch(s, W, K, rid, None) for rid, s in enumerate(self.seqs)])
        self.mz = mz
        self.h = oracle().wmo_idx_build(_p(np.ascontiguousarray(mz.reshape(-1)), _u64p), len(mz))
        h, y = mz[:, 0] >> np.uint64(8), mz[:, 1]
        o = np.lexsort((y, h))
        h, y = h[o], y[o]
        self.keys, first = np.unique(h, return_index=True)
        self.pos_off = np.append(first, len(h)).astype(np.uint64)
        self.pos = np.ascontiguousarray(y)
        self.seq_len = np.array([len(s) for s in self.seqs], np.uint32)
        self.name_rank = np.array([sum(m < n for m in self.names) for n in self.names], np.uint32)
        self.c_names = (C.c_char_p * len(self.names))(*self.names)

    def count(self, hsh):
        i = np.searchsorted(self.keys, np.uint64(hsh))
        return int(self.pos_off[i + 1] - self.pos_off[i]) if i < len(self.keys) and self.keys[i] == hsh else 0

    def write_fasta(self, d):
        fn = os.path.join(d, "heap_index.fa")
        with open(fn, "wb") as f:
            for n, s in zip(self.names, self.seqs):
                f.write(b">" + n + b"\n" + s + b"\n")
        return fn

    def __del__(self):
        try:
            oracle().wmo_idx_free(self.h)
        except Exception:
            pass


def oracle_heap(ix, mv, qlen, max_occ, flag=0, qname=None):
    """(anchors (n, 2), rep_len, mini_pos) of collect_seed_hits_heap, restated"""
    mv = np.ascontiguousarray(mv, dtype=np.uint64).reshape(-1)
    cap = sum(ix.count(int(x) >> 8) for x in mv[0::2]) + 1
    a = np.zeros(2 * cap, np.uint64)
    mp = np.zeros(len(mv) // 2 + 1, np.uint64)
    rep, nmp = C.c_int32(), C.c_int32()
    n = oracle().wmo_collect_seed_hits_heap(ix.h, flag, max_occ, qname, ix.c_names, _p(ix.seq_len, _u32p), _p(mv, _u64p), len(mv) // 2, qlen,
                                            _p(a, _u64p), cap, C.byref(rep), _p(mp, _u64p), C.byref(nmp))
    assert n <= cap
    return a[: 2 * n].reshape(-1, 2).copy(), rep.value, mp[: nmp.value].copy()


def oracle_sorted(ix, mv, qlen, max_occ):
    """collect_seed_hits without a filter: radix_sort_128x's order (the default path), restated"""
    mv = np.ascontiguousarray(mv, dtype=np.uint64).reshape(-1)
    cap = sum(ix.count(int(x) >> 8) for x in mv[0::2]) + 1
    a = np.zeros(2 * cap, np.uint64)
    mp = np.zeros(len(mv) // 2 + 1, np.uint64)
    rep, nmp = C.c_int32(), C.c_int32()
    n = oracle().wmo_collect_seed_hits(ix.h, max_occ, _p(mv, _u64p), len(mv) // 2, qlen, _p(a, _u64p), cap, C.byref(rep), _p(mp, _u64p), C.byref(nmp))
    return a[: 2 * n].reshape(-1, 2).copy()


class RefIndex:
    def __init__(self, fasta):
        self.h = ref().ref_heap_idx(fasta.encode(), W, K)
        assert self.h

    def hits(self, mv, qlen, max_occ, flag=0, qname=None, heap=True, cap=1 << 20):
        mv = np.ascontiguousarray(mv, dtype=np.uint64).reshape(-1)
        a = np.zeros(2 * cap, np.uint64)
        mp = np.zeros(len(mv) // 2 + 1, np.uint64)
        rep, nmp = C.c_int32(), C.c_int32()
        n = ref().ref_heap_seed_hits(self.h, int(heap), flag, max_occ, qname, _p(mv, _u64p), len(mv) // 2, qlen, _p(a, _u64p), cap,
                                     C.byref(rep), _p(mp, _u64p), C.byref(nmp))
        assert n <= cap
        return a[: 2 * n].reshape(-1, 2).copy(), rep.value, mp[: nmp.value].copy()

    def __del__(self):
        try:
            ref().ref_heap_idx_free(self.h)
        except Exception:
            pass


# ---- crafted match sets ----
def _mv(entries):
    """query minimizers from (hash, q_pos, strand) in position order"""
    out = np.zeros((len(entries), 2), np.uint64)
    for i, (h, qp, st) in enumerate(entries):
        out[i, 0] = (np.uint64(h) << np.uint64(8)) | np.uint64(K)
        out[i, 1] = np.uint64((qp << 1) | st)
    return out


def cases(ix):
    """{name: (mv, qlen, max_occ)}: the match sets of the checks"""
    rng = np.random.default_rng(7)
    cnt = np.diff(ix.pos_off.astype(np.int64))
    multi = ix.keys[cnt >= 8]
    mid = ix.keys[(cnt >= 2) & (cnt < 8)]
    single = ix.keys[cnt == 1]
    out = {}

    def mk(hashes, qlen=None):
        qp = np.sort(rng.choice(np.arange(K, (qlen or 20 * len(hashes) + 100)), size=len(hashes), replace=False))
        return _mv([(int(h), int(p), int(rng.integers(0, 2))) for h, p in zip(hashes, qp)]), int(qlen or 20 * len(hashes) + 100)

    big = multi[np.argmax([ix.count(int(h)) for h in multi])]
    out["one_hash_many_copies"] = (*mk([big] * 40), 5000)
    inter = []
    for i in range(60):
        inter.append(rng.choice(multi[:6]) if i % 3 == 0 else (rng.choice(single) if i % 3 == 1 else rng.choice(mid)))
    out["duplicate_groups_interleaved"] = (*mk(inter), 5000)
    uniq = list(rng.choice(single, 60, replace=False)) + list(rng.choice(mid[:len(mid) // 2], 40, replace=False))
    out["unique_lists"] = (*mk([uniq[i] for i in rng.permutation(len(uniq))]), 5000)
    out["lists_of_length_one"] = (*mk(list(rng.choice(single, 50, replace=False)) + [single[0]] * 5), 5000)
    out["max_occ_cut"] = (*mk(list(rng.choice(multi, 20)) + list(rng.choice(mid, 20)) + [big] * 6), 6)
    absent = np.uint64(int(ix.keys.max()) + 12345)
    out["absent_hashes"] = (*mk([absent, big, absent, big] + list(rng.choice(mid, 10))), 5000)
    for r in range(6):
        s = ix.seqs[r % 4]
        st = int(rng.integers(0, len(s) - 3000))
        q = bytearray(s[st:st + 3000])
        for i in np.nonzero(rng.random(len(q)) < 0.03)[0]:
            q[i] = b"ACGT"[int(rng.integers(0, 4))]
        q = bytes(q) if r % 2 == 0 else _revcomp(bytes(q))
        out[f"read_{r}"] = (ol.oracle_sketch(q, W, K, 0, None), len(q), 5000)
    return out


# flag sets of skip_seed: (name, mapping flag, query name)
FLAG_SETS = [
    ("plain", 0, None),
    ("D_self", F_NO_DIAG, b"qself"),
    ("dual_no", F_NO_DUAL, b"m2"),
    ("X", F_NO_DIAG | F_NO_DUAL, b"m2"),
    ("D_unnamed", F_NO_DIAG, None),
    ("for_only", F_FOR_ONLY, None),
    ("rev_only", F_REV_ONLY, b"a1"),
]


def skip_bits(ix, flag, qname):
    """the device's seed-filter words of a read (host_map.cpp: skip_bits)"""
    b = 0
    if flag & F_FOR_ONLY:
        b |= SKIP_FOR_ONLY
    if flag & F_REV_ONLY:
        b |= SKIP_REV_ONLY
    if qname is None or not flag & (F_NO_DIAG | F_NO_DUAL):
        return b, 0
    if flag & F_NO_DIAG:
        b |= SKIP_NO_DIAG
    if flag & F_NO_DUAL:
        b |= SKIP_NO_DUAL
    if qname in ix.names:
        b |= SKIP_NAME_EQ
    return b, sum(n < qname for n in ix.names)


def self_query(ix):
    """the minimizers of index sequence 0 itself (a read named like it, as long as it): the -D diagonal and MM_SEED_SELF"""
    s = ix.seqs[0]
    return ol.oracle_sketch(s, W, K, 0, None), len(s), 5000


def lookup(ix, mv, max_occ):
    """per query minimizer: cnt (0 when absent or at / above max_occ), list_off, tandem (collect_matches)"""
    h = (mv[:, 0] >> np.uint64(8)).astype(np.uint64)
    i = np.searchsorted(ix.keys, h)
    i = np.minimum(i, len(ix.keys) - 1)
    found = ix.keys[i] == h
    n = np.where(found, (ix.pos_off[i + 1] - ix.pos_off[i]).astype(np.int64), 0)
    cnt = np.where(n >= max_occ, 0, n).astype(np.int32)
    loff = np.where(found, ix.pos_off[i], 0).astype(np.uint64)
    td = np.zeros(len(h), np.uint8)
    if len(h) > 1:
        eq = h[1:] == h[:-1]
        td[1:] |= eq
        td[:-1] |= eq
    return cnt, loff, td


def emul_heap(ix, mv, qlen, max_occ, flag=0, qname=None, stage=True, sorted_a=None):
    """the device's replay on the software warp, over the task's anchors in ascending x"""
    a = np.ascontiguousarray(sorted_a.copy(), dtype=np.uint64)
    cnt, loff, td = lookup(ix, mv, max_occ)
    sb, lt = skip_bits(ix, flag, qname)
    mv = np.ascontiguousarray(mv, dtype=np.uint64)
    r = emul().wmt_heap_replay_dev(_p(mv, _u64p), len(mv), _p(cnt, _i32p), _p(loff, _u64p), _p(td, _u8p), _p(ix.pos, _u64p),
                                   _p(ix.seq_len, _u32p), _p(ix.name_rank, _u32p), qlen, sb, lt, int(sb != 0), int(stage),
                                   _p(a, _u64p), len(a))
    return r, a
