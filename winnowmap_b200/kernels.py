"""numpy-facing wrappers over the kernel-level C-ABI entry points."""
import ctypes as C

import numpy as np

from ._lib import ExtZ, i8p, i32p, i64p, lib, u8p, u32p, u64p

EZ_FIELDS = ("max", "zdropped", "max_q", "max_t", "mqe", "mqe_t", "mte", "mte_q", "score", "reach_end", "n_cigar")


def _p(a, t):
    return a.ctypes.data_as(t)


def _concat(seqs):
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    if len(seqs):
        off[1:] = np.cumsum([len(s) for s in seqs])
    buf = np.concatenate([np.asarray(s, dtype=np.uint8) for s in seqs]) if len(seqs) and off[-1] else np.zeros(0, np.uint8)
    return np.ascontiguousarray(buf), off


def ksw_extd2_batch(queries, targets, mat, q, e, q2, e2, w, zdrop, end_bonus, flag, cigar_cap=None):
    """Batched ksw_extd2 (reference src/ksw2_extd2_sse.c:26).  Returns (ez[n,11] int32, [cigar arrays])."""
    n = len(queries)
    qb, qoff = _concat(queries)
    tb, toff = _concat(targets)
    as32 = lambda v: np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.int32), (n,)))
    w, zdrop, end_bonus, flag = as32(w), as32(zdrop), as32(end_bonus), as32(flag)
    if cigar_cap is None:
        cap = np.array([len(a) + len(b) + 2 for a, b in zip(queries, targets)], dtype=np.int64)
    else:
        cap = np.broadcast_to(np.asarray(cigar_cap, dtype=np.int64), (n,))
    coff = np.zeros(n + 1, dtype=np.int64)
    coff[1:] = np.cumsum(cap)
    ez = (ExtZ * max(n, 1))()
    cig = np.zeros(max(int(coff[-1]), 1), dtype=np.uint32)
    mat = np.ascontiguousarray(mat, dtype=np.int8)
    if len(qb) == 0:
        qb = np.zeros(1, np.uint8)
    if len(tb) == 0:
        tb = np.zeros(1, np.uint8)
    lib().wm_ksw_extd2_batch(n, _p(qb, u8p), _p(qoff, i64p), _p(tb, u8p), _p(toff, i64p), _p(mat, i8p), q, e, q2, e2,
                             _p(w, i32p), _p(zdrop, i32p), _p(end_bonus, i32p), _p(flag, i32p), ez, _p(cig, u32p), _p(coff, i64p))
    out = np.array([[getattr(ez[i], f) for f in EZ_FIELDS] for i in range(n)], dtype=np.int32).reshape(n, len(EZ_FIELDS))
    cigs = [cig[coff[i]: coff[i] + min(out[i, 10], cap[i])].copy() for i in range(n)]
    return out, cigs


def ksw_exts2_batch(queries, targets, mat, q, e, q2, noncan, junc_bonus, zdrop, flag, juncs=None):
    """Batched ksw_exts2 (reference src/ksw2_exts2_sse.c:26), the splice-aware extension.  juncs: per-target annotation bytes
    (arrays as long as the targets) or None.  Returns (ez[n,11] int32, [cigar arrays])."""
    n = len(queries)
    qb, qoff = _concat(queries)
    tb, toff = _concat(targets)
    as32 = lambda v: np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.int32), (n,)))
    zdrop, flag = as32(zdrop), as32(flag)
    cap = np.array([len(a) + len(b) + 2 for a, b in zip(queries, targets)], dtype=np.int64)
    coff = np.zeros(n + 1, dtype=np.int64)
    coff[1:] = np.cumsum(cap)
    ez = (ExtZ * max(n, 1))()
    cig = np.zeros(max(int(coff[-1]), 1), dtype=np.uint32)
    mat = np.ascontiguousarray(mat, dtype=np.int8)
    jb = None
    if juncs is not None:
        jb, _ = _concat([j if j is not None else np.zeros(len(t), np.uint8) for j, t in zip(juncs, targets)])
        if len(jb) == 0:
            jb = np.zeros(1, np.uint8)
    if len(qb) == 0:
        qb = np.zeros(1, np.uint8)
    if len(tb) == 0:
        tb = np.zeros(1, np.uint8)
    L = lib()
    L.wm_ksw_exts2_batch.argtypes = [C.c_int, u8p, i64p, u8p, i64p, u8p, i8p] + [C.c_int] * 5 + [i32p, i32p, C.c_void_p, u32p, i64p]
    L.wm_ksw_exts2_batch(n, _p(qb, u8p), _p(qoff, i64p), _p(tb, u8p), _p(toff, i64p), _p(jb, u8p) if jb is not None else None, _p(mat, i8p),
                         q, e, q2, noncan, junc_bonus, _p(zdrop, i32p), _p(flag, i32p), C.cast(ez, C.c_void_p), _p(cig, u32p), _p(coff, i64p))
    out = np.array([[getattr(ez[i], f) for f in EZ_FIELDS] for i in range(n)], dtype=np.int32).reshape(n, len(EZ_FIELDS))
    cigs = [cig[coff[i]: coff[i] + min(out[i, 10], cap[i])].copy() for i in range(n)]
    return out, cigs


def ksw_ll_batch(queries, targets, mat, gapo, gape):
    """Batched ksw_ll_qinit + ksw_ll_i16 (reference src/ksw2_ll_sse.c:32,80).  Returns (n,3) int32: score, query end, target end."""
    n = len(queries)
    qb, qoff = _concat(queries)
    tb, toff = _concat(targets)
    if len(qb) == 0:
        qb = np.zeros(1, np.uint8)
    if len(tb) == 0:
        tb = np.zeros(1, np.uint8)
    mat = np.ascontiguousarray(mat, dtype=np.int8)
    sc, qe, te = (np.zeros(max(n, 1), np.int32) for _ in range(3))
    L = lib()
    L.wm_ksw_ll_batch.argtypes = [C.c_int, u8p, i64p, u8p, i64p, i8p, C.c_int, C.c_int, i32p, i32p, i32p]
    L.wm_ksw_ll_batch(n, _p(qb, u8p), _p(qoff, i64p), _p(tb, u8p), _p(toff, i64p), _p(mat, i8p), gapo, gape, _p(sc, i32p), _p(qe, i32p), _p(te, i32p))
    return np.stack([sc, qe, te], axis=1)[:n]


_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


class Bloom:
    """Down-weighted k-mer filter (reference: bloom_filter built at src/index.c:404-432)."""

    def __init__(self, canon_kmers):
        k = np.ascontiguousarray(canon_kmers, dtype=np.uint64)
        self._k = k
        self.h = lib().wm_bloom_build(_p(k, u64p) if len(k) else None, len(k))

    def bits(self):
        return lib().wm_bloom_bits(self.h)

    def table(self):
        n = self.bits() // 8
        return np.ctypeslib.as_array(C.cast(lib().wm_bloom_table(self.h), u8p), shape=(n,)).copy()

    def __del__(self):
        try:
            lib().wm_bloom_destroy(self.h)
        except Exception:
            pass


def sketch_batch(bloom, seqs, w, k, rids=None, hpc=False):
    """Batched mm_sketch (reference src/sketch.c:128).  seqs: list of bytes.  Returns list of (n,2) uint64.
    hpc=True sketches homopolymer-compressed k-mers (is_hpc = 1)."""
    n = len(seqs)
    off = np.zeros(n + 1, dtype=np.int64)
    if n:
        off[1:] = np.cumsum([len(s) for s in seqs])
    buf = b"".join(seqs) + b"\0"
    rid = np.ascontiguousarray(rids if rids is not None else np.zeros(n), dtype=np.uint32)
    out, out_off = C.c_void_p(), C.c_void_p()
    fn = lib().wm_sketch_batch_hpc if hpc else lib().wm_sketch_batch
    rc = fn(bloom.h, n, buf, _p(off, i64p), _p(rid, u32p), w, k, C.byref(out), C.byref(out_off))
    if rc != 0:
        raise ValueError("wm_sketch_batch failed")
    o = np.ctypeslib.as_array(C.cast(out_off, i64p), shape=(n + 1,)).copy()
    tot = int(o[-1])
    xy = np.ctypeslib.as_array(C.cast(out, u64p), shape=(max(tot, 1) * 2,)).copy()[: tot * 2].reshape(-1, 2)
    _libc.free(out)
    _libc.free(out_off)
    return [xy[o[i]: o[i + 1]].copy() for i in range(n)]


def sdust_batch(seqs, T, W=64):
    """Batched sdust_core (reference src/sdust.c:134), the regions -T masks.  seqs: list of bytes.  Returns a list of (n,2)
    int64 arrays of [start, end) per sequence."""
    n = len(seqs)
    off = np.zeros(n + 1, dtype=np.int64)
    if n:
        off[1:] = np.cumsum([len(s) for s in seqs])
    buf = b"".join(seqs) + b"\0"
    reg, reg_off = C.c_void_p(), C.c_void_p()
    L = lib()
    L.wm_sdust_batch.argtypes = [C.c_int, C.c_char_p, i64p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    if L.wm_sdust_batch(n, buf, _p(off, i64p), T, W, C.byref(reg), C.byref(reg_off)) != 0:
        raise ValueError(f"wm_sdust_batch failed (T = {T}, W = {W})")
    o = np.ctypeslib.as_array(C.cast(reg_off, i64p), shape=(n + 1,)).copy()
    tot = int(o[-1])
    r = np.ctypeslib.as_array(C.cast(reg, u64p), shape=(max(tot, 1),)).copy()[:tot]
    _libc.free(reg)
    _libc.free(reg_off)
    se = np.stack([(r >> np.uint64(32)).astype(np.int64), (r & np.uint64(0xffffffff)).astype(np.int64)], axis=1)
    return [se[o[i]: o[i + 1]].copy() for i in range(n)]


def seed_batch(keys, pos_off, pos, tasks, max_occ, heap=False, seq_len=None, name_rank=None, skip=None):
    """The seed stage alone on the device (wm_seed_batch): mm_idx_get, collect_matches, skip_seed and radix_sort_128x, or with
    heap=True the order of collect_seed_hits_heap (reference src/map.c:97-254).  The index: keys (sorted unique hashes), pos_off
    (CSR offsets, len(keys) + 1) and pos (occurrences, each list ascending); seq_len / name_rank per index sequence (for the
    filter).  tasks: list of (mz_xy (n, 2) uint64, qlen).  skip: None, or per task (WM seed-filter bits, names below the read's).
    Returns per task (anchors (n, 2) uint64, rep_len, n_mini_pos, mini_pos uint32 per minimizer: position | kept << 31)."""
    L = lib()
    L.wm_seed_batch.argtypes = [C.c_int64, u64p, u64p, u64p, C.c_int, u32p, u32p, C.c_int, u64p, i64p, i32p, u32p, C.c_int, C.c_int,
                                C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), i32p, i32p, u32p]
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    pos_off = np.ascontiguousarray(pos_off, dtype=np.uint64)
    pos = np.ascontiguousarray(pos, dtype=np.uint64)
    if len(pos) == 0:
        pos = np.zeros(1, np.uint64)
    n_seq = 0 if seq_len is None else len(seq_len)
    seq_len = np.ascontiguousarray(seq_len if seq_len is not None else [0], dtype=np.uint32)
    name_rank = np.ascontiguousarray(name_rank if name_rank is not None else [0], dtype=np.uint32)
    n = len(tasks)
    mz_off = np.zeros(n + 1, dtype=np.int64)
    mz_off[1:] = np.cumsum([len(t[0]) for t in tasks])
    mz = np.ascontiguousarray(np.concatenate([np.asarray(t[0], dtype=np.uint64).reshape(-1, 2) for t in tasks] + [np.zeros((1, 2), np.uint64)]))
    qlen = np.ascontiguousarray([t[1] for t in tasks] + [0], dtype=np.int32)
    sk = None if skip is None else np.ascontiguousarray(np.asarray(skip, dtype=np.uint32).reshape(-1, 2))
    rep, nmp = np.zeros(n + 1, np.int32), np.zeros(n + 1, np.int32)
    mpos = np.zeros(int(mz_off[-1]) + 1, np.uint32)
    a, a_off = C.c_void_p(), C.c_void_p()
    if L.wm_seed_batch(len(keys), _p(keys, u64p), _p(pos_off, u64p), _p(pos, u64p), n_seq, _p(seq_len, u32p), _p(name_rank, u32p), n,
                       _p(mz, u64p), _p(mz_off, i64p), _p(qlen, i32p), None if sk is None else _p(sk, u32p), int(max_occ), int(bool(heap)),
                       C.byref(a), C.byref(a_off), _p(rep, i32p), _p(nmp, i32p), _p(mpos, u32p)) != 0:
        raise ValueError("wm_seed_batch failed")
    o = np.ctypeslib.as_array(C.cast(a_off, i64p), shape=(n + 1,)).copy()
    tot = int(o[-1])
    xy = np.ctypeslib.as_array(C.cast(a, u64p), shape=(max(tot, 1) * 2,)).copy()[: tot * 2].reshape(-1, 2)
    _libc.free(a)
    _libc.free(a_off)
    return [(xy[o[i]: o[i + 1]].copy(), int(rep[i]), int(nmp[i]), mpos[mz_off[i]: mz_off[i + 1]].copy()) for i in range(n)]


HEAP_STAT_NAMES = ("tasks", "anchors", "clocks", "global_heaps", "mismatches")


def seed_heap_stats(reset=False):
    """Counters of the heap merge on the current device (wm_seed_heap_stats), as a dict of HEAP_STAT_NAMES."""
    L = lib()
    L.wm_seed_heap_stats.restype = None
    L.wm_seed_heap_stats.argtypes = [C.POINTER(C.c_double), C.c_int]
    v = (C.c_double * 5)()
    L.wm_seed_heap_stats(v, int(bool(reset)))
    return dict(zip(HEAP_STAT_NAMES, [int(x) for x in v]))


class Intv1(C.Structure):
    """mm_idx_intv1_t (reference src/index.c): st, en, max, then score:30 and strand:2 in one int32."""
    _fields_ = [("st", C.c_int32), ("en", C.c_int32), ("max", C.c_int32), ("score", C.c_int32, 30), ("strand", C.c_int32, 2)]


class Intv(C.Structure):
    _fields_ = [("n", C.c_int32), ("m", C.c_int32), ("a", C.POINTER(Intv1))]


def intv_records(per_seq):
    """(array of Intv, keep-alive) from per-sequence lists of (st, en, strand[, score]) tuples, each sorted by st here."""
    keep, I = [], (Intv * max(1, len(per_seq)))()
    for r, ivs in enumerate(per_seq):
        ivs = sorted(ivs, key=lambda x: x[0])
        a = (Intv1 * max(1, len(ivs)))()
        for j, v in enumerate(ivs):
            a[j].st, a[j].en, a[j].max, a[j].strand = int(v[0]), int(v[1]), -1, int(v[2])
            a[j].score = int(v[3]) if len(v) > 3 else 0
        keep.append(a)
        I[r].n, I[r].m, I[r].a = len(ivs), len(ivs), C.cast(a, C.POINTER(Intv1))
    return I, keep


def bed_junc_batch(per_seq, windows):
    """Batched mm_idx_bed_junc (reference src/index.c:780) on the device.  per_seq: for each sequence, a list of (st, en,
    strand) intervals (strand 1, -1 or 0); windows: (rid, off, len, reversed) tuples.  Returns one uint8 array per window."""
    I, keep = intv_records(per_seq)
    n = len(windows)
    win = np.array(windows, dtype=np.int32).reshape(n, 4) if n else np.zeros((0, 4), np.int32)
    out_off = np.zeros(n + 1, dtype=np.int64)
    if n:
        out_off[1:] = np.cumsum(win[:, 2])
    out = np.zeros(int(out_off[-1]) + 1, dtype=np.uint8)
    L = lib()
    L.wm_bed_junc_batch.argtypes = [C.POINTER(Intv), C.c_int, C.c_int, i32p, u8p, i64p]
    if L.wm_bed_junc_batch(I, len(per_seq), n, _p(np.ascontiguousarray(win), i32p), _p(out, u8p), _p(out_off, i64p)) != 0:
        raise ValueError("wm_bed_junc_batch failed")
    del keep
    return [out[out_off[i]: out_off[i + 1]].copy() for i in range(n)]


def radix_sort_128x_batch(arrays):
    """radix_sort_128x (reference src/misc.c:156) on each (n,2) uint64 array, tie order included."""
    n = len(arrays)
    off = np.zeros(n + 1, dtype=np.int64)
    if n:
        off[1:] = np.cumsum([len(a) for a in arrays])
    flat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in arrays] + [np.zeros((1, 2), np.uint64)]))
    lib().wm_radix_sort_128x_batch(n, _p(flat, u64p), _p(off, i64p))
    return [flat[off[i]: off[i + 1]].copy() for i in range(n)]


def chain_dp_batch(arrays, max_dist_x, min_dist_x, max_dist_y, bw, max_skip=25, max_iter=5000, min_cnt=3, min_sc=40, gap_scale=1.0,
                   is_cdna=False):
    """Batched mm_chain_dp (reference src/chain.c:22).  is_cdna=True is the gap cost of spliced mapping (src/chain.c:69-77).
    Returns list of (u, b)."""
    n = len(arrays)
    off = np.zeros(n + 1, dtype=np.int64)
    if n:
        off[1:] = np.cumsum([len(a) for a in arrays])
    flat = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.uint64).reshape(-1, 2) for a in arrays] + [np.zeros((1, 2), np.uint64)]))
    tot = int(off[-1])
    n_u = np.zeros(max(n, 1), dtype=np.int32)
    n_b = np.zeros(max(n, 1), dtype=np.int64)
    u = np.zeros(max(tot, 1), dtype=np.uint64)
    b = np.zeros((max(tot, 1), 2), dtype=np.uint64)
    if is_cdna:
        lib().wm_chain_dp_batch_cdna(n, _p(flat, u64p), _p(off, i64p), max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt,
                                     min_sc, C.c_float(gap_scale), 1, _p(n_u, i32p), _p(u, u64p), _p(b, u64p), _p(n_b, i64p))
    else:
        lib().wm_chain_dp_batch(n, _p(flat, u64p), _p(off, i64p), max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc,
                                C.c_float(gap_scale), _p(n_u, i32p), _p(u, u64p), _p(b, u64p), _p(n_b, i64p))
    return [(u[off[i]: off[i] + n_u[i]].copy(), b[off[i]: off[i] + n_b[i]].copy()) for i in range(n)]
