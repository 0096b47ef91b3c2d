"""ctypes bindings for the tee backend (tests/hostsim/tee_backend.cpp): the mapping path's three device calls sent to the
CUDA backend and to the oracle backend at once, compared field by field.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.path.join(ROOT, "tests", "hostsim")
PKG = os.path.join(ROOT, "winnowmap_b200")

# dev_kind of the entry points: which backend serves the caller
DEV_GPU, DEV_ORACLE, DEV_MUTANT = 0, 1, 2
# the changes the mutant backend makes (tee_backend.cpp MUT_*), with where the report must place them
MUTATIONS = {"rep_len": 1, "kept": 2, "u": 3, "b": 4, "cigar": 5, "zd_pos": 6, "ll": 7}
SEED_MASKED, SEED_NO_SKETCH = 1, 2
SEQ_Q0, SEQ_Q1, SEQ_REF = 0, 1, 2


def build(out_dir):
    """The tee library, linked against the product library for all host code (built by build())."""
    so = os.path.join(out_dir, "libwm_tee.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", f"-I{cuda}/include",
                           os.path.join(HOSTSIM, "tee_backend.cpp"), "-x", "c", os.path.join(ROOT, "oracle", "wm_oracle.c"),
                           os.path.join(ROOT, "oracle", "wm_oracle_hpc.c"), "-x", "none", f"-L{PKG}", "-lwinnowmap_b200",
                           f"-Wl,-rpath,{PKG}", "-o", so, "-lz", "-lm", "-lpthread"])
    return so


def load(so):
    L = C.CDLL(so)
    s, i, i64, p = C.c_char_p, C.c_int, C.c_int64, C.c_void_p
    L.wmt_set_gap.argtypes = [i, i, i, i]
    L.wmt_set_scoring.argtypes = [i] * 7
    L.wmt_tee_map_file.argtypes = [s, s, s, s, s, i, i, i64, i, i, s]
    L.wmt_tee_seed_chain.argtypes = [s, s, i, i, i, i, i, i, p, p, i, p, i, p, p, p, i, s]
    L.wmt_tee_align.argtypes = [s, i, i, i, i, i64, i, p, p, i, p, i, p, i, p, p, p, s]
    return L


class Report:
    """What one tee run saw: counters, mismatches (first 200, all counted) and, with the mutant, where it changed a value."""

    def __init__(self, fn):
        self.count, self.mismatches, self.mutated = {}, [], None
        for line in open(fn).read().splitlines():
            f = line.split("\t")
            if f[0] == "count":
                self.count[f[1]] = int(f[2])
            elif f[0] == "mismatch":
                self.mismatches.append(dict(kind=f[1], call=int(f[2]), index=int(f[3]), field=f[4], elem=int(f[5]), expected=f[6], got=f[7], desc=f[8]))
            elif f[0] == "mutated":
                self.mutated = dict(kind=f[1], call=int(f[2]), index=int(f[3]), field=f[4], elem=int(f[5]))

    @property
    def n_mismatch(self):
        return self.count["mismatches"]

    def __getitem__(self, k):
        return self.count.get(k, 0)

    def text(self):
        lines = [f"{k}={v}" for k, v in sorted(self.count.items())]
        lines += ["{kind} call {call} #{index}: {field}[{elem}] expected {expected} got {got} | {desc}".format(**m) for m in self.mismatches[:20]]
        return "\n".join(lines)


def _pool(seqs):
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    return b"".join(seqs), off


def seed_chain(L, report_fn, ref_fn, k, w, reads, rows1, reads2, cp, max_occ, hpc=False, dev=DEV_GPU, mutation=0, kmer_fn=None):
    """A stage-1 seed_chain call over windows (rows1: read, wb, wl, source) and the stage-2 call over the whole reads
    `reads2`, whose stage-1 anchors come from the chains of the source windows (tee_backend.cpp wmt_tee_seed_chain);
    cp: two dicts of ChainParams."""
    seq, off = _pool(reads)
    r1 = np.ascontiguousarray(np.asarray(rows1, dtype=np.int32).reshape(-1, 4))
    r2 = np.ascontiguousarray(np.asarray(reads2, dtype=np.int32).reshape(-1))
    keys = ("max_dist_x", "min_dist_x", "max_dist_y", "bw", "max_skip", "max_iter", "min_cnt", "min_sc")
    ci = np.array([[c[k_] for k_ in keys] for c in cp], dtype=np.int32)
    cf = np.array([c["gap_scale"] for c in cp], dtype=np.float32)
    rc = L.wmt_tee_seed_chain(ref_fn.encode(), kmer_fn.encode() if kmer_fn else None, k, w, int(hpc), dev, mutation, len(reads), seq, off.ctypes.data,
                              len(r1), r1.ctypes.data, len(r2), r2.ctypes.data, ci.ctypes.data, cf.ctypes.data, max_occ, report_fn.encode())
    assert rc == 0, rc
    return Report(report_fn)


def align(L, report_fn, ref_fn, k, w, reads, wins, dp_rows, ll_rows, mat, gaps, budget=0, dev=DEV_GPU, mutation=0):
    """One crafted run_dp batch and one run_ll batch.  dp rows: task, q (kind, rid, off, len, reversed), t (the same), w, zdrop,
    end_bonus, flag; ll rows: the first eleven.  gaps: q, e, q2, e2."""
    seq, off = _pool(reads)
    wr = np.ascontiguousarray(np.asarray(wins, dtype=np.int32).reshape(-1, 3))
    d = np.ascontiguousarray(np.asarray(dp_rows, dtype=np.int64).reshape(-1, 15))
    ll = np.ascontiguousarray(np.asarray(ll_rows, dtype=np.int64).reshape(-1, 11))
    m = np.ascontiguousarray(mat, dtype=np.int8)
    g = np.asarray(gaps, dtype=np.int32)
    rc = L.wmt_tee_align(ref_fn.encode(), k, w, dev, mutation, budget, len(reads), seq, off.ctypes.data, len(wr), wr.ctypes.data,
                         len(d), d.ctypes.data, len(ll), ll.ctypes.data, m.ctypes.data, g.ctypes.data, report_fn.encode())
    assert rc == 0, rc
    return Report(report_fn)


# ---- crafted batches: shapes the orchestrator sends (host_map.cpp, host_align.cpp), at the edges of the device kernels ----
_COMP = bytes.maketrans(b"ACGTacgtNRYKMSWBDHVn", b"TGCAtgcaNYRMKSWVHDBn")


def revcomp(s):
    return s.translate(_COMP)[::-1]


def _rand(rng, n):
    return np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=n)].tobytes()


def _noisy(rng, s, err):
    """A read-like copy: substitutions, insertions and deletions at rate err.  Returns the copy and, for every base of it,
    the index of the source base it stands for."""
    a = np.frombuffer(s, dtype=np.uint8)
    r = rng.random(len(a))
    src = np.flatnonzero(r >= err / 3)
    keep = a[src]
    sub = rng.random(len(keep)) < err / 3
    keep = keep.copy()
    keep[sub] = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=int(sub.sum()))]
    ins = np.flatnonzero(rng.random(len(keep)) < err / 3)
    out = np.insert(keep, ins, np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=len(ins))]).tobytes()
    return out, np.insert(src, ins, src[np.minimum(ins, len(src) - 1)])


CONTIG_LENS = (131800, 40000)
N_RUN = (101500, 101800)  # the run of N in contig 0


def crafted_reference(path, seed=7):
    """Two contigs: unique sequence around two tandem arrays of 40 and 39 copies of different 500-bp units (so that the index
    holds minimizers with occurrence counts c and c - 1 for a c near 40), a run of N, and a second contig that ends in
    unique sequence.  Returns the two contigs."""
    rng = np.random.default_rng(seed)
    ua, ub = _rand(rng, 500), _rand(rng, 500)
    c0 = _rand(rng, 30000) + ua * 40 + _rand(rng, 20000) + ub * 39 + _rand(rng, 12000) + b"N" * 300 + _rand(rng, 30000)
    c1 = _rand(rng, 40000)
    assert c0[N_RUN[0]:N_RUN[1]] == b"N" * (N_RUN[1] - N_RUN[0]) and (len(c0), len(c1)) == CONTIG_LENS
    with open(path, "w") as f:
        for i, c in enumerate((c0, c1)):
            f.write(f">ctg{i}\n")
            for j in range(0, len(c), 80):
                f.write(c[j:j + 80].decode() + "\n")
    return [c0, c1]


class ReadOrigin:
    """Where a crafted read comes from: contig `rid`, bases [start, start + len(src)) copied with noise, on the forward strand
    or reverse-complemented; src[j] is the source base of base j of the (forward) noisy copy."""

    def __init__(self, rid, start, rev, src):
        self.rid, self.start, self.rev, self.src = rid, start, rev, src

    def ref_pos(self, wb, wl, o):
        """The reference position of base o of the window's strand that runs along the reference (strand 0 of a forward
        read, strand 1 of a reverse one)."""
        n = len(self.src)
        j = n - 1 - (wb + wl - 1 - o) if self.rev else wb + o  # base of the forward noisy copy
        return self.start + int(self.src[j])


def crafted_reads_with_origin(contigs, seed=8):
    """Read-like copies of the crafted reference: across both tandem arrays (tens of kb), unique stretches, the reverse
    strand, across the N run, to a contig's end, a short read, and one with N runs, lower case and IUPAC codes."""
    rng = np.random.default_rng(seed)
    reads, origin = [], []

    def copy(rid, st, en, err, rev=False):
        s, src = _noisy(rng, contigs[rid][st:en], err)
        reads.append(revcomp(s) if rev else s)
        origin.append(ReadOrigin(rid, st, rev, src))

    copy(0, 25000, 75000, 0.03)               # 0: both arrays: tens of thousands of anchors
    copy(0, 4000, 9000, 0.05, rev=True)       # 1: reverse strand
    copy(1, 1000, 4000, 0.02)                 # 2
    copy(0, N_RUN[0] - 1500, N_RUN[1] + 1500, 0.04)  # 3: across the N run of the reference
    copy(1, 30000, 40000, 0.03)               # 4: to the contig's end
    copy(1, 10000, 16000, 0.03)               # 5: N runs, lower case, IUPAC codes
    r = bytearray(reads[5])
    for p in range(100, 5000, 700):
        r[p:p + int(rng.integers(1, 40))] = b"N" * 40
    r[2000:2600] = bytes(r[2000:2600]).lower()
    for p in rng.integers(0, len(r), size=30):
        r[int(p)] = b"RYKMSWBDHV"[int(rng.integers(0, 10))]
    reads[5] = bytes(r)
    copy(1, 20000, 20300, 0.01)               # 6: a short read
    return reads, origin


def crafted_reads(contigs, seed=8):
    return crafted_reads_with_origin(contigs, seed)[0]


CHAIN_SETS = [  # stage 1 / fallback against stage 2 (map-ont-like): every field that the two sets of the orchestrator differ in
    dict(max_dist_x=5000, min_dist_x=50, max_dist_y=5000, bw=500, max_skip=3, max_iter=20, min_cnt=3, min_sc=40, gap_scale=1.0),
    dict(max_dist_x=16000, min_dist_x=1000, max_dist_y=16000, bw=2000, max_skip=25, max_iter=5000, min_cnt=2, min_sc=25, gap_scale=1.0),
]


def crafted_seed_tasks(reads, k, w):
    """The stage-1 windows (rows: read, wb, wl, source) and the reads of the stage-2 call.  Stage 1: windows at odd starts
    and at the read end, of lengths around k, w + k - 1, the 128-base chunk, the 1024-base sketch tile and tens of kb.  The
    source windows' chains become stage-1 anchors of their read in stage 2, and their union its masked intervals: on the
    long read, intervals at both read ends and across 32-base groups; on read 1 (reverse strand), two intervals that leave
    one base unmasked; on read 4, windows that cover the read (stage-1 anchors only); on the short read, a stage-1 merge
    of at most 64 anchors.  Reads 2 and 5 have no source window: stage 2 mixes both chain sets."""
    L = [len(r) for r in reads]
    rows = []
    for i, wl in enumerate([k - 1, k, k + 1, w + k - 2, w + k - 1, w + k, 127, 128, 129, 1023, 1024, 1025, 2047, 3001]):
        rd = (2, 5)[i & 1]
        rows.append([rd, 2 * i + 1, wl, 0])             # odd starts
        rows.append([rd, L[rd] - wl, wl, 0])            # ending at the read end
    rows.append([0, 0, L[0], 0])                        # the whole long read: giant chaining tasks
    rows.append([0, 46001, 500, 0])                     # 500 bases of the 39-copy array: 2049 to 4096 anchors
    rows += [[0, 0, 3001, 1], [0, 7003, 1001, 1], [0, L[0] - 2001, 2001, 1]]
    rows += [[1, 0, 2000, 1], [1, 2001, L[1] - 2001, 1]]
    rows += [[3, 101, 999, 1]]
    rows += [[4, 0, 5001, 1], [4, 5001, L[4] - 5001, 1]]
    rows += [[6, 0, 140, 1]]
    return rows, list(range(len(reads)))


def max_occ_with_neighbours(contigs, k, w, hpc=False):
    """An occurrence count c of the crafted reference's index (plain or -H) for which c - 1 is also a count: with
    max_occ = c, minimizers at the boundary (t >= max_occ) and just below it both occur."""
    if hpc:
        import hpc_lib
        mz = np.concatenate([hpc_lib.oracle_sketch_hpc(c, w, k, i) for i, c in enumerate(contigs)])
    else:
        import oracle_lib as ol
        mz = np.concatenate([ol.oracle_sketch(c, w, k, i, None) for i, c in enumerate(contigs)])
    _, cnt = np.unique(mz[:, 0] >> np.uint64(8), return_counts=True)
    have = set(cnt.tolist())
    return max(x for x in have if x - 1 in have and x >= 10)


def crafted_dp_windows(reads):
    """Query windows of the DP batches: the long read, the reverse-strand read (a window that ends at the read end), the read
    that ends at a contig's end, and the read across the N run."""
    L = [len(r) for r in reads]
    return [(0, 0, L[0]), (1, 1, L[1] - 1), (4, 0, L[4]), (3, 3, L[3] - 3)]


EZ_APPROX_MAX, EZ_EXTZ_ONLY, EZ_RIGHT, EZ_REV_CIGAR, EZ_SCAN_ZDROP = 0x08, 0x40, 0x02, 0x80, 0x10000
GAP_FILL, GAP_FILL2, RIGHT_EXT, LEFT_EXT = EZ_APPROX_MAX | EZ_SCAN_ZDROP, 0, EZ_EXTZ_ONLY, EZ_EXTZ_ONLY | EZ_RIGHT | EZ_REV_CIGAR
ALL_KINDS, EXTENSIONS = (GAP_FILL, GAP_FILL2, RIGHT_EXT, LEFT_EXT), (RIGHT_EXT, LEFT_EXT)
# (qlen, tlen, w, kinds) on both sides of the fill kernels' boundaries: tlen 512 / 528 (the per-job state in shared memory or
# in global scratch), qlen 640 / 641, the longest diagonal 383 / 384, and for the cooperative sweep qlen + tlen 1599 / 1600
# and 300 000 band cells (1210 x 390 against 1208 x 392 at w = 383, both with diagonals of 384: a query that runs on past
# the reference slice, which only extensions have)
BOUNDARY_SIZES = [(600, 512, 500, ALL_KINDS), (600, 528, 500, ALL_KINDS), (640, 500, 500, ALL_KINDS), (641, 500, 500, ALL_KINDS),
                  (383, 383, 500, ALL_KINDS), (384, 384, 500, ALL_KINDS), (1000, 1000, 382, ALL_KINDS), (1000, 1000, 383, ALL_KINDS),
                  (800, 799, 500, ALL_KINDS), (800, 800, 500, ALL_KINDS), (1210, 390, 383, EXTENSIONS), (1208, 392, 383, EXTENSIONS),
                  (5, 7, 500, ALL_KINDS), (33, 31, 500, ALL_KINDS), (300, 280, 40, ALL_KINDS)]


def crafted_dp_jobs(origin, wins, rng, sizes=BOUNDARY_SIZES):
    """DP rows as host_align.cpp issues them, over windows `wins` (read, wb, wl) of crafted reads: every slice pair is a true
    alignment (the query slice of the strand that runs along the reference, the reference slice it was copied from), so the
    extensions run to their ends.  Each size of `sizes` as a gap fill (first pass, APPROX_MAX | SCAN_ZDROP, and second pass),
    a right extension and a left extension (both slices reversed, REV_CIGAR), at odd offsets in turn over the windows; a right
    extension to the window's and the contig's end; slices through the reference's N run; one base.  Jobs are shuffled.
    dp_job_reaches_end checks on the oracle that the alignments do run through."""
    rows = []

    def job(task, qoff, qlen, toff, tlen, rev, flag, wband):
        rd, wb, wl = wins[task]
        o = origin[rd]
        rows.append([task, SEQ_Q1 if o.rev else SEQ_Q0, 0, qoff, qlen, rev, SEQ_REF, o.rid, toff, tlen, rev, wband, 400, -1, flag])

    def at(task, qoff, ql, tl, flag, wband):
        rd, wb, wl = wins[task]
        o = origin[rd]
        if flag == LEFT_EXT:  # slices that end at the anchor (qoff + ql, its reference position)
            te = o.ref_pos(wb, wl, qoff + ql)
            job(task, qoff, ql, te - tl, tl, 1, flag, wband)
        else:
            job(task, qoff, ql, o.ref_pos(wb, wl, qoff), tl, 0, flag, wband)

    big = [t for t, (rd, wb, wl) in enumerate(wins) if wl >= 4000]
    i = 0
    for ql, tl, wband, kinds in sizes:
        for flag in kinds:
            task = big[i % len(big)]
            room = wins[task][2] - max(ql, tl) - 40
            at(task, 2 * (i * 211 % (room // 2)) + 1, ql, tl, flag, wband)  # odd offsets
            i += 1
    for task, (rd, wb, wl) in enumerate(wins):
        o = origin[rd]
        if o.rid == 1 and not o.rev and o.start + len(o.src) == CONTIG_LENS[1]:  # the window's end and the contig's end
            q0 = wl - 700
            t0 = o.ref_pos(wb, wl, q0)
            job(task, q0, 700, t0, CONTIG_LENS[1] - t0, 0, RIGHT_EXT, 500)
        if o.rid == 0 and o.start < N_RUN[0] < o.start + len(o.src):  # through the N run of the reference
            q0 = int(np.searchsorted(o.src, N_RUN[0] - o.start)) - 300 - wb
            t0 = o.ref_pos(wb, wl, q0)
            job(task, q0, 900, t0, 900, 0, GAP_FILL, 500)
            job(task, q0, 900, t0, 900, 0, RIGHT_EXT, 500)
            qe = q0 + 900
            job(task, q0, 900, o.ref_pos(wb, wl, qe) - 900, 900, 1, LEFT_EXT, 500)
    job(0, 1, 1, origin[wins[0][0]].ref_pos(wins[0][1], wins[0][2], 1), 1, 0, GAP_FILL, 10)  # one base
    order = rng.permutation(len(rows))  # not sorted by size
    return [rows[i] for i in order]


KSW_NEG_INF = -0x40000000


def dp_job_reaches_end(row, ez, cigar):
    """An extension's fill reached the last row or column of its matrix (ksw_extz_t mqe / mte are set); a gap fill was not
    Z-dropped and has a CIGAR."""
    if row[14] & EZ_EXTZ_ONLY:
        return ez[4] != KSW_NEG_INF or ez[6] != KSW_NEG_INF
    return ez[1] == 0 and len(cigar) > 0


def job_codes(reads, contigs, wins, row):
    """The query and target codes (0..4) of a DP or ll row, as the backends fetch them."""
    def fetch(kind, rid, off, ln, rev, win):
        rd, wb, wl = win
        if kind == SEQ_REF:
            s = contigs[rid][off:off + ln]
        else:
            s = reads[rd][wb:wb + wl]
            s = (revcomp(s) if kind == SEQ_Q1 else s)[off:off + ln]
        c = np.frombuffer(s.upper().translate(_CODE), dtype=np.uint8)
        return c[::-1].copy() if rev else c.copy()
    win = wins[row[0]]
    return fetch(*row[1:6], win), fetch(*row[6:11], win)


_CODE = bytes.maketrans(bytes(range(256)), bytes(4 if chr(i) not in "ACGT" else "ACGT".index(chr(i)) for i in range(256)))


def crafted_ll_jobs(wins, contigs, rng, n=60):
    rows = []
    for i in range(n):
        task = i % len(wins)
        wl = wins[task][2]
        ql = int(rng.integers(1, min(600, wl)))
        qoff = int(rng.integers(0, wl - ql + 1))
        tl = int(rng.integers(1, 600))
        rid = i & 1
        toff = int(rng.integers(0, len(contigs[rid]) - tl))
        rows.append([task, SEQ_Q1 if i & 2 else SEQ_Q0, 0, qoff, ql, 0, SEQ_REF, rid, toff, tl, 0])
    return rows


SCORINGS = {  # (-A, -B, -O q, -E e, -O q2, -E e2, --score-N): every scoring class the mapper accepts, each pinned at every layer
    "map-ont": (2, 4, 4, 2, 24, 1, 1),
    "asm20": (1, 4, 6, 2, 26, 1, 1),
    "single": (2, 4, 4, 2, 4, 2, 1),          # one gap pair: ksw_extz2 (src/align.c:328-331)
    # a mismatch above 2(q + e): ksw_extd2_sse returns before the sweep (src/ksw2_extd2_sse.c:92)
    "early-out": (1, 13, 4, 2, 24, 1, 1),
    "asm10": (1, 9, 16, 2, 41, 1, 1),
    # gap sum 124; e - e2 = 2: long_thres 20, long_diff -3 (every scoring above has e - e2 = 1 and long_diff -2)
    "asm5": (1, 19, 39, 3, 81, 1, 1),
    "long_inc": (2, 5, 4, 3, 25, 1, 1),       # the ++long_thres branch (src/ksw2_extd2_sse.c:95-96): 9 -> 10
    # gap sum exactly 127 (the option check's limit) and a mismatch of exactly 2(q + e): the last scoring that still sweeps
    "limit": (1, 86, 40, 3, 83, 1, 1),
    "single_asm5": (1, 19, 39, 3, 39, 3, 1),  # ksw_extz2 with a large mismatch
    "N0": (2, 4, 4, 2, 24, 1, 0),             # N cells score -e2 in extd2, -e in extz2 (src/ksw2_extd2_sse.c:79)
    "N3": (2, 4, 4, 2, 24, 1, 3),
    "N13": (2, 4, 4, 2, 24, 1, 13),           # the N entries of the matrix, not the mismatch, make the early return
    "match_hi": (20, 4, 4, 2, 24, 1, 1),
}
# -A + q + 2e > 128: the reference's int8 lanes wrap (src/ksw2_extd2_sse.c:52-58), the device fill does not.  The oracle
# follows the reference here; the mapper refuses the scoring (check_opt returns -7).
REFUSED_SCORINGS = {"wrap_probe": (100, 4, 40, 3, 83, 1, 1)}


def write_fasta(path, seqs):
    with open(path, "w") as f:
        for i, s in enumerate(seqs):
            f.write(f">r{i}\n{s.decode()}\n")
