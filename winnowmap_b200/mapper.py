"""Python face of the drop-in boundary: index construction and file/batch mapping through the C ABI."""
import ctypes as C
import os

from ._lib import lib


class IdxOpt(C.Structure):  # wm_idxopt_t == mm_idxopt_t (reference src/minimap.h:106-110)
    _fields_ = [("k", C.c_short), ("w", C.c_short), ("flag", C.c_short), ("bucket_bits", C.c_short),
                ("mini_batch_size", C.c_int), ("batch_size", C.c_uint64)]


class MapOpt(C.Structure):  # wm_mapopt_t == mm_mapopt_t (reference src/minimap.h:112-176)
    _fields_ = [("flag", C.c_int64), ("seed", C.c_int), ("sdust_thres", C.c_int), ("max_qlen", C.c_int), ("bw", C.c_int),
                ("max_gap", C.c_int), ("max_gap_ref", C.c_int), ("min_gap_ref", C.c_int), ("max_frag_len", C.c_int),
                ("max_chain_skip", C.c_int), ("max_chain_iter", C.c_int), ("min_cnt", C.c_int), ("min_chain_score", C.c_int),
                ("chain_gap_scale", C.c_float), ("SVaware", C.c_bool), ("SVawareMinReadLength", C.c_int), ("suffixSampleOffset", C.c_int),
                ("min_mapq", C.c_int), ("min_qcov", C.c_float), ("minPrefixLength", C.c_int), ("maxPrefixLength", C.c_int),
                ("prefixIncrementFactor", C.c_float), ("stage2_bw", C.c_int), ("stage2_zdrop_inv", C.c_int), ("stage2_max_gap", C.c_int),
                ("stage2_extension_inc", C.c_int), ("mask_level", C.c_float), ("mask_len", C.c_int), ("pri_ratio", C.c_float),
                ("best_n", C.c_int), ("max_join_long", C.c_int), ("max_join_short", C.c_int), ("min_join_flank_sc", C.c_int),
                ("min_join_flank_ratio", C.c_float), ("alt_drop", C.c_float), ("a", C.c_int), ("b", C.c_int), ("q", C.c_int),
                ("e", C.c_int), ("q2", C.c_int), ("e2", C.c_int), ("sc_ambi", C.c_int), ("noncan", C.c_int), ("junc_bonus", C.c_int),
                ("zdrop", C.c_int), ("zdrop_inv", C.c_int), ("end_bonus", C.c_int), ("min_dp_max", C.c_int), ("min_ksw_len", C.c_int),
                ("anchor_ext_len", C.c_int), ("anchor_ext_shift", C.c_int), ("max_clip_ratio", C.c_float), ("pe_ori", C.c_int),
                ("pe_bonus", C.c_int), ("mid_occ_frac", C.c_float), ("min_mid_occ", C.c_int32), ("mid_occ", C.c_int32),
                ("max_occ", C.c_int32), ("mini_batch_size", C.c_int), ("max_sw_mat", C.c_int64), ("kmer_freq_filename", C.c_char_p),
                ("split_prefix", C.c_char_p)]


F_CIGAR, F_OUT_SAM, F_OUT_CG, F_NO_PRINT_2ND, F_PAF_NO_HIT = 0x004, 0x008, 0x020, 0x4000, 0x8000000
F_NO_DIAG, F_NO_DUAL, F_NO_LJOIN, F_FOR_ONLY, F_REV_ONLY, F_ALL_CHAINS = 0x001, 0x002, 0x400, 0x100000, 0x200000, 0x800000
F_SPLICE, F_SPLICE_FOR, F_SPLICE_REV, F_SPLICE_FLANK = 0x080, 0x100, 0x200, 0x40000
F_HEAP_SORT = 0x400000  # MM_F_HEAP_SORT (reference src/minimap.h)
I_HPC = 0x1  # MM_I_HPC (reference src/minimap.h:41)
SDUST_MAX_T = 1 << 20  # the largest -T the library takes (csrc/sdust.cuh)

STAT_NAMES = ("n_reads", "n_bases", "n_minimaps", "n_chained", "n_dp_jobs", "n_ll_jobs", "n_rounds", "t_seed", "t_dp", "t_host",
              "t_index", "t_map", "n_keys", "n_pos", "n_topfreq", "topfreq_threshold", "t_topfreq")


def _setup(L):
    if getattr(L, "_wm_mapper_ready", False):
        return L
    L.wm_set_opt.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.POINTER(MapOpt)]
    L.wm_idx_bed_read.argtypes = [C.c_void_p, C.c_char_p]
    L.wm_idx_set_junc.argtypes = [C.c_void_p, C.c_void_p]
    L.wm_junc_stats.restype = None
    L.wm_junc_stats.argtypes = [C.POINTER(C.c_double), C.c_int]
    L.wm_check_opt.argtypes = [C.POINTER(IdxOpt), C.POINTER(MapOpt)]
    L.wm_mapopt_max_intron_len.restype = None
    L.wm_mapopt_max_intron_len.argtypes = [C.POINTER(MapOpt), C.c_int]
    L.wm_index_build.restype = C.c_void_p
    L.wm_index_build.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
    L.wm_index_build_opt.restype = C.c_void_p
    L.wm_index_build_opt.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(IdxOpt), C.c_int]
    L.wm_index_build_topfreq.restype = C.c_void_p
    L.wm_index_build_topfreq.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.c_double, C.c_int]
    L.wm_topfreq.restype = C.c_int64
    L.wm_topfreq.argtypes = [C.c_char_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_uint64), C.c_int]
    L.wm_topfreq_threshold.restype = C.c_uint64
    L.wm_topfreq_threshold.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_double]
    L.wm_index_build_parts.restype = C.c_void_p
    L.wm_index_build_parts.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(IdxOpt), C.c_double, C.c_int]
    L.wm_idx_n_parts.argtypes = [C.c_void_p]
    L.wm_idx_part.restype = C.c_void_p
    L.wm_idx_part.argtypes = [C.c_void_p, C.c_int]
    L.wm_part_plan.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_void_p, C.c_int]
    L.wm_idx_cal_max_occ.restype = C.c_int32
    L.wm_idx_cal_max_occ.argtypes = [C.c_void_p, C.c_float]
    L.wm_mapopt_update.argtypes = [C.POINTER(MapOpt), C.c_void_p]
    L.wm_idx_flag.argtypes = [C.c_void_p]
    L.wm_gpu_destroy.argtypes = [C.c_void_p]
    L.wm_idx_blob_size.restype = C.c_int64
    L.wm_idx_blob_size.argtypes = [C.c_void_p]
    L.wm_idx_blob_write.argtypes = [C.c_void_p, C.c_void_p]
    L.wm_idx_blob_load.restype = C.c_void_p
    L.wm_idx_blob_load.argtypes = [C.c_void_p, C.c_int64, C.c_int]
    L.wm_map_file.argtypes = [C.c_void_p, C.POINTER(MapOpt), C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]
    L.wm_get_stats.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int]
    L.wm_reset_stats.argtypes = [C.c_void_p]
    assert L.wm_sizeof_mapopt() == C.sizeof(MapOpt), (L.wm_sizeof_mapopt(), C.sizeof(MapOpt))
    L._wm_mapper_ready = True
    return L


F_OUT_SAM = 0x008


E_SPLICE_CIGAR = -8  # wm_check_opt: MM_F_SPLICE together with MM_F_CIGAR


def _check(L, io, mo, spliced_alignment):
    rc = L.wm_check_opt(C.byref(io), C.byref(mo))
    if rc == E_SPLICE_CIGAR and spliced_alignment:
        return
    if rc < 0:
        raise ValueError(f"mm_check_opt-style validation failed: {rc}")


def make_options(preset=None, cigar=True, sam=False, no_diag=False, dual=True, all_vs_all=False, strand=None, splice=False,
                 max_intron_len=None, spliced_alignment=False, heap_sort=False):
    """mm_set_opt(0) then mm_set_opt(preset) (reference main.c:144-159); -c sets MM_F_OUT_CG|MM_F_CIGAR, -a sets
    MM_F_OUT_SAM|MM_F_CIGAR (main.c).  Self and all-vs-all mapping: no_diag is -D, dual=False is --dual=no, all_vs_all
    is -X (-D -P --no-long-join --dual=no); strand="for" / "rev" is --for-only / --rev-only.  Spliced mapping: the presets
    "splice", "splice:hq" and "cdna" (any "splice:..." is "splice"), splice=True is --splice (cDNA chaining on any preset),
    max_intron_len=N is -G, applied after the preset and --splice; it changes nothing unless one of them set MM_F_SPLICE.
    Spliced base-level alignment (-c / -a with spliced mapping: the two-strand ksw_exts2 rounds, ts:A, N in the CIGAR) is a
    library path that has to be asked for: spliced_alignment=True accepts cigar / sam with spliced mapping, and the -8 that
    wm_check_opt returns for that combination.  Without it, spliced mapping needs cigar=False and sam=False, as the command
    line does until its refusal is lifted.  heap_sort=True is --heap-sort=yes: anchors are collected in the order of the
    reference's heap merge of the occurrence lists (collect_seed_hits_heap), which differs from the default only among anchors
    with equal reference positions; the command line still refuses it, the library applies it."""
    L = _setup(lib())
    io, mo = IdxOpt(), MapOpt()
    L.wm_set_opt(None, C.byref(io), C.byref(mo))
    if preset is not None and L.wm_set_opt(preset.encode(), C.byref(io), C.byref(mo)) != 0:
        raise ValueError(f"unknown preset {preset}")
    if splice:
        mo.flag |= F_SPLICE
    if max_intron_len is not None:
        L.wm_mapopt_max_intron_len(C.byref(mo), int(max_intron_len))
    if (mo.flag & F_SPLICE) and (sam or cigar) and not spliced_alignment:
        raise ValueError("spliced base-level alignment (-c / -a with a splice preset or --splice) is a library path: "
                         "ask for it with spliced_alignment=True, or map with cigar=False and sam=False for approximate PAF")
    if sam:
        mo.flag |= F_OUT_SAM | F_CIGAR
    elif cigar:
        mo.flag |= F_OUT_CG | F_CIGAR
    if no_diag:
        mo.flag |= F_NO_DIAG
    if not dual:
        mo.flag |= F_NO_DUAL
    if all_vs_all:
        mo.flag |= F_ALL_CHAINS | F_NO_DIAG | F_NO_DUAL | F_NO_LJOIN
    if strand is not None:
        if strand not in ("for", "rev", "both"):
            raise ValueError(f"strand must be 'for', 'rev' or 'both', not {strand!r}")
        mo.flag |= {"for": F_FOR_ONLY, "rev": F_REV_ONLY, "both": 0}[strand]
    if heap_sort:
        mo.flag |= F_HEAP_SORT
    _check(L, io, mo, spliced_alignment)
    return io, mo


class Mapper:
    """winnowmap [-W rep.txt] -x preset [-H] -c ref.fa reads.fa  on one GPU.  hpc=True is -H: the index and the reads are
    sketched with homopolymer-compressed k-mers (reference src/main.c:166).  A blob carries its own flag.  no_diag, dual,
    all_vs_all and strand are the self / all-vs-all and single-strand options of make_options (-D, --dual, -X,
    --for-only / --rev-only): Mapper(reads, preset="map-ont", all_vs_all=True).map_file(reads, out) computes overlaps.
    distinct=D takes the -W list from the reference itself instead of the file kmer_freq: the k-mers that
    `meryl count k=K` + `meryl print greater-than distinct=D` list (top_kmers), counted on the GPU; 0.9998 is the
    reference README's recipe.
    part_bases is -I: the reference is cut into index parts of about that many bases (wm_index_build_parts), which stay on the
    GPU together; the output is then part-major, or, with split=True (--split-prefix), the parts' hits are merged per read
    in memory (no temporary file is written).  mid_occ_frac is -f: each index part gets its own mid_occ, selected on the
    GPU from its occurrence counts.
    preset="splice" / "splice:hq" / "cdna" with cigar=False maps spliced reads (approximate PAF, cDNA chaining); splice=True is
    --splice and max_intron_len is -G (make_options).  With spliced_alignment=True they also align at base level (-c, or -a
    with sam=True): ksw_exts2 on the GPU, both transcript strands tried per hit, ts:A, introns as N; the other flags of the
    reference (--eqx, --cs, --MD, -u, --splice-flank, -C, --cap-sw-mem) are the fields of self.mo.
    sdust_thres=T is -T: minimizers that lie mostly in low-complexity regions (SDUST with threshold T, window 64) are dropped
    before seeding, in every stage; 0 (the default) is off.  The command line still refuses -T; the library applies it.
    junc_bed is --junc-bed: a BED file (plain or gzip) of known introns (BED12 blocks, or one interval per line), read into every
    index part after the index is built.  With spliced_alignment=True every splice DP then adds junc_bonus (self.mo.junc_bonus;
    9 under splice / cdna, 5 under splice:hq) at annotated donors and acceptors; other mapping is unchanged, as in the reference.
    heap_sort=True is --heap-sort=yes (make_options): every stage collects its anchors in the order of the reference's heap merge."""

    def __init__(self, ref, kmer_freq=None, preset="map-ont", cigar=True, device=0, n_threads=None, blob=None, sam=False, hpc=False,
                 no_diag=False, dual=True, all_vs_all=False, strand=None, distinct=None, part_bases=None, split=False, mid_occ_frac=None,
                 splice=False, max_intron_len=None, spliced_alignment=False, sdust_thres=0, junc_bed=None, heap_sort=False):
        if kmer_freq is not None and distinct is not None:
            raise ValueError("give either a -W file (kmer_freq) or distinct=, not both")
        if distinct is not None and not 0.0 < distinct <= 1.0:
            raise ValueError(f"distinct must be in (0, 1], not {distinct!r}")
        if part_bases is not None and (blob is not None or int(part_bases) <= 0):
            raise ValueError("part_bases must be a positive number of bases and cannot be combined with blob=")
        if mid_occ_frac is not None and not 0.0 <= mid_occ_frac < 1.0:
            raise ValueError(f"mid_occ_frac must be in [0, 1), not {mid_occ_frac!r}")
        if not 0 <= int(sdust_thres) <= SDUST_MAX_T:
            raise ValueError(f"sdust_thres must be in 0..{SDUST_MAX_T}, not {sdust_thres!r}")
        self.L = _setup(lib())
        self.io, self.mo = make_options(preset, cigar, sam, no_diag=no_diag, dual=dual, all_vs_all=all_vs_all, strand=strand,
                                        splice=splice, max_intron_len=max_intron_len, spliced_alignment=spliced_alignment,
                                        heap_sort=heap_sort)
        if hpc:
            self.io.flag |= I_HPC
        if mid_occ_frac is not None:
            self.mo.mid_occ_frac = mid_occ_frac
        self.mo.sdust_thres = int(sdust_thres)
        if split:
            self.mo.split_prefix = b"split"  # any prefix: the merge runs in memory and writes no file
            _check(self.L, self.io, self.mo, spliced_alignment)
        self.n_threads = n_threads or max(1, min(64, (os.cpu_count() or 2) // 2))
        if blob is not None:  # index received from another rank (numpy uint8 array)
            self._blob_keep = blob
            self.ctx = self.L.wm_idx_blob_load(blob.ctypes.data, blob.nbytes, device)
        elif part_bases is not None:
            self.io.batch_size = int(part_bases)
            self.ctx = self.L.wm_index_build_parts(ref.encode(), kmer_freq.encode() if kmer_freq else None, C.byref(self.io),
                                                   float(distinct or 0.0), device)
        elif distinct is not None:
            self.ctx = self.L.wm_index_build_topfreq(ref.encode(), C.byref(self.io), float(distinct), device)
        else:
            self.ctx = self.L.wm_index_build_opt(ref.encode(), kmer_freq.encode() if kmer_freq else None, C.byref(self.io), device)
        if not self.ctx:
            raise RuntimeError("index construction failed")
        if junc_bed is not None and self.L.wm_idx_bed_read(self.ctx, os.fsencode(junc_bed)) != 0:
            self.close()
            raise RuntimeError(f"cannot read the BED file {junc_bed!r}")

    @property
    def hpc(self):
        """True when the index holds homopolymer-compressed minimizers (MM_I_HPC)."""
        return bool(self.L.wm_idx_flag(self.ctx) & I_HPC)

    @property
    def n_parts(self):
        """The number of index parts (1 unless part_bases cut the reference)."""
        return self.L.wm_idx_n_parts(self.ctx)

    def index_blob(self):
        """The flattened index as one numpy uint8 array (for the one-time NCCL fan-out)."""
        import numpy as np
        if self.n_parts > 1:
            raise RuntimeError("the blob fan-out of a multi-part index is not supported")
        n = self.L.wm_idx_blob_size(self.ctx)
        buf = np.empty(n, dtype=np.uint8)
        self.L.wm_idx_blob_write(self.ctx, buf.ctypes.data)
        return buf

    def map_file(self, reads, out, rank=0, world=1, tag_order=False, max_batch_bases=200_000_000):
        rc = self.L.wm_map_file(self.ctx, C.byref(self.mo), reads.encode(), out.encode(), self.n_threads, rank, world, int(tag_order), max_batch_bases)
        if rc != 0:
            raise RuntimeError("wm_map_file failed")

    def stats(self):
        v = (C.c_double * len(STAT_NAMES))()
        self.L.wm_get_stats(self.ctx, v, len(STAT_NAMES))
        return dict(zip(STAT_NAMES, list(v)))

    def reset_stats(self):
        self.L.wm_reset_stats(self.ctx)

    def close(self):
        if self.ctx:
            self.L.wm_gpu_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def part_plan(ref, part_bases, mini_batch_size=50_000_000):
    """The number of sequences in each index part that part_bases (-I) gives, on the host: the plan wm_index_build_parts
    follows and the reference's index reader cuts (no GPU needed)."""
    L = _setup(lib())
    cap = 1
    while True:
        buf = (C.c_int32 * cap)()
        n = L.wm_part_plan(ref.encode(), int(part_bases), int(mini_batch_size), buf, cap)
        if n < 0:
            raise RuntimeError(f"cannot read {ref}")
        if n <= cap:
            return list(buf[:n])
        cap = n


def top_kmers(ref, k, distinct=0.9998, device=0):
    """(kmers, counts, threshold) of `meryl count k=K ref` + `meryl print greater-than distinct=D`, counted on the GPU:
    canonical k-mer codes (encodeKmer's, reference src/index.c:362-376) ascending as uint64, their counts as uint32, and the
    count they are all above."""
    import numpy as np
    L = _setup(lib())
    if not 1 <= k <= 28 or not 0.0 < distinct <= 1.0:
        raise ValueError(f"k = {k} must be in 1..28 and distinct = {distinct} in (0, 1]")
    thr = C.c_uint64(0)
    n = L.wm_topfreq(ref.encode(), k, float(distinct), None, None, 0, C.byref(thr), device)
    if n < 0:
        raise RuntimeError("wm_topfreq failed")
    kmers, counts = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint32)
    if n:
        m = L.wm_topfreq(ref.encode(), k, float(distinct), kmers.ctypes.data, counts.ctypes.data, n, C.byref(thr), device)
        assert m == n, (m, n)
    return kmers, counts, int(thr.value)


def write_top_kmers(ref, out, k, distinct=0.9998, device=0):
    """The -W file of top_kmers: one `KMER<TAB>COUNT` line per k-mer, spelled from its code (the format the reference reads,
    src/index.c:390-432).  Returns (number of k-mers, threshold)."""
    kmers, counts, thr = top_kmers(ref, k, distinct, device)
    shifts = [2 * (k - 1 - i) for i in range(k)]
    with open(out, "w") as f:
        for v, c in zip(kmers.tolist(), counts.tolist()):
            f.write("".join("ACGT"[(v >> s) & 3] for s in shifts) + f"\t{c}\n")
    return len(kmers), thr
