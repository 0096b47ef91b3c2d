#!/usr/bin/env python
"""Generates the end-to-end golden fixtures under tests/golden/ by running the REAL reference
(oracle/_ref/winnowmap = /root/reference + the documented rep_len=0 init, built by oracle/build_ref.sh)
on small deterministic synthetic inputs.  Inputs are regenerated from seeds at test time (tools/gen_data.py);
the manifest stores their md5 so that generator drift is detected.  Run only where /root/reference exists."""
import gzip
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_data  # noqa: E402
import numpy as np  # noqa: E402

CASES = {
    # name: (ref_len, contigs, tandem, ref_seed, n_reads, n50, err, read_seed, min_len, preset, use_W, extra)
    "ont_small": dict(ref_len=300000, contigs=2, tandem=False, ref_seed=1011, n_reads=60, n50=9000, err=0.05, read_seed=2011, min_len=500,
                      preset="map-ont", use_W=False, k=15),
    "ont_tandem": dict(ref_len=400000, contigs=2, tandem=True, ref_seed=1005, n_reads=60, n50=12000, err=0.05, read_seed=2005, min_len=1000,
                       preset="map-ont", use_W=True, k=15),
    # w_distinct: the `distinct=` argument of the meryl rule; 0.99 here so that the list holds the k-mers of the planted array
    "hifi_small": dict(ref_len=300000, contigs=1, tandem=True, ref_seed=1013, n_reads=40, n50=12000, err=0.005, read_seed=2013, min_len=1000,
                       preset="map-pb", use_W=True, k=15, w_distinct=0.99),
    # reads drawn from a donor genome carrying deletions / insertions / inversions: Z-drop splits, long joins, inversion rescue
    "ont_sv": dict(ref_len=400000, contigs=2, tandem=False, ref_seed=1021, n_reads=60, n50=14000, err=0.04, read_seed=2021, min_len=2000,
                   preset="map-ont", use_W=False, k=15, sv=True),
    # a 300-bp family present > 5000 times: minimizers above mid_occ are skipped and rl:i: becomes non-zero
    "ont_highocc": dict(ref_len=2600000, contigs=1, tandem=False, ref_seed=1022, n_reads=40, n50=9000, err=0.05, read_seed=2022, min_len=1500,
                        preset="map-ont", use_W=True, k=15, highocc=True),
    # -O4 -E2: one gap pair (q == q2, e == e2), every DP call is ksw_extz2_sse (src/align.c:328-331)
    # (the structural-variant reads: long gaps are where one gap pair and two differ)
    "ont_single_gap": dict(ref_len=400000, contigs=2, tandem=False, ref_seed=1021, n_reads=60, n50=14000, err=0.04, read_seed=2021, min_len=2000,
                           preset="map-ont", use_W=False, k=15, sv=True, extra=["-O4", "-E2"], gap=(4, 2, 4, 2)),
    "asm20_small": dict(ref_len=300000, contigs=1, tandem=True, ref_seed=1014, n_reads=12, n50=40000, err=0.02, read_seed=2014, min_len=5000,
                        preset="asm20", use_W=True, k=19, w_distinct=0.99),
    # the other assembly presets: asm5 (gap sum 124, e - e2 = 2) and asm10
    "asm5_small": dict(ref_len=300000, contigs=1, tandem=True, ref_seed=1015, n_reads=12, n50=40000, err=0.005, read_seed=2015, min_len=5000,
                       preset="asm5", use_W=True, k=19, w_distinct=0.99),
    "asm10_small": dict(ref_len=300000, contigs=1, tandem=True, ref_seed=1016, n_reads=12, n50=40000, err=0.01, read_seed=2016, min_len=5000,
                        preset="asm10", use_W=True, k=19, w_distinct=0.99),
    # -A2 -B5 -O4,25 -E3,1 on the structural-variant reads: long_thres is raised by one (src/ksw2_extd2_sse.c:95-96), and
    # the long gaps of the SV reads are where the second gap pair decides.  scoring: (a, b, q, e, q2, e2, sc_ambi)
    "ont_sv_long_inc": dict(ref_len=400000, contigs=2, tandem=False, ref_seed=1021, n_reads=60, n50=14000, err=0.04, read_seed=2021, min_len=2000,
                            preset="map-ont", use_W=False, k=15, sv=True, extra=["-A2", "-B5", "-O4,25", "-E3,1"], scoring=(2, 5, 4, 3, 25, 1, 1)),
}


def scoring_override(params):
    """The -A / -B / --score-N / -O / -E of a case as (a, b, sc_ambi, q, e, q2, e2), -1 where the preset's value stays: from
    params["scoring"] (a, b, q, e, q2, e2, sc_ambi) or params["gap"] (q, e, q2, e2)."""
    if params.get("scoring"):
        a, b, q, e, q2, e2, n = params["scoring"]
        return [a, b, n, q, e, q2, e2]
    if params.get("gap"):
        return [-1, -1, -1] + list(params["gap"])
    return [-1] * 7


def apply_scoring(mo, params):
    """The same override on a mapping-options structure (winnowmap_b200.mapper.MapOpt)."""
    for f, v in zip(("a", "b", "sc_ambi", "q", "e", "q2", "e2"), scoring_override(params)):
        if v >= 0:
            setattr(mo, f, v)


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def make_inputs(name, outdir):
    c = CASES[name]
    os.makedirs(outdir, exist_ok=True)
    ref = os.path.join(outdir, name + ".ref.fa")
    reads = os.path.join(outdir, name + ".reads.fa")
    wfile = os.path.join(outdir, name + ".rep.txt")
    rng = np.random.default_rng(c["ref_seed"])
    contigs = gen_data.make_ref(rng, c["ref_len"], c["contigs"], c["tandem"])
    if c.get("highocc"):
        name, seq = contigs[0]
        seq = seq.copy()
        unit = gen_data.random_seq(rng, 300)
        pos = 20000
        for _ in range(6200):  # interspersed copies, 2 % divergence each, ~100 bp apart
            cp = gen_data.mutate(rng, unit, 0.02, (1.0, 0.0, 0.0))
            if pos + 300 >= len(seq) - 20000:
                break
            seq[pos:pos + 300] = cp
            pos += 300 + int(rng.integers(60, 140))
        contigs = [(name, seq)]
    gen_data.write_fasta(ref, contigs)
    rng = np.random.default_rng(c["read_seed"])
    donor = contigs
    if c.get("sv"):
        donor = []
        for name, seq in contigs:
            parts, p = [], 0
            while p < len(seq):
                step = int(rng.integers(6000, 16000))
                seg = seq[p:p + step]
                kind = int(rng.integers(0, 4))
                if kind == 0 and len(seg) > 6000:      # deletion
                    d = int(rng.integers(300, 3000))
                    seg = np.concatenate([seg[:2000], seg[2000 + d:]])
                elif kind == 1:                         # insertion of novel sequence
                    seg = np.concatenate([seg[:2500], gen_data.random_seq(rng, int(rng.integers(300, 2500))), seg[2500:]])
                elif kind == 2 and len(seg) > 6000:    # inversion
                    L = int(rng.integers(800, 3000))
                    seg = np.concatenate([seg[:2000], gen_data.COMP[seg[2000:2000 + L][::-1]], seg[2000 + L:]])
                parts.append(seg)
                p += step
            donor.append((name, np.concatenate(parts)))
    recs = gen_data.make_reads(rng, donor, c["n_reads"], c["n50"], c["err"], min_len=c["min_len"])
    gen_data.write_fasta(reads, recs)
    if c["use_W"]:
        gen_data.write_top_kmers(wfile, contigs, c["k"], c.get("w_distinct", 0.9998))
    else:
        wfile = None
    return ref, reads, wfile


SAM_CASES = ["ont_small", "ont_sv"]
# key -> (case, reference options); flags for the library: MM_F_OUT_CS 0x40, MM_F_OUT_CS_LONG 0x800, MM_F_OUT_MD 0x1000000
TAG_CASES = {
    "paf_cs": ("ont_small", ["-c", "--cs"]),
    "paf_cs_long": ("ont_small", ["-c", "--cs=long"]),
    "sam_md": ("ont_sv", ["-a", "--MD"]),
    "paf_eqx": ("ont_sv", ["-c", "--eqx"]),                      # MM_F_EQX 0x4000000
    "sam_softclip": ("ont_sv", ["-a", "-Y"]),                    # MM_F_SOFTCLIP 0x80000
    "sam_no2nd_hitonly": ("ont_highocc", ["-a", "--secondary=no", "--sam-hit-only"]),  # 0x4000 | 0x40000000
    "paf_no_hit": ("ont_highocc", ["-c", "--paf-no-hit"]),       # MM_F_PAF_NO_HIT 0x8000000
    "sam_fastq_comment": ("ont_small", ["-a", "-y"], "fastq"),   # gzipped FASTQ with comments: QUAL column, MM_F_COPY_COMMENT 0x2000000
    "paf_edge": ("ont_small", ["-c"], "edge"),                   # empty / tiny / N-rich / lower-case / chimeric / unmappable reads
    "sam_edge": ("ont_small", ["-a"], "edge"),
    # the N-rich edge reads under other N scores, with the scoring as params["scoring"] has it: --score-N 0 scores N cells
    # -e2 in the fill (src/ksw2_extd2_sse.c:79) but 0 in the alignment statistics
    "paf_edge_N0": ("ont_small", ["-c", "--score-N", "0"], "edge", (2, 4, 4, 2, 24, 1, 0)),
    "paf_edge_N3": ("ont_small", ["-c", "--score-N", "3"], "edge", (2, 4, 4, 2, 24, 1, 3)),
}


def read_fasta(path):
    recs, name, seq = [], None, []
    for ln in open(path):
        ln = ln.rstrip("\n")
        if ln.startswith(">"):
            if name is not None:
                recs.append((name, "".join(seq)))
            name, seq = ln[1:], []
        else:
            seq.append(ln)
    if name is not None:
        recs.append((name, "".join(seq)))
    return recs


def edge_reads_of(reads_fa, out):
    """Awkward inputs derived from the case's reads: empty, shorter than k, around k, short, lower case, N runs and IUPAC
    codes, an unmappable random read, a chimera of two reads (second half reverse-complemented), a long read with a big
    N block, and two untouched reads for reference."""
    recs = read_fasta(reads_fa)
    rng = np.random.default_rng(77)
    comp = str.maketrans("ACGTacgt", "TGCAtgca")
    a, b, c = recs[0][1], recs[1][1], max(recs, key=lambda r: len(r[1]))[1]
    out_recs = [
        ("e_empty", ""), ("e_len10", a[100:110]), ("e_len14", a[200:214]), ("e_len15", a[300:315]), ("e_len30", a[400:430]),
        ("e_len200", a[500:700]), ("e_len999", b[100:1099]), ("e_lower", b.lower()),
        ("e_nrun", a[:1500] + "N" * 300 + a[1800:]), ("e_iupac", b[:800] + "RYKMSWN" * 20 + b[940:]),
        ("e_random", "".join("ACGT"[i] for i in rng.integers(0, 4, 5000))),
        ("e_chimera", a[:len(a) // 2] + b[:len(b) // 2].translate(comp)[::-1]),
        ("e_bigN", c[:4000] + "N" * 3000 + c[7000:]),
        ("e_plain0", a), ("e_plain1", b),
    ]
    with open(out, "w") as f:
        for nm, sq in out_recs:
            f.write(f">{nm}\n")
            for i in range(0, len(sq), 80):
                f.write(sq[i:i + 80] + "\n")
    return out



def fastq_gz_of(reads_fa, out):
    """The reads as gzipped FASTQ with a comment and a deterministic quality string (input for the QUAL / -y tests)."""
    recs, name, seq = [], None, []
    for ln in open(reads_fa):
        ln = ln.rstrip("\n")
        if ln.startswith(">"):
            if name is not None:
                recs.append((name, "".join(seq)))
            name, seq = ln[1:], []
        else:
            seq.append(ln)
    if name is not None:
        recs.append((name, "".join(seq)))
    with gzip.GzipFile(out, "wb", mtime=0) as f:
        for i, (nm, sq) in enumerate(recs):
            q = "".join(chr(33 + (7 * j + 3 * i) % 41) for j in range(len(sq)))
            f.write(f"@{nm} RG:Z:grp{i % 3}\tXX:i:{i}\n{sq}\n+\n{q}\n".encode())
    return out



def sam_without_pg(sam):
    """The @PG line records the command line (temporary paths): everything else must match byte for byte."""
    return b"".join(ln for ln in sam.splitlines(keepends=True) if not ln.startswith(b"@PG"))


def sam_strip_seq(sam):
    """SEQ and QUAL replaced by their lengths: a small committed fixture to locate a difference; the full text is
    pinned by its md5 in the manifest."""
    out = []
    for ln in sam.splitlines(keepends=True):
        if ln.startswith(b"@"):
            out.append(ln)
            continue
        f = ln.rstrip(b"\n").split(b"\t")
        f[9] = b"len=%d" % len(f[9]) if f[9] != b"*" else b"*"
        f[10] = b"len=%d" % len(f[10]) if f[10] != b"*" else b"*"
        out.append(b"\t".join(f) + b"\n")
    return b"".join(out)


# cases whose index, as the reference itself builds it (mm_idx_reader_read), is stored for tests/test_gpu_boundary.py
REF_INDEX_CASES = ["ont_tandem"]


def pack_seq4(recs):
    """The reference's packed sequence mm_idx_t::S (4 bits per base, 8 bases per word, A/C/G/T = 0..3, anything else 4)
    and the offset of every sequence in it."""
    codes, off, o = [], [], 0
    lut = np.full(256, 4, np.uint32)
    for i, c in enumerate(b"ACGT"):
        lut[c] = lut[c + 32] = i
    for _, sq in recs:
        codes.append(lut[np.frombuffer(sq.encode(), np.uint8)])
        off.append(o)
        o += len(sq)
    c = np.concatenate(codes) if codes else np.zeros(0, np.uint32)
    c = np.concatenate([c, np.zeros(-len(c) % 8, np.uint32)]).reshape(-1, 8)
    return np.bitwise_or.reduce(c << (4 * np.arange(8, dtype=np.uint32)), axis=1).astype(np.uint32), np.array(off, np.uint64)


def save_ref_index(name, gdir, tmp):
    """tests/golden/<name>.refidx.npz: the reference's flattened index of the case (oracle/ref_harness.cpp ref_idx_build_flat).
    S is not stored: the test packs it from the FASTA and checks it against the digest of the reference's S stored here."""
    import ctypes as C
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import oracle_lib as ol
    from winnowmap_b200.mapper import make_options
    R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_harness.so"))
    R.ref_idx_build_flat.restype = C.c_void_p
    R.ref_idx_build_flat.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int]
    for f in ("keys", "pos_off", "pos", "S", "seq_len", "seq_off", "bloom"):
        getattr(R, "ref_idx_flat_" + f).restype = C.c_void_p
        getattr(R, "ref_idx_flat_" + f).argtypes = [C.c_void_p]
    R.ref_idx_flat_sizes.argtypes = [C.c_void_p, C.c_void_p]
    R.ref_idx_flat_free.argtypes = [C.c_void_p]
    ref, _, wfile = make_inputs(name, tmp)
    io, _ = make_options(CASES[name]["preset"], True)
    h = R.ref_idx_build_flat(ref.encode(), wfile.encode() if wfile else None, io.w, io.k, 3)
    sz = np.zeros(7, np.uint64)
    R.ref_idx_flat_sizes(h, sz.ctypes.data)
    n_seq, s_words, n_keys, n_pos, bloom_bits, k, w = (int(x) for x in sz)

    def arr(f, t, n):
        return np.ctypeslib.as_array(C.cast(getattr(R, "ref_idx_flat_" + f)(h), C.POINTER(t)), (n,)).copy()
    pos_off = arr("pos_off", C.c_uint64, n_keys + 1)
    np.savez_compressed(os.path.join(gdir, name + ".refidx.npz"), k=k, w=w, keys=arr("keys", C.c_uint64, n_keys),
                        n_pos=np.diff(pos_off).astype(np.uint32), pos=arr("pos", C.c_uint64, n_pos), bloom=arr("bloom", C.c_uint8, bloom_bits // 8), bloom_bits=bloom_bits,
                        seq_len=arr("seq_len", C.c_uint32, n_seq), seq_off=arr("seq_off", C.c_uint64, n_seq),
                        S_digest=ol.digest(arr("S", C.c_uint32, s_words)))
    R.ref_idx_flat_free(h)


def main():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(gdir, exist_ok=True)
    tmp = "/tmp/wm_golden"
    manifest = {}
    for name, c in CASES.items():
        ref, reads, wfile = make_inputs(name, tmp)
        cmd = [refbin, "-t", "4", "-c", "-x", c["preset"]] + c.get("extra", [])
        if wfile:
            cmd += ["-W", wfile]
        cmd += [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        with gzip.GzipFile(os.path.join(gdir, name + ".paf.gz"), "wb", mtime=0) as f:
            f.write(out)
        manifest[name] = dict(params=c, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile) if wfile else None,
                              cmd=" ".join(["winnowmap"] + cmd[1:]), n_lines=out.count(b"\n"), paf_md5=hashlib.md5(out).hexdigest())
        print(name, manifest[name]["n_lines"], "lines", len(out), "bytes")
    for name in SAM_CASES:  # the same inputs with -a: SAM records (flags, clipping, SEQ/QUAL, SA:Z) and @SQ header
        c = CASES[name]
        ref, reads, wfile = make_inputs(name, tmp)
        cmd = [refbin, "-t", "4", "-a", "-x", c["preset"]]
        if wfile:
            cmd += ["-W", wfile]
        cmd += [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        body = sam_without_pg(out)
        with gzip.GzipFile(os.path.join(gdir, name + ".sam.stripped.gz"), "wb", mtime=0) as f:
            f.write(sam_strip_seq(body))
        manifest[name]["sam_md5"] = hashlib.md5(body).hexdigest()
        manifest[name]["sam_lines"] = body.count(b"\n")
        print(name, "SAM", manifest[name]["sam_lines"], "lines", len(body), "bytes")
    for key, case in TAG_CASES.items():  # output options: --cs, --cs=long, --MD, --eqx, -Y, ...
        name, args = case[0], case[1]
        c = CASES[name]
        ref, reads, wfile = make_inputs(name, tmp)
        if len(case) > 2 and case[2] == "fastq":
            reads = fastq_gz_of(reads, reads + ".fq.gz")
        if len(case) > 2 and case[2] == "edge":
            reads = edge_reads_of(reads, reads + ".edge.fa")
        cmd = [refbin, "-t", "4", "-x", c["preset"]] + args
        if wfile:
            cmd += ["-W", wfile]
        cmd += [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        body = sam_without_pg(out)
        manifest[name].setdefault("tag_md5", {})[key] = hashlib.md5(body).hexdigest()
        if key == "paf_cs":
            with gzip.GzipFile(os.path.join(gdir, name + ".cs.paf.gz"), "wb", mtime=0) as f:
                f.write(body)
        print(name, key, body.count(b"\n"), "lines", len(body), "bytes")
    json.dump(manifest, open(os.path.join(gdir, "manifest.json"), "w"), indent=1, sort_keys=True)
    for name in REF_INDEX_CASES:
        save_ref_index(name, gdir, tmp)


# ---- homopolymer-compressed (-H) goldens: tests/golden/hpc_manifest.json and hpc_*.paf.gz; manifest.json is not touched ----
HPC_CASES = {
    # name: inputs (a case of CASES, or "clr": make_clr_inputs), preset, -a as well
    "hpc_ont_small": dict(inputs="ont_small", preset="map-ont", sam=True),   # two-stage SV-aware path
    "hpc_hifi_small": dict(inputs="hifi_small", preset="map-pb", sam=False),  # -W on compressed k-mers, tandem arrays
    "hpc_clr": dict(inputs="clr", preset="map-pb-clr", sam=False),            # SV-aware off; planted homopolymers up to 400 bp
}
CLR = dict(ref_len=200000, contigs=2, ref_seed=1031, n_reads=50, n50=8000, err=0.10, read_seed=2031, min_len=1000, n_hp=120)


def _hp_errors(rng, seq, err):
    """Errors of an older long-read chemistry: i.i.d. errors at rate err / 2, plus homopolymer-length errors (a run
    grows or shrinks by one or two bases) at about err / 2 per run, plus a few short N runs."""
    s = gen_data.mutate(rng, seq, err / 2)
    out, i, n = [], 0, len(s)
    while i < n:
        j = i + 1
        while j < n and s[j] == s[i]:
            j += 1
        L = j - i
        if rng.random() < err / 2:
            L = max(1, L + int(rng.choice([-2, -1, 1, 2])))
        out.append(np.full(L, s[i], dtype=np.uint8))
        i = j
    r = np.concatenate(out)
    for _ in range(int(rng.integers(0, 3))):
        p, m = int(rng.integers(0, len(r))), int(rng.integers(1, 20))
        r[p:p + m] = ord("N")
    return r


def make_clr_inputs(outdir):
    """A reference with planted homopolymers of 20-400 bp (some >= 256, so that spans >= 256 reach the output) and reads
    with about 10 % errors, homopolymer-length indels and a few N runs."""
    c = CLR
    os.makedirs(outdir, exist_ok=True)
    ref, reads = os.path.join(outdir, "hpc_clr.ref.fa"), os.path.join(outdir, "hpc_clr.reads.fa")
    rng = np.random.default_rng(c["ref_seed"])
    contigs = gen_data.make_ref(rng, c["ref_len"], c["contigs"], False)
    planted = []
    for name, seq in contigs:
        seq = seq.copy()
        for _ in range(c["n_hp"] // len(contigs)):
            L = int(rng.integers(20, 401))
            p = int(rng.integers(1000, len(seq) - 1000 - L))
            seq[p:p + L] = gen_data.ACGT[int(rng.integers(0, 4))]
        planted.append((name, seq))
    gen_data.write_fasta(ref, planted)
    rng = np.random.default_rng(c["read_seed"])
    recs = gen_data.make_reads(rng, planted, c["n_reads"], c["n50"], 0.0, min_len=c["min_len"])
    recs = [(nm, _hp_errors(rng, sq, c["err"])) for nm, sq in recs]
    gen_data.write_fasta(reads, recs)
    return ref, reads, None


def make_hpc_inputs(name, outdir):
    src = HPC_CASES[name]["inputs"]
    return make_clr_inputs(outdir) if src == "clr" else make_inputs(src, outdir)


def main_hpc():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_hpc"
    manifest = {}
    for name, c in HPC_CASES.items():
        ref, reads, wfile = make_hpc_inputs(name, tmp)
        base = ["-t", "4", "-H", "-x", c["preset"]] + (["-W", wfile] if wfile else [])
        cmd = [refbin, "-c"] + base + [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        with gzip.GzipFile(os.path.join(gdir, name + ".paf.gz"), "wb", mtime=0) as f:
            f.write(out)
        m = dict(params=dict(c, clr=CLR if c["inputs"] == "clr" else None), ref_md5=md5(ref), reads_md5=md5(reads),
                 w_md5=md5(wfile) if wfile else None, cmd=" ".join(["winnowmap", "-c"] + base + [ref, reads]),
                 n_lines=out.count(b"\n"), paf_md5=hashlib.md5(out).hexdigest())
        if c["sam"]:
            out = subprocess.run([refbin, "-a"] + base + [ref, reads], stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
            body = sam_without_pg(out)
            with gzip.GzipFile(os.path.join(gdir, name + ".sam.stripped.gz"), "wb", mtime=0) as f:
                f.write(sam_strip_seq(body))
            m["sam_md5"], m["sam_lines"] = hashlib.md5(body).hexdigest(), body.count(b"\n")
        manifest[name] = m
        print(name, m["n_lines"], "lines")
    json.dump(manifest, open(os.path.join(gdir, "hpc_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- self and all-vs-all mapping (-X, -D, --dual=no) and single-strand mapping (--for-only, --rev-only) ----
# tests/golden/overlap_manifest.json and overlap_*.paf.gz; the other manifests are not touched.
# Inputs: "ava" maps a read set against itself (reads of 2-40 kb: both the stage-1 route, reads >= 10 kb, and the
# whole-read route); "asm" maps the reads of hifi_small against themselves; "tandem" is the ont_tandem case.
AVA = dict(ref_len=200000, contigs=1, ref_seed=7, n_reads=80, n50=12000, err=0.05, read_seed=8, min_len=2000)
OVERLAP_CASES = {
    # name: (inputs, reference options, library options of Mapper)
    "overlap_ava_X": ("ava", ["-x", "map-ont", "-X"], dict(preset="map-ont", cigar=False, all_vs_all=True)),
    "overlap_ava_X_c": ("ava", ["-x", "map-ont", "-X", "-c"], dict(preset="map-ont", all_vs_all=True)),
    "overlap_ava_D_c": ("ava", ["-x", "map-ont", "-D", "-c"], dict(preset="map-ont", no_diag=True)),
    "overlap_asm_D_c": ("asm", ["-x", "asm20", "-D", "-c"], dict(preset="asm20", no_diag=True)),
    "overlap_ava_dual_no": ("ava", ["-x", "map-ont", "--dual=no", "-c"], dict(preset="map-ont", dual=False)),
    "overlap_tandem_for_only": ("tandem", ["-x", "map-ont", "--for-only", "-c"], dict(preset="map-ont", strand="for")),
    "overlap_tandem_rev_only": ("tandem", ["-x", "map-ont", "--rev-only", "-c"], dict(preset="map-ont", strand="rev")),
    "overlap_ava_X_H": ("ava", ["-x", "map-ont", "-X", "-H"], dict(preset="map-ont", cigar=False, all_vs_all=True, hpc=True)),
    "overlap_ava_X_sam": ("ava", ["-x", "map-ont", "-X", "-a"], dict(preset="map-ont", sam=True, all_vs_all=True)),
}


def make_overlap_inputs(inputs, outdir):
    """(index FASTA, reads FASTA, -W file or None) of one overlap input set."""
    if inputs == "ava":
        os.makedirs(outdir, exist_ok=True)
        c = AVA
        genome = gen_data.make_ref(np.random.default_rng(c["ref_seed"]), c["ref_len"], c["contigs"], False)
        reads = os.path.join(outdir, "overlap_ava.reads.fa")
        recs = gen_data.make_reads(np.random.default_rng(c["read_seed"]), genome, c["n_reads"], c["n50"], c["err"], min_len=c["min_len"])
        gen_data.write_fasta(reads, recs)
        return reads, reads, None
    if inputs == "asm":  # low-error sequences of 1-40 kb from a genome with tandem arrays, as contigs
        _, reads, _ = make_inputs("hifi_small", outdir)
        return reads, reads, None
    return make_inputs("ont_tandem", outdir)


def main_overlap():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_overlap"
    manifest = {}
    for name, (inputs, args, lib_opts) in OVERLAP_CASES.items():
        ref, reads, wfile = make_overlap_inputs(inputs, tmp)
        cmd = [refbin, "-t", "4"] + args + (["-W", wfile] if wfile else []) + [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        m = dict(inputs=inputs, lib=lib_opts, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile) if wfile else None,
                 cmd=" ".join(["winnowmap"] + cmd[1:]))
        if lib_opts.get("sam"):
            body = sam_without_pg(out)
            with gzip.GzipFile(os.path.join(gdir, name + ".sam.stripped.gz"), "wb", mtime=0) as f:
                f.write(sam_strip_seq(body))
            m["sam_md5"], m["n_lines"] = hashlib.md5(body).hexdigest(), body.count(b"\n")
        else:
            with gzip.GzipFile(os.path.join(gdir, name + ".paf.gz"), "wb", mtime=0) as f:
                f.write(out)
            m["paf_md5"], m["n_lines"] = hashlib.md5(out).hexdigest(), out.count(b"\n")
        manifest[name] = m
        print(name, m["n_lines"], "lines")
    json.dump(manifest, open(os.path.join(gdir, "overlap_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- index parts (-I), --split-prefix and -f: tests/golden/parts_manifest.json and parts_*; the other manifests are not touched ----
# "multi": six contigs of unequal length with tandem arrays and ONT reads, -W from the stand-in list; -I 330k cuts it into
# three parts.  Plan inputs: FASTA files whose part boundaries sit on the rules' edges, mapped with one read so that the
# reference prints its per-part sequence counts.
MULTI = dict(ref_len=900000, ref_seed=1041, n_reads=50, n50=9000, err=0.05, read_seed=2041, min_len=1000, k=15)
PLAN_CASES = {
    # name: (contig lengths or ("random", n, lo, hi, seed), -I)
    "plan_many_small": (("random", 300, 50, 4000, 5), 60000),
    "plan_equal_I": ([1000] * 12, 3000),            # a mini-batch of exactly -I bases does not end the part
    "plan_long_contig": ([500, 20000, 700, 800, 9000, 300], 5000),
    "plan_zero_len": ([3000, 0, 2000, 0, 0, 4000, 0, 1000, 0], 2500),
    "plan_I_above_ref": (("random", 40, 100, 2000, 6), 1000000000),
}
PARTS_CASES = {
    # name: (inputs, reference options, library options of Mapper)
    "parts_ont_c": ("multi", ["-x", "map-ont", "-c", "-I", "330k"], dict(preset="map-ont", part_bases=330000)),
    "parts_ont_c_split": ("multi", ["-x", "map-ont", "-c", "-I", "330k", "--split-prefix", "SPLIT"], dict(preset="map-ont", part_bases=330000, split=True)),
    "parts_ont_a": ("multi", ["-x", "map-ont", "-a", "-I", "330k"], dict(preset="map-ont", sam=True, part_bases=330000)),
    "parts_ont_a_split": ("multi", ["-x", "map-ont", "-a", "-I", "330k", "--split-prefix", "SPLIT"],
                          dict(preset="map-ont", sam=True, part_bases=330000, split=True)),
    "parts_single_split_a": ("multi", ["-x", "map-ont", "-a", "--split-prefix", "SPLIT"], dict(preset="map-ont", sam=True, split=True)),
    "parts_single_split_c": ("multi", ["-x", "map-ont", "-c", "--split-prefix", "SPLIT"], dict(preset="map-ont", split=True)),
    "parts_hpc_c": ("multi", ["-x", "map-ont", "-H", "-c", "-I", "330k"], dict(preset="map-ont", hpc=True, part_bases=330000)),
    "parts_ava_X_split": ("ava", ["-x", "map-ont", "-X", "-I", "120k", "--split-prefix", "SPLIT"],
                          dict(preset="map-ont", cigar=False, all_vs_all=True, part_bases=120000, split=True)),
    "parts_tandem_f0002": ("tandem", ["-x", "map-ont", "-c", "-f", "0.0002"], dict(preset="map-ont", mid_occ_frac=0.0002)),
    "parts_tandem_f01": ("tandem", ["-x", "map-ont", "-c", "-f", "0.01"], dict(preset="map-ont", mid_occ_frac=0.01)),
    "parts_tandem_f0002_I": ("tandem", ["-x", "map-ont", "-c", "-f", "0.0002", "-I", "199999"],
                             dict(preset="map-ont", mid_occ_frac=0.0002, part_bases=199999)),
    "parts_tandem_f01_I_split": ("tandem", ["-x", "map-ont", "-c", "-f", "0.01", "-I", "199999", "--split-prefix", "SPLIT"],
                                 dict(preset="map-ont", mid_occ_frac=0.01, part_bases=199999, split=True)),
}


def make_multi_inputs(outdir):
    """Six contigs of unequal length (tandem arrays in each), ONT-like reads and the stand-in -W list."""
    c = MULTI
    os.makedirs(outdir, exist_ok=True)
    ref, reads, wfile = (os.path.join(outdir, "parts_multi" + x) for x in (".ref.fa", ".reads.fa", ".rep.txt"))
    rng = np.random.default_rng(c["ref_seed"])
    lens = [90000, 210000, 60000, 240000, 120000, 180000]
    contigs = []
    for i, L in enumerate(lens):
        (_, seq), = gen_data.make_ref(rng, L, 1, True)
        contigs.append((f"ctg{i + 1}", seq))
    gen_data.write_fasta(ref, contigs)
    recs = gen_data.make_reads(np.random.default_rng(c["read_seed"]), contigs, c["n_reads"], c["n50"], c["err"], min_len=c["min_len"])
    gen_data.write_fasta(reads, recs)
    gen_data.write_top_kmers(wfile, contigs, c["k"], 0.9998)
    return ref, reads, wfile


def make_parts_inputs(inputs, outdir):
    """(index FASTA, reads FASTA, -W file or None) of one parts input set."""
    if inputs == "multi":
        return make_multi_inputs(outdir)
    if inputs == "ava":
        return make_overlap_inputs("ava", outdir)
    return make_inputs("ont_tandem", outdir)


def make_plan_input(name, outdir):
    """The FASTA of a plan case (sequence names s0, s1, ...; zero-length sequences are empty records)."""
    spec, _ = PLAN_CASES[name]
    if isinstance(spec, tuple):
        _, n, lo, hi, seed = spec
        spec = [int(x) for x in np.random.default_rng(seed).integers(lo, hi + 1, n)]
    rng = np.random.default_rng(len(spec))
    os.makedirs(outdir, exist_ok=True)
    fn = os.path.join(outdir, name + ".fa")
    gen_data.write_fasta(fn, [(f"s{i}", gen_data.random_seq(rng, L)) for i, L in enumerate(spec)])
    return fn


def ref_part_log(err):
    """(per-part sequence counts, per-part mid_occ) from the reference's stderr."""
    import re
    n_seq = [int(x) for x in re.findall(rb"loaded/built the index for (\d+) target sequence", err)]
    mid = [int(x) for x in re.findall(rb"mid-occ:(\d+)", err)]
    return n_seq, mid


def main_parts():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_parts"
    os.makedirs(tmp, exist_ok=True)
    manifest = {"plan": {}, "cases": {}}
    one_read = os.path.join(tmp, "one_read.fa")
    gen_data.write_fasta(one_read, [("r0", gen_data.random_seq(np.random.default_rng(3), 3000))])
    for name, (_, I) in PLAN_CASES.items():
        fa = make_plan_input(name, tmp)
        err = subprocess.run([refbin, "-t", "1", "-x", "map-ont", "-I", str(I), fa, one_read], stdout=subprocess.PIPE,
                             stderr=subprocess.PIPE, check=True).stderr
        n_seq, _ = ref_part_log(err)
        manifest["plan"][name] = dict(I=I, fa_md5=md5(fa), n_seq=n_seq)
        print(name, n_seq)
    for name, (inputs, args, lib_opts) in PARTS_CASES.items():
        ref, reads, wfile = make_parts_inputs(inputs, tmp)
        args = [a if a != "SPLIT" else os.path.join(tmp, name + ".split") for a in args]
        cmd = [refbin, "-t", "4"] + args + (["-W", wfile] if wfile else []) + [ref, reads]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)
        out = p.stdout
        n_seq, mid = ref_part_log(p.stderr)
        m = dict(inputs=inputs, lib=lib_opts, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile) if wfile else None,
                 cmd=" ".join(["winnowmap"] + [a if not a.startswith(tmp) else "<prefix>" for a in cmd[1:-2]] + ["ref.fa", "reads.fa"]),
                 n_seq=n_seq, mid_occ=mid)
        if lib_opts.get("sam"):
            body = sam_without_pg(out)
            with gzip.GzipFile(os.path.join(gdir, name + ".sam.stripped.gz"), "wb", mtime=0) as f:
                f.write(sam_strip_seq(body))
            m["sam_md5"], m["n_lines"] = hashlib.md5(body).hexdigest(), body.count(b"\n")
        else:
            with gzip.GzipFile(os.path.join(gdir, name + ".paf.gz"), "wb", mtime=0) as f:
                f.write(out)
            m["paf_md5"], m["n_lines"] = hashlib.md5(out).hexdigest(), out.count(b"\n")
        manifest["cases"][name] = m
        print(name, m["n_lines"], "lines, parts", n_seq, "mid_occ", mid)
    manifest["occ"] = record_occ(tmp)
    json.dump(manifest, open(os.path.join(gdir, "parts_manifest.json"), "w"), indent=1, sort_keys=True)


# -f values whose mm_idx_cal_max_occ the reference computes on each part of every parts input (the tiny one is refused)
OCC_F = [0.0, 0.0002, 0.001, 0.01, 0.1, 0.5, 0.9]


_ref_parts = []


def ref_parts_lib():
    """oracle/ref_harness_parts.cpp compiled (once per process, into a temporary directory) against the reference built by
    oracle/build_ref.sh; None where the reference's sources ($REF, default /root/reference) or that build are absent."""
    import ctypes as C
    import tempfile
    if not _ref_parts:
        src = os.path.join(os.environ.get("REF", "/root/reference"), "src")
        lib_a = os.path.join(ROOT, "oracle", "_ref", "libwinnowmap.a")
        so = None
        if os.path.isdir(src) and os.path.exists(lib_a):
            so = os.path.join(tempfile.mkdtemp(prefix="wm_ref_parts_"), "libref_harness_parts.so")
            subprocess.check_call(["/usr/bin/g++", "-O2", "-fopenmp", "-std=c++11", "-w", "-fPIC", "-shared", "-DHAVE_KALLOC", "-I" + src,
                                   os.path.join(ROOT, "oracle", "ref_harness_parts.cpp"), lib_a, "-o", so, "-lm", "-lz", "-lpthread"])
        _ref_parts.append(C.CDLL(so) if so else None)
    return _ref_parts[0]


def ref_parts(ref, wfile, k, w, flag, batch_size):
    """The reference's index parts of a FASTA: [(n_seq, occurrence counts as uint32, {f: mm_idx_cal_max_occ})]."""
    import ctypes as C
    R = ref_parts_lib()
    assert R is not None, "the reference's sources and oracle/_ref (oracle/build_ref.sh) are needed"
    R.ref_idx_reader_open.restype = C.c_void_p
    R.ref_idx_reader_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_uint64]
    R.ref_idx_reader_next.restype = C.c_void_p
    R.ref_idx_reader_next.argtypes = [C.c_void_p, C.c_char_p]
    R.ref_idx_reader_close.argtypes = [C.c_void_p]
    R.ref_idx_part_n_seq.argtypes = [C.c_void_p]
    R.ref_idx_part_counts.restype = C.c_int64
    R.ref_idx_part_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    R.ref_idx_cal_max_occ.restype = C.c_int32
    R.ref_idx_cal_max_occ.argtypes = [C.c_void_p, C.c_float]
    R.ref_idx_part_free.argtypes = [C.c_void_p]
    r = R.ref_idx_reader_open(ref.encode(), w, k, flag, batch_size)
    out = []
    while True:
        mi = R.ref_idx_reader_next(r, wfile.encode() if wfile else None)
        if not mi:
            break
        n = R.ref_idx_part_counts(mi, None, 0)
        cnt = np.zeros(n, np.uint32)
        R.ref_idx_part_counts(mi, cnt.ctypes.data, n)
        out.append((R.ref_idx_part_n_seq(mi), cnt, {f: int(R.ref_idx_cal_max_occ(mi, f)) for f in OCC_F}))
        R.ref_idx_part_free(mi)
    R.ref_idx_reader_close(r)
    return out


def record_occ(tmp):
    """Per parts input and -I: each part's count histogram ({count: keys}) and the reference's mm_idx_cal_max_occ."""
    rec = {}
    for inputs, I, flag in (("multi", 330000, 0), ("multi", 330000, 1), ("tandem", 199999, 0), ("tandem", 4000000000, 0), ("ava", 120000, 0)):
        ref, _, wfile = make_parts_inputs(inputs, tmp)
        parts = ref_parts(ref, wfile, 15, 50, flag, I)
        rec[f"{inputs}_I{I}_flag{flag}"] = dict(inputs=inputs, I=I, flag=flag, k=15, w=50, parts=[
            dict(n_seq=n, hist={str(v): int(c) for v, c in zip(*np.unique(cnt, return_counts=True))}, max_occ={str(f): v for f, v in occ.items()})
            for n, cnt, occ in parts])
    return rec


if __name__ == "__main__":
    if "--hpc" in sys.argv:
        main_hpc()
    elif "--overlap" in sys.argv:
        main_overlap()
    elif "--parts" in sys.argv:
        main_parts()
    else:
        main()
