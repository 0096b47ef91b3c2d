#!/usr/bin/env python
"""Generates the end-to-end golden fixtures under tests/golden/ by running the REAL reference
(oracle/_ref/winnowmap = /root/reference + the documented rep_len=0 init, built by oracle/build_ref.sh)
on small deterministic synthetic inputs.  Inputs are regenerated from seeds at test time (tools/gen_data.py);
the manifest stores their md5 so that generator drift is detected.  Run only where /root/reference exists."""
import gzip
import hashlib
import json
import os
import shutil
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


# ---- spliced mapping without base alignment (-x splice / splice:hq / cdna, --splice, -G): tests/golden/splice_manifest.json and
# splice_*; the other manifests are not touched.  Inputs: a transcriptome of gen_data.make_transcriptome (genes on both strands,
# GT-AG / CT-AC introns from 60 bp to over 200 kb, isoforms, paralogs) and cDNA-like reads of it: "tx" ONT-like, "tx_hq" low
# error, "tx_long" only transcripts of 10 kb or more (--splice on map-ont: stage 1 runs, with cDNA chaining).
SPLICE = dict(genome_len=1600000, n_genes=40, ref_seed=1051, read_seed=2051, n_reads=160, n_genomic=16, n_random=4, k=15)
SPLICE_READS = {"tx": dict(err=0.06, long=False), "tx_hq": dict(err=0.01, long=False), "tx_long": dict(err=0.05, long=True)}
SPLICE_CASES = {
    # name: (reads, reference options, -W, library options of Mapper)
    "splice_W": ("tx", ["-x", "splice"], True, dict(preset="splice", cigar=False)),
    "splice_noW": ("tx", ["-x", "splice"], False, dict(preset="splice", cigar=False)),
    "splice_hq": ("tx_hq", ["-x", "splice:hq"], True, dict(preset="splice:hq", cigar=False)),
    "splice_G20k": ("tx", ["-x", "splice", "-G", "20000"], True, dict(preset="splice", cigar=False, max_intron_len=20000)),
    "splice_ont_long": ("tx_long", ["-x", "map-ont", "--splice"], True, dict(preset="map-ont", cigar=False, splice=True)),
    "splice_H": ("tx", ["-x", "splice", "-H"], True, dict(preset="splice", cigar=False, hpc=True)),
    "splice_I_split": ("tx", ["-x", "splice", "-I", "500k", "--split-prefix", "SPLIT"], True,
                       dict(preset="splice", cigar=False, part_bases=500000, split=True)),
}


def make_splice_inputs(reads_kind, outdir):
    """(genome FASTA, reads FASTA, -W file) of one spliced read set."""
    c, r = SPLICE, SPLICE_READS[reads_kind]
    os.makedirs(outdir, exist_ok=True)
    ref, reads, wfile = (os.path.join(outdir, "splice" + x) for x in (".ref.fa", "_" + reads_kind + ".reads.fa", ".rep.txt"))
    contigs, tx = gen_data.make_transcriptome(np.random.default_rng(c["ref_seed"]), c["genome_len"], c["n_genes"])
    gen_data.write_fasta(ref, contigs)
    if r["long"]:
        tx = [t for t in tx if len(t[1]) >= 10000]
    rng = np.random.default_rng(c["read_seed"] + len(reads_kind))
    n = c["n_reads"] // 4 if r["long"] else c["n_reads"]
    recs = gen_data.make_spliced_reads(rng, contigs, tx, n, r["err"], 0 if r["long"] else c["n_genomic"], 0 if r["long"] else c["n_random"])
    gen_data.write_fasta(reads, recs)
    gen_data.write_top_kmers(wfile, contigs, c["k"], 0.9998)
    return ref, reads, wfile


def main_splice():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_splice"
    manifest = {}
    for name, (reads_kind, args, use_w, lib_opts) in SPLICE_CASES.items():
        ref, reads, wfile = make_splice_inputs(reads_kind, tmp)
        args = [a if a != "SPLIT" else os.path.join(tmp, name + ".split") for a in args]
        cmd = [refbin, "-t", "4"] + args + (["-W", wfile] if use_w else []) + [ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        with gzip.GzipFile(os.path.join(gdir, name + ".paf.gz"), "wb", mtime=0) as f:
            f.write(out)
        manifest[name] = dict(reads=reads_kind, use_W=use_w, lib=lib_opts, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile) if use_w else None,
                              cmd=" ".join(["winnowmap"] + [a if not a.startswith(tmp) else "<prefix>" for a in cmd[1:-2]] + ["ref.fa", "reads.fa"]),
                              paf_md5=hashlib.md5(out).hexdigest(), n_lines=out.count(b"\n"))
        print(name, manifest[name]["n_lines"], "lines")
    json.dump(manifest, open(os.path.join(gdir, "splice_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- spliced base-level alignment (-c / -a with -x splice / splice:hq / cdna or --splice): tests/golden/splice_aln_manifest.json
# and splice_aln_*; the inputs of the splice_* cases.  The "tx" reads include unspliced genomic reads, whose two strand rounds tie
# (trans_strand 3: no ts:A).  Library options: the MM_F_* bits the reference's options set / clear beyond -c / -a, -C, --cap-sw-mem.
F_OUT_CS, F_OUT_MD, F_EQX, F_SOFTCLIP = 0x40, 0x1000000, 0x4000000, 0x80000
F_SPLICE_FOR, F_SPLICE_REV, F_SPLICE_FLANK = 0x100, 0x200, 0x40000
SPLICE_ALN_CASES = {
    # name: (reads, reference options, library options)
    "splice_aln_c": ("tx", ["-x", "splice", "-c"], dict(preset="splice")),
    "splice_aln_a": ("tx", ["-x", "splice", "-a"], dict(preset="splice", sam=True)),
    "splice_aln_hq_cs": ("tx_hq", ["-x", "splice:hq", "-c", "--cs"], dict(preset="splice:hq", set_flags=F_OUT_CS)),
    "splice_aln_cdna_md": ("tx", ["-x", "cdna", "-a", "--MD"], dict(preset="cdna", sam=True, set_flags=F_OUT_MD)),
    "splice_aln_eqx_Y": ("tx", ["-x", "splice", "-a", "--eqx", "-Y"], dict(preset="splice", sam=True, set_flags=F_EQX | F_SOFTCLIP)),
    "splice_aln_uf": ("tx", ["-x", "splice", "-c", "-u", "f"], dict(preset="splice", set_flags=F_SPLICE_FOR, clear_flags=F_SPLICE_REV)),
    "splice_aln_ur": ("tx", ["-x", "splice", "-c", "-u", "r"], dict(preset="splice", set_flags=F_SPLICE_REV, clear_flags=F_SPLICE_FOR)),
    "splice_aln_un": ("tx", ["-x", "splice", "-c", "-u", "n"], dict(preset="splice", clear_flags=F_SPLICE_FOR | F_SPLICE_REV)),
    "splice_aln_noflank": ("tx", ["-x", "splice", "-c", "--splice-flank=no"], dict(preset="splice", clear_flags=F_SPLICE_FLANK)),
    "splice_aln_C3": ("tx", ["-x", "splice", "-c", "-C", "3"], dict(preset="splice", noncan=3)),
    "splice_aln_H": ("tx", ["-x", "splice", "-c", "-H"], dict(preset="splice", hpc=True)),
    "splice_aln_I_split": ("tx", ["-x", "splice", "-c", "-I", "500k", "--split-prefix", "SPLIT"],
                           dict(preset="splice", part_bases=500000, split=True)),
    "splice_aln_ont_long": ("tx_long", ["-x", "map-ont", "--splice", "-c"], dict(preset="map-ont", splice=True)),
    "splice_aln_cap5M": ("tx", ["-x", "splice", "-c", "--cap-sw-mem", "5M"], dict(preset="splice", max_sw_mat=5000000)),
    "splice_aln_G20k": ("tx", ["-x", "splice", "-c", "-G", "20000"], dict(preset="splice", max_intron_len=20000)),
}


def main_splice_aln():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_splice"
    manifest = {}
    for name, (reads_kind, args, lib_opts) in SPLICE_ALN_CASES.items():
        ref, reads, wfile = make_splice_inputs(reads_kind, tmp)
        args = [a if a != "SPLIT" else os.path.join(tmp, name + ".split") for a in args]
        cmd = [refbin, "-t", "4"] + args + ["-W", wfile, ref, reads]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        sam = "-a" in args
        if sam:
            out = sam_without_pg(out)
        with gzip.GzipFile(os.path.join(gdir, name + (".sam.stripped.gz" if sam else ".paf.gz")), "wb", mtime=0) as f:
            f.write(sam_strip_seq(out) if sam else out)
        manifest[name] = dict(reads=reads_kind, lib=lib_opts, sam=sam, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile),
                              # not "cmd": the command-line parse check replays every "cmd" of the manifests, and the
                              # command line refuses spliced alignment
                              ref_cmd=" ".join(["winnowmap"] + [a if not a.startswith(tmp) else "<prefix>" for a in cmd[1:-2]] + ["ref.fa", "reads.fa"]),
                              out_md5=hashlib.md5(out).hexdigest(), n_lines=out.count(b"\n"))
        print(name, manifest[name]["n_lines"], "lines")
    json.dump(manifest, open(os.path.join(gdir, "splice_aln_manifest.json"), "w"), indent=1, sort_keys=True)


# The command line (winnowmap_b200/winnowmap-b200, tests/test_cli_host.py, tests/test_gpu_cli.py): reference runs on inputs
# written under fixed relative names (ref.fa, reads.fa, reads_a.fa + reads_b.fa: the reads split in two files, rep.txt), run
# from their directory so that the @PG CL: of the SAM header is stable.  {W} stands for "-W rep.txt" where the input has a list.
CLI_CASES = {
    "cli_sv_cap50M": dict(inputs="ont_sv", args="-t 4 -c -x map-ont --cap-sw-mem 50M {W} ref.fa reads.fa"),
    "cli_sv_cap5M": dict(inputs="ont_sv", args="-t 4 -c -x map-ont --cap-sw-mem 5M {W} ref.fa reads.fa"),
    "cli_sv_maxqlen": dict(inputs="ont_sv", args="-t 4 -c -x map-ont --max-qlen 8000 {W} ref.fa reads.fa"),
    "cli_small_rg": dict(inputs="ont_small", args="-t 4 -a -x map-ont -R @RG\\tID:rg1\\tSM:s1 {W} ref.fa reads.fa"),
    "cli_two_files_paf": dict(inputs="ont_small", args="-t 4 -c -x map-ont {W} ref.fa reads_a.fa reads_b.fa"),
    "cli_two_files_sam": dict(inputs="ont_small", args="-t 4 -a -x map-ont {W} ref.fa reads_a.fa reads_b.fa"),
    "cli_parts_two_files": dict(inputs="ont_tandem", args="-t 4 -c -x map-ont -I 330k {W} ref.fa reads_a.fa reads_b.fa"),
}


def make_cli_inputs(inputs, outdir):
    """The files of a command-line case under their fixed names in outdir."""
    os.makedirs(outdir, exist_ok=True)
    tmp = os.path.join(outdir, "gen")
    ref, reads, wfile = make_inputs(inputs, tmp)
    shutil.copy(ref, os.path.join(outdir, "ref.fa"))
    shutil.copy(reads, os.path.join(outdir, "reads.fa"))
    recs = read_fasta(reads)
    for half, part in (("a", recs[: len(recs) // 2]), ("b", recs[len(recs) // 2:])):
        with open(os.path.join(outdir, f"reads_{half}.fa"), "w") as f:
            for nm, sq in part:
                f.write(f">{nm}\n{sq}\n")
    if wfile:
        shutil.copy(wfile, os.path.join(outdir, "rep.txt"))
    return wfile is not None


def cli_args(name, has_w):
    """argv[1..] of a case (no argument holds a space)"""
    return CLI_CASES[name]["args"].replace("{W}", "-W rep.txt" if has_w else "").split()


def cli_golden_bytes(out, sam):
    """What is committed of a run's output: PAF as it is, SAM with SEQ and QUAL replaced by their lengths."""
    return sam_strip_seq(out) if sam else out


def main_cli():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    gdir = os.path.join(ROOT, "tests", "golden")
    manifest = {}
    for name in CLI_CASES:
        td = os.path.join("/tmp/wm_golden_cli", name)
        has_w = make_cli_inputs(CLI_CASES[name]["inputs"], td)
        args = cli_args(name, has_w)
        out = subprocess.run([refbin] + args, cwd=td, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout
        sam = "-a" in args
        with gzip.GzipFile(os.path.join(gdir, name + (".sam.stripped.gz" if sam else ".paf.gz")), "wb", mtime=0) as f:
            f.write(cli_golden_bytes(out, sam))
        manifest[name] = dict(CLI_CASES[name], sam=sam, cmd=" ".join(["winnowmap"] + args), ref_md5=md5(os.path.join(td, "ref.fa")),
                              reads_md5=md5(os.path.join(td, "reads.fa")), n_lines=out.count(b"\n"), out_md5=hashlib.md5(out).hexdigest())
        print(name, manifest[name]["n_lines"], "lines")
    json.dump(manifest, open(os.path.join(gdir, "cli_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- SDUST (-T): tests/golden/sdust_manifest.json and sdust_*; the other manifests are not touched ----
# Inputs with microsatellites and tandem arrays: "tandem" is the ont_tandem case (mapped, or overlapped with itself for -X),
# "tx" the spliced read set of the splice_* cases.  Every case must differ from the same command without -T.
SDUST_CASES = {
    # name: (inputs, reference options, library options of Mapper)
    "sdust_tandem_T10": ("tandem", ["-x", "map-ont", "-c", "-T", "10"], dict(preset="map-ont", sdust_thres=10)),
    "sdust_tandem_T20": ("tandem", ["-x", "map-ont", "-c", "-T", "20"], dict(preset="map-ont", sdust_thres=20)),
    "sdust_tandem_a": ("tandem", ["-x", "map-ont", "-a", "-T", "20"], dict(preset="map-ont", sam=True, sdust_thres=20)),
    "sdust_tandem_H": ("tandem", ["-x", "map-ont", "-H", "-c", "-T", "10"], dict(preset="map-ont", hpc=True, sdust_thres=10)),
    "sdust_tandem_I_split": ("tandem", ["-x", "map-ont", "-c", "-I", "199999", "--split-prefix", "SPLIT", "-T", "20"],
                             dict(preset="map-ont", part_bases=199999, split=True, sdust_thres=20)),
    "sdust_tandem_X": ("tandem_ava", ["-x", "map-ont", "-X", "-T", "20"], dict(preset="map-ont", cigar=False, all_vs_all=True, sdust_thres=20)),
    "sdust_splice": ("tx", ["-x", "splice", "-T", "20"], dict(preset="splice", cigar=False, sdust_thres=20)),
    "sdust_tx_ont_c": ("tx", ["-x", "map-ont", "-c", "-T", "20"], dict(preset="map-ont", sdust_thres=20)),
}


def make_sdust_inputs(inputs, outdir):
    """(index FASTA, reads FASTA, -W file or None) of one SDUST input set."""
    if inputs == "tx":
        return make_splice_inputs("tx", outdir)
    ref, reads, wfile = make_inputs("ont_tandem", outdir)
    return (reads, reads, None) if inputs == "tandem_ava" else (ref, reads, wfile)


def main_sdust():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_sdust"
    manifest = {}
    for name, (inputs, args, lib_opts) in SDUST_CASES.items():
        ref, reads, wfile = make_sdust_inputs(inputs, tmp)
        outs = []
        for a in (args, args[:args.index("-T")] + args[args.index("-T") + 2:]):
            a = [x if x != "SPLIT" else os.path.join(tmp, name + ".split") for x in a]
            cmd = [refbin, "-t", "4"] + a + (["-W", wfile] if wfile else []) + [ref, reads]
            outs.append(subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout)
        sam = "-a" in args
        out, out0 = (sam_without_pg(o) if sam else o for o in outs)
        assert out != out0, f"{name}: -T changes nothing"
        with gzip.GzipFile(os.path.join(gdir, name + (".sam.stripped.gz" if sam else ".paf.gz")), "wb", mtime=0) as f:
            f.write(sam_strip_seq(out) if sam else out)
        manifest[name] = dict(inputs=inputs, lib=lib_opts, sam=sam, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile) if wfile else None,
                              # not "cmd": the command-line parse check replays every "cmd" of the manifests, and the command line
                              # refuses -T
                              ref_cmd=" ".join(["winnowmap"] + [x if x != "SPLIT" else "<prefix>" for x in args] +
                                               (["-W", "rep.txt"] if wfile else []) + ["ref.fa", "reads.fa"]),
                              out_md5=hashlib.md5(out).hexdigest(), n_lines=out.count(b"\n"),
                              n_lines_differing=len(set(out.split(b"\n")) ^ set(out0.split(b"\n"))))
        print(name, manifest[name]["n_lines"], "lines,", manifest[name]["n_lines_differing"], "differ from the run without -T")
    json.dump(manifest, open(os.path.join(gdir, "sdust_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- heap sort (--heap-sort=yes): tests/golden/heap_manifest.json and heap_*; the other manifests are not touched ----
# Short-unit tandem data: a random reference with 40 tandem arrays of 5-40 copies of 15-120 bp units at 2 % divergence, and 300
# reads of 2-20 kb at 5 % error from it, half reverse-complemented ("tandem"; "tandem_ava": the first 60 reads against themselves).
# Copies of one query hash share an occurrence list, so their anchors tie in x and the heap's order differs from the sort's.
HEAP_CASES = {
    # name: (inputs, reference options, library options of Mapper)
    "heap_tandem_c": ("tandem", ["-x", "map-ont", "-c"], dict(preset="map-ont")),
    "heap_tandem_pb": ("tandem", ["-x", "map-pb", "-c"], dict(preset="map-pb")),
    "heap_tandem_a": ("tandem", ["-x", "map-ont", "-a"], dict(preset="map-ont", sam=True)),
    "heap_tandem_H": ("tandem", ["-x", "map-ont", "-H", "-c"], dict(preset="map-ont", hpc=True)),
    "heap_tandem_I_split": ("tandem", ["-x", "map-ont", "-c", "-I", "150000", "--split-prefix", "SPLIT"],
                            dict(preset="map-ont", part_bases=150000, split=True)),
    "heap_tandem_X": ("tandem_ava", ["-x", "map-ont", "-X", "-c"], dict(preset="map-ont", all_vs_all=True)),
    "heap_splice": ("tx", ["-x", "splice"], dict(preset="splice", cigar=False)),
}


def make_heap_inputs(inputs, outdir):
    """(index FASTA, reads FASTA) of one heap-sort input set."""
    if inputs == "tx":
        ref, reads, _ = make_splice_inputs("tx", outdir)
        return ref, reads
    os.makedirs(outdir, exist_ok=True)
    ref, reads = os.path.join(outdir, "heap_tandem.ref.fa"), os.path.join(outdir, "heap_tandem.reads.fa")
    rng = np.random.default_rng(11)
    A = np.frombuffer(b"ACGT", dtype=np.uint8)

    def rs(n):
        return A[rng.integers(0, 4, n)]

    def mutate(s, e):
        r = rng.random(len(s))
        sub = A[rng.integers(0, 4, len(s))]
        ins = A[rng.integers(0, 4, len(s))]
        out = []
        for c, x, b1, b2 in zip(s.tolist(), r.tolist(), sub.tolist(), ins.tolist()):
            if x < e * 0.6:
                out.append(b1)
            elif x < e * 0.8:
                continue
            elif x < e:
                out += (c, b2)
            else:
                out.append(c)
        return np.array(out, dtype=np.uint8)

    parts = [rs(50000)]
    for _ in range(40):
        u = rs(int(rng.integers(15, 120)))
        parts += [mutate(u, 0.02) for _ in range(int(rng.integers(5, 40)))] + [rs(int(rng.integers(2000, 8000)))]
    g = np.concatenate(parts)
    with open(ref, "w") as f:
        f.write(">c1\n" + g.tobytes().decode() + "\n")
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    ava = os.path.join(outdir, "heap_tandem_ava.reads.fa")
    with open(reads, "w") as f, open(ava, "w") as fa:
        for i in range(300):
            L = int(rng.integers(2000, 20000))
            p = int(rng.integers(0, len(g) - L))
            r = mutate(g[p:p + L], 0.05).tobytes()
            if rng.random() < 0.5:
                r = r.translate(comp)[::-1]
            f.write(f">r{i}\n{r.decode()}\n")
            if i < 60:
                fa.write(f">r{i}\n{r.decode()}\n")
    return (ava, ava) if inputs == "tandem_ava" else (ref, reads)


def main_heap():
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if not os.path.exists(refbin):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_heap"
    manifest = {}
    for name, (inputs, args, lib_opts) in HEAP_CASES.items():
        ref, reads = make_heap_inputs(inputs, tmp)
        outs = []
        for hs in ("yes", "no"):
            a = [x if x != "SPLIT" else os.path.join(tmp, name + ".split") for x in args]
            cmd = [refbin, "-t", "8"] + a + ["--heap-sort=" + hs, ref, reads]
            outs.append(subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout)
        sam = "-a" in args
        out, out0 = (sam_without_pg(o) if sam else o for o in outs)
        with gzip.GzipFile(os.path.join(gdir, name + (".sam.stripped.gz" if sam else ".paf.gz")), "wb", mtime=0) as f:
            f.write(sam_strip_seq(out) if sam else out)
        manifest[name] = dict(inputs=inputs, lib=lib_opts, sam=sam, ref_md5=md5(ref), reads_md5=md5(reads),
                              # not "cmd": the command-line parse check replays every "cmd" of the manifests, and the command line
                              # refuses --heap-sort=yes
                              ref_cmd=" ".join(["winnowmap"] + [x if x != "SPLIT" else "<prefix>" for x in args] +
                                               ["--heap-sort=yes", "ref.fa", "reads.fa"]),
                              out_md5=hashlib.md5(out).hexdigest(), n_lines=out.count(b"\n"),
                              n_lines_differing=len(set(out.split(b"\n")) ^ set(out0.split(b"\n"))))
        print(name, manifest[name]["n_lines"], "lines,", manifest[name]["n_lines_differing"], "differ from --heap-sort=no", flush=True)
    json.dump(manifest, open(os.path.join(gdir, "heap_manifest.json"), "w"), indent=1, sort_keys=True)


# ---- junction annotation (--junc-bed with spliced base-level alignment): tests/golden/splice_junc_manifest.json and splice_junc_*;
# the other manifests are not touched.  The inputs are those of the splice_aln_* cases plus a BED of the transcriptome: "full" lists
# every transcript (isoforms and paralogs included) as BED12 with the gene's strand, "mixed" (gzipped) half of them as BED12 and
# the other lines a reader has to drop or cut short.  Every case must differ from the same command without --junc-bed.
JUNC_BED_SEED = 3051
SPLICE_JUNC_CASES = {
    # name: (reads, BED, reference options, library options)
    "splice_junc_c": ("tx", "full", ["-x", "splice", "-c"], dict(preset="splice")),
    "splice_junc_a": ("tx", "full", ["-x", "splice", "-a"], dict(preset="splice", sam=True)),
    "splice_junc_hq_cs": ("tx_hq", "full", ["-x", "splice:hq", "-c", "--cs"], dict(preset="splice:hq", set_flags=F_OUT_CS)),
    "splice_junc_cdna_md": ("tx", "full", ["-x", "cdna", "-a", "--MD"], dict(preset="cdna", sam=True, set_flags=F_OUT_MD)),
    "splice_junc_uf": ("tx", "full", ["-x", "splice", "-c", "-u", "f"], dict(preset="splice", set_flags=F_SPLICE_FOR, clear_flags=F_SPLICE_REV)),
    "splice_junc_ur": ("tx", "full", ["-x", "splice", "-c", "-u", "r"], dict(preset="splice", set_flags=F_SPLICE_REV, clear_flags=F_SPLICE_FOR)),
    "splice_junc_mixed": ("tx", "mixed", ["-x", "splice", "-c"], dict(preset="splice")),
    "splice_junc_H": ("tx", "full", ["-x", "splice", "-c", "-H"], dict(preset="splice", hpc=True)),
    "splice_junc_I_split": ("tx", "full", ["-x", "splice", "-c", "-I", "500k", "--split-prefix", "SPLIT"],
                            dict(preset="splice", part_bases=500000, split=True)),
}


def _bed12(name, chrom, strand, exons, score):
    st, en = exons[0][0], exons[-1][1]
    return "\t".join([chrom, str(st), str(en), name, str(score), strand, str(st), str(en), "0", str(len(exons)),
                      ",".join(str(b - a) for a, b in exons) + ",", ",".join(str(a - st) for a, _ in exons) + ","])


def make_junc_beds(outdir):
    """(full BED, mixed BED.gz) of the splice transcriptome."""
    c = SPLICE
    layout = []
    contigs, _ = gen_data.make_transcriptome(np.random.default_rng(c["ref_seed"]), c["genome_len"], c["n_genes"], layout=layout)
    rng = np.random.default_rng(JUNC_BED_SEED)
    full = [_bed12(n, ch, sd, ex, int(rng.integers(0, 1001))) for n, ch, sd, ex in layout]
    mixed = ["track name=junctions description=\"test\"", "# introns of half the transcripts"]
    flip = {"+": "-", "-": "+"}
    for i, (n, ch, sd, ex) in enumerate(layout):
        sc = int(rng.integers(0, 1001))
        if i % 2 == 0:
            mixed.append(_bed12(n, ch, sd, ex, sc))
            continue
        introns = [(ex[j][1], ex[j + 1][0]) for j in range(len(ex) - 1)]
        for j, (a, b) in enumerate(introns):
            kind = int(rng.integers(0, 6))
            if kind <= 2:  # BED6, the right strand
                mixed.append(f"{ch}\t{a}\t{b}\t{n}.i{j}\t{sc}\t{sd}")
            elif kind == 3:  # no strand
                mixed.append(f"{ch}\t{a}\t{b}\t{n}.i{j}\t{sc}\t.")
            elif kind == 4:  # the wrong strand
                mixed.append(f"{ch}\t{a}\t{b}\t{n}.i{j}\t{sc}\t{flip[sd]}")
            else:  # BED4: no score, no strand
                mixed.append(f"{ch}\t{a}\t{b}\t{n}.i{j}")
    n, ch, sd, ex = layout[1]
    b12 = _bed12(n, ch, sd, ex, 7).split("\t")
    L = len(contigs[0][1])
    mixed += [
        f"chrUn\t{ex[0][1]}\t{ex[1][0]}\tunknown\t0\t+",                       # a contig the index does not have
        f"{ch}\t{ex[0][1]}\t{ex[0][1]}\tempty\t0\t{sd}",                         # st == en
        f"{ch}\t{ex[1][0]}\t{ex[0][1]}\treversed\t0\t{sd}",                      # st > en
        f"{ch}\t-10\t{ex[0][1]}\tnegative\t0\t{sd}",                             # a negative start
        "\t".join(b12[:11]),                                                     # 11 columns: [chromStart, chromEnd) itself
        "\t".join(b12[:9] + ["x" + b12[9]] + b12[10:]),                           # a non-digit block count: the same
        "\t".join(b12[:3] + ["crlf", "0", sd]) + "\r",                            # CRLF line ending
        f"chr1\t{L - 300}\t{L - 100}\tnear_end\t0\t+",
    ]
    os.makedirs(outdir, exist_ok=True)
    fb, mb = os.path.join(outdir, "junc_full.bed"), os.path.join(outdir, "junc_mixed.bed.gz")
    with open(fb, "w") as f:
        f.write("\n".join(full) + "\n")
    with gzip.GzipFile(mb, "wb", mtime=0) as f:
        f.write(("\n".join(mixed) + "\n").encode())
    return fb, mb


def make_junc_inputs(name, outdir):
    """(genome FASTA, reads FASTA, -W file, BED) of one splice_junc_* case."""
    reads_kind, bed = SPLICE_JUNC_CASES[name][:2]
    ref, reads, wfile = make_splice_inputs(reads_kind, outdir)
    fb, mb = make_junc_beds(outdir)
    return ref, reads, wfile, fb if bed == "full" else mb


def main_junc():
    # the reference with the one patch its BED reader needs to read a line at all (oracle/build_junc.sh)
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap_junc")
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "winnowmap")):
        subprocess.check_call([os.path.join(ROOT, "oracle", "build_ref.sh")])
    subprocess.check_call([os.path.join(ROOT, "oracle", "build_junc.sh")])
    gdir = os.path.join(ROOT, "tests", "golden")
    tmp = "/tmp/wm_golden_junc"
    manifest = {}
    for name, (reads_kind, bed_kind, args, lib_opts) in SPLICE_JUNC_CASES.items():
        ref, reads, wfile, bed = make_junc_inputs(name, tmp)
        args = [a if a != "SPLIT" else os.path.join(tmp, name + ".split") for a in args]
        outs = []
        for extra in (["--junc-bed", bed], []):
            cmd = [refbin, "-t", "4"] + args + extra + ["-W", wfile, ref, reads]
            outs.append(subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True).stdout)
        sam = "-a" in args
        out, out0 = (sam_without_pg(o) if sam else o for o in outs)
        n_diff = len(set(out.split(b"\n")) ^ set(out0.split(b"\n")))
        assert n_diff > 0, f"{name}: --junc-bed changes nothing"
        with gzip.GzipFile(os.path.join(gdir, name + (".sam.stripped.gz" if sam else ".paf.gz")), "wb", mtime=0) as f:
            f.write(sam_strip_seq(out) if sam else out)
        manifest[name] = dict(reads=reads_kind, bed=bed_kind, lib=lib_opts, sam=sam, ref_md5=md5(ref), reads_md5=md5(reads), w_md5=md5(wfile),
                              bed_md5=md5(bed),
                              # not "cmd": the command-line parse check replays every "cmd" of the manifests, and the command line
                              # refuses spliced alignment
                              ref_cmd=" ".join(["winnowmap"] + [a if not a.startswith(tmp) else "<prefix>" for a in args] +
                                               ["--junc-bed", os.path.basename(bed), "-W", "rep.txt", "ref.fa", "reads.fa"]),
                              out_md5=hashlib.md5(out).hexdigest(), n_lines=out.count(b"\n"), n_lines_differing=n_diff)
        print(name, manifest[name]["n_lines"], "lines,", n_diff, "differ from the run without --junc-bed")
    json.dump(manifest, open(os.path.join(gdir, "splice_junc_manifest.json"), "w"), indent=1, sort_keys=True)
    record_junc_intervals(tmp, gdir)


def record_junc_intervals(tmp, gdir):
    """tests/golden/splice_junc_ref_intervals.npz: the reference's mm_idx_t::I after mm_idx_bed_read of both BEDs on the splice
    genome's names, as raw 16-byte records (<bed>_recs) with per-contig offsets (<bed>_off)."""
    import ctypes as C
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_harness_junc.so"))
    names = [nm for nm, _ in read_fasta(make_splice_inputs("tx", tmp)[0])]
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    out = {}
    for kind, bed in zip(("full", "mixed"), make_junc_beds(tmp)):
        assert L.ref_bed_read(len(names), arr, bed.encode()) == 0
        recs, off = [], [0]
        for rid in range(len(names)):
            n = L.ref_bed_intervals(rid, None, 0)
            buf = np.zeros(4 * n, np.int32)
            L.ref_bed_intervals(rid, buf.ctypes.data_as(C.c_void_p), n)
            recs.append(buf)
            off.append(off[-1] + n)
        out[kind + "_recs"] = np.concatenate(recs).reshape(-1, 4) if recs else np.zeros((0, 4), np.int32)
        out[kind + "_off"] = np.array(off, np.int64)
        out[kind + "_md5"] = np.array(md5(bed))
    np.savez_compressed(os.path.join(gdir, "splice_junc_ref_intervals.npz"), names=np.array(names), **out)


if __name__ == "__main__":
    if "--heap" in sys.argv:
        main_heap()
    elif "--junc" in sys.argv:
        main_junc()
    elif "--sdust" in sys.argv:
        main_sdust()
    elif "--cli" in sys.argv:
        main_cli()
    elif "--splice-aln" in sys.argv:
        main_splice_aln()
    elif "--splice" in sys.argv:
        main_splice()
    elif "--hpc" in sys.argv:
        main_hpc()
    elif "--overlap" in sys.argv:
        main_overlap()
    elif "--parts" in sys.argv:
        main_parts()
    else:
        main()
