#!/usr/bin/env python
"""Deterministic synthetic inputs for the BASELINE.json configs (SURVEY.md section 8d).

ref:   i.i.d. uniform ACGT contigs (optionally tandem-repeat enriched, config 5 style)
reads: log-normal lengths with the requested N50, uniform start, 50/50 strand,
       i.i.d. per-base errors (40% sub / 30% del / 30% ins)
-W:    meryl stand-in (ext/meryl does not build offline): canonical k-mers whose count is
       above the threshold chosen by meryl's `distinct=0.9998` rule
       (reference: ext/meryl/src/meryl/merylOp-nextMer.C:103-115).

Everything is numpy + PCG64 (numpy.random.default_rng(seed)); nothing here is on the
product path.
"""
import argparse
import math
import sys
import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for a, b in zip(b"ACGTN", b"TGCAN"):
    COMP[a] = b


def random_seq(rng, n):
    return ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]


def mutate(rng, seq, err, split=(0.4, 0.3, 0.3)):
    """Apply i.i.d. per-base errors; returns a new uint8 array."""
    n = len(seq)
    if err <= 0 or n == 0:
        return seq.copy()
    r = rng.random(n)
    sub = r < err * split[0]
    dele = (r >= err * split[0]) & (r < err * (split[0] + split[1]))
    ins = (r >= err * (split[0] + split[1])) & (r < err)
    out = seq.copy()
    ns = int(sub.sum())
    if ns:
        # substitute with a different base
        shift = rng.integers(1, 4, size=ns, dtype=np.uint8)
        codes = np.searchsorted(ACGT, out[sub]).astype(np.uint8)
        out[sub] = ACGT[(codes + shift) & 3]
    keep = ~dele
    # insertion: emit the base followed by one random base
    reps = np.ones(n, dtype=np.int64)
    reps[ins] = 2
    reps[~keep] = 0
    idx = np.repeat(np.arange(n), reps)
    res = out[idx]
    # positions of the second copy of inserted bases
    first = np.ones(len(idx), dtype=bool)
    first[1:] = idx[1:] != idx[:-1]
    n_ins = int((~first).sum())
    if n_ins:
        res[~first] = random_seq(rng, n_ins)
    return res


def make_ref(rng, total, n_contigs, tandem=False):
    """Return list of (name, uint8 array)."""
    contigs = []
    per = total // n_contigs
    fam = None
    if tandem:
        fam = [random_seq(rng, L) for L in (171, 340, 2000, 5000)]
    for c in range(n_contigs):
        L = per if c < n_contigs - 1 else total - per * (n_contigs - 1)
        seq = random_seq(rng, L)
        if tandem:
            # every 1 Mbp (or once per contig when smaller) insert a tandem array
            step = 1_000_000 if L > 1_500_000 else max(L // 2, 1)
            pos = step // 2
            while pos < L:
                unit = mutate(rng, fam[int(rng.integers(0, len(fam)))], 0.05, (1.0, 0.0, 0.0))
                copies = int(rng.integers(200, 2001))
                budget = min(int(0.15 * step), L - pos)
                copies = max(2, min(copies, budget // len(unit)))
                arr = np.concatenate([mutate(rng, unit, 0.01, (1.0, 0.0, 0.0)) for _ in range(copies)])
                arr = arr[: L - pos]
                seq[pos:pos + len(arr)] = arr
                pos += step
        contigs.append((f"chr{c + 1}", seq))
    return contigs


def write_fasta(path, recs, width=0):
    with open(path, "wb") as f:
        for name, seq in recs:
            f.write(b">" + name.encode() + b"\n")
            f.write(seq.tobytes())
            f.write(b"\n")


def read_fasta(path):
    recs = []
    name, chunks = None, []
    with open(path, "rb") as f:
        for line in f:
            line = line.rstrip()
            if line.startswith(b">"):
                if name is not None:
                    recs.append((name, np.frombuffer(b"".join(chunks), dtype=np.uint8)))
                name, chunks = line[1:].split()[0].decode(), []
            else:
                chunks.append(line)
    if name is not None:
        recs.append((name, np.frombuffer(b"".join(chunks), dtype=np.uint8)))
    return recs


def make_reads(rng, contigs, n_reads, n50, err, min_len=1000, max_len=200000):
    sigma = 0.5
    mu = math.log(n50) - sigma * sigma
    lens = np.clip(rng.lognormal(mu, sigma, n_reads), min_len, max_len).astype(np.int64)
    clens = np.array([len(s) for _, s in contigs], dtype=np.int64)
    recs = []
    for i in range(n_reads):
        L = int(lens[i])
        ci = int(rng.choice(len(contigs), p=clens / clens.sum()))
        cl = int(clens[ci])
        if L > cl:
            L = cl
        st = int(rng.integers(0, cl - L + 1))
        frag = contigs[ci][1][st:st + L]
        strand = "+"
        if rng.random() < 0.5:
            frag = COMP[frag[::-1]]
            strand = "-"
        frag = mutate(rng, frag, err)
        recs.append((f"r{i}_{contigs[ci][0]}_{st}_{L}_{strand}", frag))
    return recs


def _revcomp(seq):
    return COMP[seq[::-1]]


def make_transcriptome(rng, genome_len, n_genes, n_contigs=2, long_introns=2, long_genes=3, n_paralogs=3, layout=None):
    """A seeded spliced-transcript setting: (contigs, transcripts).  contigs: i.i.d. genome sequence with multi-exon genes on
    both strands.  Introns are GT-AG on the plus strand and CT-AC (their reverse complement) on the minus strand, except about
    one in twenty, which keeps random donor / acceptor bases; their lengths are log-uniform from 60 bp to 20 kb, plus
    `long_introns` introns above 200 kb.  The first `long_genes` genes have a long last exon, so that their transcripts exceed
    10 kb.  Every gene of three or more exons also gets an isoform that skips one internal exon, and `n_paralogs` genes get a
    copy elsewhere (exons 3 % divergent, introns of their own).  transcripts: (name, mRNA as uint8 in the gene's sense, 5' to 3').
    layout, when a list, gets one (name, contig name, strand, [(start, end) of each exon on the contig, ascending]) per
    transcript, in the order of `transcripts` (the random draws are the same either way)."""
    contigs = [random_seq(rng, genome_len // n_contigs) for _ in range(n_contigs)]
    cursor = [1000] * n_contigs
    exon_seqs, transcripts, n_long = [], [], 0

    def intron_lengths(ne, g):
        nonlocal n_long
        introns = [int(round(math.exp(rng.uniform(math.log(60), math.log(20000))))) for _ in range(ne - 1)]
        if n_long < long_introns and g >= long_genes and ne > 2:
            introns[(ne - 1) // 2] = int(rng.integers(200500, 230000))
            n_long += 1
        return introns

    def place(name, bodies, introns, strand, ci):
        seq = contigs[ci]
        span = sum(len(x) for x in bodies) + sum(introns)
        start = cursor[ci] + int(rng.integers(2000, 20000))
        if start + span + 1000 > len(seq):
            return None
        cursor[ci] = start + span
        pos, parts, coords = start, [], []
        for e, body in enumerate(bodies):
            seq[pos:pos + len(body)] = body
            parts.append(body)
            coords.append((pos, pos + len(body)))
            pos += len(body)
            if e < len(introns):
                end = pos + introns[e]
                if rng.random() >= 0.05:
                    seq[pos:pos + 2] = np.frombuffer(b"GT" if strand == "+" else b"CT", np.uint8)
                    seq[end - 2:end] = np.frombuffer(b"AG" if strand == "+" else b"AC", np.uint8)
                pos = end
        isoforms = [(parts, coords)]
        if len(parts) >= 3:
            skip = int(rng.integers(1, len(parts) - 1))
            isoforms.append((parts[:skip] + parts[skip + 1:], coords[:skip] + coords[skip + 1:]))
        for iso, (ps, cs) in enumerate(isoforms):
            m = np.concatenate(ps)
            transcripts.append((f"{name}.{iso}{strand}", m if strand == "+" else _revcomp(m)))
            if layout is not None:
                layout.append((transcripts[-1][0], f"chr{ci + 1}", strand, cs))
        return parts

    for g in range(n_genes):
        ne = int(rng.integers(2, 11))
        lens = [int(x) for x in rng.integers(80, 400, ne)]
        lens[0] += int(rng.integers(50, 300))
        lens[-1] = int(rng.integers(9000, 13000)) if g < long_genes else lens[-1] + int(rng.integers(200, 1500))
        parts = place(f"g{g}", [random_seq(rng, L) for L in lens], intron_lengths(ne, g), "+" if rng.random() < 0.5 else "-", g % n_contigs)
        if parts is not None:
            exon_seqs.append(parts)
    for p in range(min(n_paralogs, len(exon_seqs))):
        src = exon_seqs[int(rng.integers(0, len(exon_seqs)))]
        bodies = [mutate(rng, x, 0.03, split=(1.0, 0.0, 0.0)) for x in src]
        place(f"p{p}", bodies, intron_lengths(len(bodies), long_genes), "+" if rng.random() < 0.5 else "-", p % n_contigs)
    return [(f"chr{i + 1}", c) for i, c in enumerate(contigs)], transcripts


def make_spliced_reads(rng, contigs, transcripts, n_reads, err, n_genomic=0, n_random=0, min_len=200):
    """cDNA-like reads of `transcripts` (make_transcriptome): full length or 5'-truncated, a poly(A) tail of 10-40 bases, either
    orientation, ONT-like i.i.d. errors at rate err; plus n_genomic unspliced genomic reads (1-5 kb) and n_random random ones."""
    recs = []
    for i in range(n_reads):
        name, m = transcripts[int(rng.integers(0, len(transcripts)))]
        if rng.random() < 0.5 and len(m) > 2 * min_len:
            m = m[int(rng.integers(0, len(m) - min_len)):]
        m = np.concatenate([m, np.full(int(rng.integers(10, 41)), ord("A"), np.uint8)])
        strand = "+"
        if rng.random() < 0.5:
            m, strand = _revcomp(m), "-"
        recs.append((f"t{i}_{name}_{strand}", mutate(rng, m, err)))
    for i in range(n_genomic):
        ci = int(rng.integers(0, len(contigs)))
        L = int(rng.integers(1000, 5001))
        st = int(rng.integers(0, len(contigs[ci][1]) - L))
        frag = contigs[ci][1][st:st + L]
        if rng.random() < 0.5:
            frag = _revcomp(frag)
        recs.append((f"gen{i}_{contigs[ci][0]}_{st}", mutate(rng, frag, err)))
    for i in range(n_random):
        recs.append((f"rand{i}", random_seq(rng, int(rng.integers(300, 3000)))))
    return recs


def count_kmers(contigs, k):
    """Canonical k-mer -> count, vectorised (k <= 31)."""
    mask = (1 << (2 * k)) - 1
    allk = []
    lut = np.full(256, 4, dtype=np.uint8)
    for i, ch in enumerate(b"ACGT"):
        lut[ch] = i
        lut[ch + 32] = i
    for _, seq in contigs:
        codes = lut[seq].astype(np.uint64)
        n = len(codes)
        if n < k:
            continue
        fw = np.zeros(n - k + 1, dtype=np.uint64)
        rv = np.zeros(n - k + 1, dtype=np.uint64)
        bad = np.zeros(n - k + 1, dtype=bool)
        for j in range(k):
            c = codes[j:n - k + 1 + j]
            bad |= c > 3
            fw = (fw << np.uint64(2)) | (c & np.uint64(3))
            rv = rv | ((np.uint64(3) - (c & np.uint64(3))) << np.uint64(2 * j))
        can = np.minimum(fw, rv)[~bad]
        allk.append(can)
    if not allk:
        return np.zeros(0, np.uint64), np.zeros(0, np.int64)
    allk = np.concatenate(allk)
    return np.unique(allk, return_counts=True)


def kmer_to_str(v, k):
    return "".join("ACGT"[(int(v) >> (2 * (k - 1 - i))) & 3] for i in range(k))


def _tools_lib():
    """tools/libwm_tools.so (built by __graft_entry__.build() from tools/wm_tools.c), or None."""
    import ctypes as C
    import os
    so = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libwm_tools.so")
    if not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.wm_tools_count.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    L.wm_tools_hist.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    L.wm_tools_hist.restype = C.c_int64
    L.wm_tools_above.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int64]
    L.wm_tools_above.restype = C.c_int64
    return L


def top_kmers(contigs, k, distinct=0.9998):
    """(kmers, counts, threshold): canonical k-mers with count > threshold, ascending.
    meryl rule: threshold = smallest count whose cumulative number of distinct k-mers reaches distinct * total
    distinct (ext/meryl/src/meryl/merylOp-nextMer.C:103-115)."""
    L = _tools_lib() if k <= 15 else None
    if L is not None:  # direct-index table in C (4^k uint32 counters): seconds per Gbp
        table = np.zeros(1 << (2 * k), dtype=np.uint32)
        for _, seq in contigs:
            seq = np.ascontiguousarray(seq)
            L.wm_tools_count(seq.ctypes.data, len(seq), k, table.ctypes.data)
        hist = np.zeros(1 << 20, dtype=np.int64)
        n_distinct = L.wm_tools_hist(table.ctypes.data, k, hist.ctypes.data, len(hist))
        cum = np.cumsum(hist)
        vals = np.nonzero(hist)[0]
        ti = int(np.searchsorted(cum[vals], distinct * n_distinct, side="left"))
        thr = int(vals[min(ti, len(vals) - 1)]) if len(vals) else 0
        m = L.wm_tools_above(table.ctypes.data, k, thr, None, None, 0)
        kmers = np.zeros(m, dtype=np.uint64); counts = np.zeros(m, dtype=np.uint32)
        if m:
            L.wm_tools_above(table.ctypes.data, k, thr, kmers.ctypes.data, counts.ctypes.data, m)
        return kmers, counts, thr
    kmers, counts = count_kmers(contigs, k)
    vals, hist = np.unique(counts, return_counts=True)
    cum = np.cumsum(hist)
    target = distinct * len(kmers)
    ti = int(np.searchsorted(cum, target, side="left"))
    thr = int(vals[min(ti, len(vals) - 1)])
    sel = counts > thr
    return kmers[sel], counts[sel], thr


def write_top_kmers(path, contigs, k, distinct=0.9998):
    kmers, counts, thr = top_kmers(contigs, k, distinct)
    with open(path, "w") as f:
        for v, c in zip(kmers, counts):
            f.write(f"{kmer_to_str(v, k)}\t{int(c)}\n")
    return len(kmers), thr


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    p = sub.add_parser("ref")
    p.add_argument("--out", required=True); p.add_argument("--len", type=int, required=True)
    p.add_argument("--contigs", type=int, default=1); p.add_argument("--seed", type=int, default=1001)
    p.add_argument("--tandem", action="store_true")
    p = sub.add_parser("reads")
    p.add_argument("--ref", required=True); p.add_argument("--out", required=True)
    p.add_argument("--n", type=int, required=True); p.add_argument("--n50", type=int, required=True)
    p.add_argument("--err", type=float, default=0.05); p.add_argument("--seed", type=int, default=2001)
    p.add_argument("--min-len", type=int, default=1000)
    p = sub.add_parser("topk")
    p.add_argument("--ref", required=True); p.add_argument("--out", required=True)
    p.add_argument("-k", type=int, default=15); p.add_argument("--distinct", type=float, default=0.9998)
    a = ap.parse_args()
    if a.cmd == "ref":
        rng = np.random.default_rng(a.seed)
        write_fasta(a.out, make_ref(rng, a.len, a.contigs, a.tandem))
    elif a.cmd == "reads":
        rng = np.random.default_rng(a.seed)
        recs = make_reads(rng, read_fasta(a.ref), a.n, a.n50, a.err, min_len=a.min_len)
        write_fasta(a.out, recs)
        print(sum(len(s) for _, s in recs), file=sys.stderr)
    elif a.cmd == "topk":
        n, thr = write_top_kmers(a.out, read_fasta(a.ref), a.k, a.distinct)
        print(f"{n} k-mers above count {thr}", file=sys.stderr)


if __name__ == "__main__":
    main()
