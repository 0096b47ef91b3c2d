"""Shared helpers of the -W list tests (test_topfreq_cpu.py, test_gpu_topfreq.py): seeded genomes with the corners the
counter has to get right, the plain-C oracle (oracle/wm_oracle_topfreq.c, compiled here) and the k-mer spelling."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMP = bytes.maketrans(b"ACGTacgt", b"TGCAtgca")
_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_topfreq_oracle_"), "libwm_oracle_topfreq.so")
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", os.path.join(ROOT, "oracle", "wm_oracle_topfreq.c"), "-o", so])
        L = C.CDLL(so)
        L.wm_oracle_topfreq.restype = C.c_int64
        L.wm_oracle_topfreq.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
        _oracle = L
    return _oracle


def _bytes(s):
    return s if isinstance(s, (bytes, bytearray)) else np.ascontiguousarray(s).tobytes()


def oracle_top_kmers(contigs, k, distinct):
    """(kmers, counts, threshold, n_distinct) of the oracle on [(name, seq)]."""
    L = oracle_lib()
    seqs = [_bytes(s) for _, s in contigs]
    cat = b"".join(seqs)
    off = np.cumsum([0] + [len(s) for s in seqs]).astype(np.int64)
    thr, nd = C.c_uint64(0), C.c_int64(0)
    n = L.wm_oracle_topfreq(cat, off.ctypes.data, len(seqs), k, distinct, None, None, 0, C.byref(thr), C.byref(nd))
    kmers, counts = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint32)
    if n:
        L.wm_oracle_topfreq(cat, off.ctypes.data, len(seqs), k, distinct, kmers.ctypes.data, counts.ctypes.data, n, C.byref(thr), C.byref(nd))
    return kmers, counts, int(thr.value), int(nd.value)


def spell(code, k):
    return "".join("ACGT"[(int(code) >> (2 * (k - 1 - i))) & 3] for i in range(k))


def revcomp(s):
    return s.translate(COMP)[::-1]


def genome(seed, k, total=400_000):
    """Several contigs of random sequence with repeats (so that counts spread over many values), N runs, IUPAC codes, lower
    case, an empty contig and contigs shorter than k; for even k, reverse-complement palindromes planted many times."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    rand = lambda n: acgt[rng.integers(0, 4, n)].tobytes()  # noqa: E731
    units = [rand(int(rng.integers(k + 3, 400))) for _ in range(12)]
    pal = []
    if k % 2 == 0:
        for _ in range(6):
            h = rand(k // 2)
            pal.append(h + revcomp(h))
    contigs = []
    for c in range(5):
        parts, n = [], 0
        while n < total // 5:
            r = rng.random()
            if r < 0.25:
                s = units[int(rng.integers(0, len(units)))] * int(rng.integers(1, 6))
            elif r < 0.30 and pal:
                s = pal[int(rng.integers(0, len(pal)))] * int(rng.integers(1, 4))
            elif r < 0.33:
                s = b"N" * int(rng.integers(1, 60))
            elif r < 0.36:
                s = bytes(rng.choice(list(b"RYKMSWBDHVNrykmswbdhvn-.*"), int(rng.integers(1, 4))).tolist())
            else:
                s = rand(int(rng.integers(1, 3000)))
            if rng.random() < 0.1:
                s = s.lower()
            parts.append(s)
            n += len(s)
        contigs.append((f"ctg{c}", b"".join(parts)))
    contigs.insert(2, ("empty", b""))
    contigs.append(("short", rand(max(1, k - 1))))
    contigs.append(("exact", rand(k)))
    contigs.append(("shortN", rand(k // 2) + b"N" + rand(k // 2)))
    return contigs


def write_fasta(path, contigs):
    with open(path, "wb") as f:
        for name, s in contigs:
            f.write(b">" + name.encode() + b"\n" + _bytes(s) + b"\n")
    return path


def read_list(path):
    """A -W file: (codes, counts) as written by gen_data.write_top_kmers, codes from the spellings (encodeKmer's forward
    code: the file spells canonical codes)."""
    codes, counts = [], []
    for line in open(path):
        km, c = line.split()
        v = 0
        for ch in km:
            v = v << 2 | "ACGT".index(ch)
        codes.append(v)
        counts.append(int(c))
    return np.array(codes, dtype=np.uint64), np.array(counts, dtype=np.uint32)


def hist_contigs(counts, k=11, seed=3):
    """Contigs whose k-mer count histogram is exactly `counts` (one distinct canonical k-mer per entry): a k-mer of count
    c above 1000 is a homopolymer run of k + c - 1 bases (at most four of those: A/T and C/G share canonical codes, so
    two), any other one k-base contig per occurrence.  k odd: no palindromes."""
    rng = np.random.default_rng(seed)
    seen, out = set(), []
    big = iter([b"A", b"C"])
    for i, c in enumerate(counts):
        if c > 1000:
            out.append((f"h{i}", next(big) * (k + c - 1)))
            continue
        while True:
            s = bytes(rng.choice(list(b"ACGT"), k).tolist())
            if len(set(s)) == 1:
                continue
            can = min(s, revcomp(s))
            if can not in seen:
                seen.add(can)
                break
        out += [(f"k{i}_{j}", s) for j in range(c)]
    return out
