"""ctypes bindings and inputs for the homopolymer-compressed (-H) tests: the oracle's HPC sketch (oracle/wm_oracle_hpc.c,
in oracle/libwm_oracle_hpc.so) and the reference's HPC sketch and -H index (oracle/_ref/libref_harness_hpc.so).
TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import json
import os
import subprocess

import numpy as np

import oracle_lib as ol

ROOT = ol.ROOT
_u64p = C.POINTER(C.c_uint64)
_hpc = None
_ref_hpc = None


# What the reference computes for the -H inputs is pinned by digests (oracle_lib.digest) in tests/golden/hpc_ref_digests.json.
# WM_RECORD_REF=1 (with oracle/_ref built) recomputes every digest a test run reaches from the reference and rewrites the file.
HPC_DIGESTS = os.path.join(ROOT, "tests", "golden", "hpc_ref_digests.json")
_digests = None


def assert_ref(key, got, ref_fn):
    """got (an array or a tuple of arrays) equals what the reference computes for the same input."""
    global _digests
    if _digests is None:
        _digests = json.load(open(HPC_DIGESTS)) if os.path.exists(HPC_DIGESTS) else {}
    if ol.recording():
        out = ref_fn()
        _digests[key] = ol.digest(*(out if isinstance(out, tuple) else (out,)))
        with open(HPC_DIGESTS, "w") as f:
            json.dump(_digests, f, indent=0, sort_keys=True)
            f.write("\n")
    assert key in _digests, f"no reference digest for {key} (record with WM_RECORD_REF=1)"
    assert ol.digest(*(got if isinstance(got, tuple) else (got,))) == _digests[key], key


def oracle_hpc():
    global _hpc
    if _hpc is None:
        so = os.path.join(ROOT, "oracle", "libwm_oracle_hpc.so")
        srcs = [os.path.join(ROOT, "oracle", f) for f in ("wm_oracle.c", "wm_oracle_hpc.c")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call([os.path.join(ROOT, "oracle", "build_hpc.sh")], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmo_bloom_init.restype = C.c_void_p
        L.wmo_bloom_init.argtypes = [C.c_uint64]
        L.wmo_bloom_insert.argtypes = [C.c_void_p, C.c_uint64]
        L.wmo_bloom_free.argtypes = [C.c_void_p]
        L.wmo_sketch_hpc.restype = C.c_long
        L.wmo_sketch_hpc.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p, _u64p, C.c_long]
        L.wmo_hpc_compress.restype = C.c_long
        L.wmo_hpc_compress.argtypes = [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]
        _hpc = L
    return _hpc


class HpcBloom:
    """The oracle's down-weight filter, in the HPC oracle library's own instance."""

    def __init__(self, kmers):
        self.L = oracle_hpc()
        kmers = np.asarray(kmers, dtype=np.uint64)
        self.h = self.L.wmo_bloom_init(len(kmers))
        for k in kmers:
            self.L.wmo_bloom_insert(self.h, int(k))

    def __del__(self):
        try:
            self.L.wmo_bloom_free(self.h)
        except Exception:
            pass


def oracle_sketch_hpc(seq: bytes, w, k, rid=0, bloom=None):
    cap = len(seq) + 64
    out = np.zeros(cap * 2, dtype=np.uint64)
    n = oracle_hpc().wmo_sketch_hpc(seq, len(seq), w, k, rid, bloom.h if bloom else None, out.ctypes.data_as(_u64p), cap)
    assert n <= cap
    return out[: 2 * n].reshape(-1, 2).copy()


def hpc_compress(seq: bytes):
    code = np.zeros(max(len(seq), 1), dtype=np.uint8)
    pos = np.zeros(max(len(seq), 1), dtype=np.int32)
    n = oracle_hpc().wmo_hpc_compress(seq, len(seq), code.ctypes.data, pos.ctypes.data)
    return code[:n].copy(), pos[:n].copy()


def ref_hpc():
    global _ref_hpc
    if _ref_hpc is None:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_harness_hpc.so"))
        L.ref_sketch_ctx.restype = C.c_void_p
        L.ref_sketch_ctx.argtypes = [C.c_int, _u64p]
        L.ref_sketch_free.argtypes = [C.c_void_p]
        L.ref_sketch_hpc.restype = C.c_long
        L.ref_sketch_hpc.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_uint32, _u64p, C.c_long]
        L.ref_idx_build_flat_flag.restype = C.c_void_p
        L.ref_idx_build_flat_flag.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.ref_idx_flat_sizes.argtypes = [C.c_void_p, _u64p]
        for f in ("keys", "pos_off", "pos"):
            getattr(L, "ref_idx_flat_" + f).restype = _u64p
            getattr(L, "ref_idx_flat_" + f).argtypes = [C.c_void_p]
        L.ref_idx_flat_free.argtypes = [C.c_void_p]
        _ref_hpc = L
    return _ref_hpc


def ref_sketch_hpc(seq: bytes, w, k, rid=0, kmers=()):
    L = ref_hpc()
    km = np.ascontiguousarray(kmers, dtype=np.uint64)
    h = L.ref_sketch_ctx(len(km), km.ctypes.data_as(_u64p))
    try:
        cap = len(seq) + 64
        out = np.zeros(cap * 2, dtype=np.uint64)
        n = L.ref_sketch_hpc(h, seq, len(seq), w, k, rid, out.ctypes.data_as(_u64p), cap)
        assert n <= cap
        return out[: 2 * n].reshape(-1, 2).copy()
    finally:
        L.ref_sketch_free(h)


def ref_index_hpc(fasta, kmer_file, k, w):
    """keys, pos_off, pos of the reference's -H index (the bucket walk of INTEGRATION.md section 3)."""
    L = ref_hpc()
    f = L.ref_idx_build_flat_flag(fasta.encode(), kmer_file.encode() if kmer_file else None, w, k, 1, 1)
    assert f
    try:
        sz = np.zeros(7, dtype=np.uint64)
        L.ref_idx_flat_sizes(f, sz.ctypes.data_as(_u64p))
        nk, npos = int(sz[2]), int(sz[3])
        keys = np.ctypeslib.as_array(L.ref_idx_flat_keys(f), shape=(max(nk, 1),))[:nk].copy()
        poff = np.ctypeslib.as_array(L.ref_idx_flat_pos_off(f), shape=(nk + 1,)).copy()
        pos = np.ctypeslib.as_array(L.ref_idx_flat_pos(f), shape=(max(npos, 1),))[:npos].copy()
        return keys, poff, pos
    finally:
        L.ref_idx_flat_free(f)


def oracle_index_hpc(names_seqs, k, w, bloom=None):
    """The flattened index of the oracle's HPC sketches: keys (hash), CSR offsets and positions sorted as mm_idx_get returns them."""
    mz = [oracle_sketch_hpc(s, w, k, rid, bloom) for rid, (_, s) in enumerate(names_seqs) if len(s)]
    mz = np.concatenate(mz) if mz else np.zeros((0, 2), dtype=np.uint64)
    h, y = mz[:, 0] >> np.uint64(8), mz[:, 1]
    o = np.lexsort((y, h))
    h, y = h[o], y[o]
    keys, first = np.unique(h, return_index=True)
    poff = np.append(first, len(h)).astype(np.uint64)
    return keys.astype(np.uint64), poff, y.astype(np.uint64)


def rand_seq(rng, n):
    return bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=n))


def crafted_sequences():
    """Slices that reach every corner of the compression: runs crossing the ends, a 300-bp run, runs summing past 255
    within k symbols, N next to and inside runs, lower case, symmetric k-mers."""
    rng = np.random.default_rng(2024)
    out = []
    out.append(b"AAAA" + rand_seq(rng, 200) + b"TTTTTTT")                          # runs at both ends
    out.append(rand_seq(rng, 120) + b"G" * 300 + rand_seq(rng, 120))             # one 300-bp run
    parts = []
    for i in range(60):                                                          # long runs: spans past 255 within k symbols
        parts.append(b"ACGT"[i % 4:i % 4 + 1] * int(rng.integers(1, 40)))
    out.append(rand_seq(rng, 50) + b"".join(parts) + rand_seq(rng, 50))
    out.append(rand_seq(rng, 80) + b"AAAANAAAA" + rand_seq(rng, 40) + b"NNN" + b"CCCCCC" + b"N" + rand_seq(rng, 80))
    out.append(rand_seq(rng, 100).lower() + b"aaaAAAaa" + rand_seq(rng, 100) + b"ccCCgg" + rand_seq(rng, 60).lower())
    out.append(b"ACGT" * 60 + b"AT" * 50 + b"GC" * 40)                           # palindromic k-mers (even k)
    out.append(b"N" * 10 + rand_seq(rng, 300) + b"N" * 5)
    out.append(b"A" * 500)                                                       # one symbol
    out.append(b"AC" * 5)                                                        # shorter than k symbols
    hp = []
    for _ in range(200):                                                         # homopolymer-rich, like PacBio CLR
        c = int(rng.integers(0, 4))
        hp.append(b"ACGT"[c:c + 1] * int(rng.geometric(0.35)))
    out.append(b"".join(hp))
    return out


def random_sequences(seed, n, lo=50, hi=3000):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        L = int(rng.integers(lo, hi))
        s = bytearray()
        while len(s) < L:
            c = int(rng.integers(0, 4))
            s += b"ACGT"[c:c + 1] * int(rng.geometric(0.4))
        s = s[:L]
        for _ in range(int(rng.integers(0, 3))):  # a few N runs
            p, m = int(rng.integers(0, L)), int(rng.integers(1, 8))
            s[p:p + m] = b"N" * len(s[p:p + m])
        out.append(bytes(s))
    return out


def hpc_kmers(seqs, k, n, seed=0):
    """n canonical compressed k-mers drawn from the sequences (a -W list that the sketches really meet)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n * 4):
        s = seqs[int(rng.integers(0, len(seqs)))]
        code, _ = hpc_compress(s)
        if len(code) < k:
            continue
        p = int(rng.integers(0, len(code) - k + 1))
        c = code[p:p + k]
        if (c > 3).any():
            continue
        f = r = 0
        for x in c:
            f = f << 2 | int(x)
        for x in c[::-1]:
            r = r << 2 | (3 - int(x))
        out.append(min(f, r))
        if len(out) == n:
            break
    return np.array(out, dtype=np.uint64)
