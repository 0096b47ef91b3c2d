"""ctypes bindings and inputs for the SDUST (-T) tests: the oracle's SDUST and minimizer squeeze (oracle/wm_oracle_sdust.c, in
oracle/libwm_oracle_sdust.so), the reference's own sdust() and mm_dust_minier (oracle/_ref/libref_harness_sdust.so) and the
device code compiled for the host (tests/hostsim/sdust_emul.cpp).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as ol

ROOT = ol.ROOT
_u64p = C.POINTER(C.c_uint64)
_libs = {}
T_SET = (1, 2, 5, 10, 20, 30, 40, 100)

# What the reference computes for these inputs is pinned by digests (oracle_lib.digest) in tests/golden/sdust_ref_digests.json.
# WM_RECORD_REF=1 (with oracle/_ref built) recomputes every digest a test run reaches from the reference and rewrites the file.
SDUST_DIGESTS = os.path.join(ROOT, "tests", "golden", "sdust_ref_digests.json")
_digests = None


def assert_ref(key, got, ref_fn):
    global _digests
    if _digests is None:
        _digests = json.load(open(SDUST_DIGESTS)) if os.path.exists(SDUST_DIGESTS) else {}
    if ol.recording():
        out = ref_fn()
        _digests[key] = ol.digest(*(out if isinstance(out, tuple) else (out,)))
        with open(SDUST_DIGESTS, "w") as f:
            json.dump(_digests, f, indent=0, sort_keys=True)
            f.write("\n")
    assert key in _digests, f"no reference digest for {key} (record with WM_RECORD_REF=1)"
    assert ol.digest(*(got if isinstance(got, tuple) else (got,))) == _digests[key], key


def oracle():
    if "oracle" not in _libs:
        so = os.path.join(ROOT, "oracle", "libwm_oracle_sdust.so")
        srcs = [os.path.join(ROOT, "oracle", f) for f in ("wm_oracle.c", "wm_oracle_sdust.c")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call([os.path.join(ROOT, "oracle", "build_sdust.sh")], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.wmo_sdust.restype = C.c_long
        L.wmo_sdust.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, _u64p, C.c_long, C.POINTER(C.c_int)]
        L.wmo_dust_minier.restype = C.c_long
        L.wmo_dust_minier.argtypes = [_u64p, C.c_long, _u64p, C.c_long]
        _libs["oracle"] = L
    return _libs["oracle"]


def ref():
    if "ref" not in _libs:
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_harness_sdust.so"))
        L.ref_sdust.restype = C.c_long
        L.ref_sdust.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, _u64p, C.c_long]
        L.ref_dust_minier.restype = C.c_long
        L.ref_dust_minier.argtypes = [_u64p, C.c_long, C.c_char_p, C.c_int, C.c_int]
        _libs["ref"] = L
    return _libs["ref"]


def emul():
    if "emul" not in _libs:
        so = os.path.join(tempfile.mkdtemp(prefix="wm_sdust_emul_"), "lib.so")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared",
                               f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                               os.path.join(ROOT, "tests", "hostsim", "sdust_emul.cpp"), "-o", so])
        L = C.CDLL(so)
        L.wmt_sdust_dev.restype = C.c_long
        L.wmt_sdust_dev.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, _u64p, C.c_long]
        L.wmt_dust_squeeze_dev.restype = C.c_long
        L.wmt_dust_squeeze_dev.argtypes = [_u64p, C.c_long, _u64p, C.c_int]
        _libs["emul"] = L
    return _libs["emul"]


def _regions(fn, seq, T, W, *extra):
    cap = len(seq) + W + 16
    out = np.zeros(cap, dtype=np.uint64)
    n = fn(seq, len(seq), T, W, out.ctypes.data_as(_u64p), cap, *extra)
    assert 0 <= n <= cap, n
    return out[:n].copy()


def oracle_sdust(seq: bytes, T, W=64):
    """The regions as start << 32 | end (uint64)."""
    return _regions(oracle().wmo_sdust, seq, T, W, None)


def oracle_max_perfect(seq: bytes, T, W=64):
    mp = C.c_int(0)
    _regions(oracle().wmo_sdust, seq, T, W, C.byref(mp))
    return mp.value


def ref_sdust(seq: bytes, T, W=64):
    return _regions(ref().ref_sdust, seq, T, W)


PCAP_FAST = 256  # csrc/sdust.cuh: WM_SDUST_PCAP_FAST


def emul_sdust(seq: bytes, T, W=64, pcap=0):
    """The device code's regions; pcap > 0: with a perfect-interval list of that size, None when the code gives the sequence up."""
    cap = len(seq) + W + 16
    out = np.zeros(cap, dtype=np.uint64)
    n = emul().wmt_sdust_dev(seq, len(seq), T, W, pcap, out.ctypes.data_as(_u64p), cap)
    if n == -2:
        return None
    assert 0 <= n <= cap, n
    return out[:n].copy()


def as_pairs(reg):
    return np.stack([(reg >> np.uint64(32)).astype(np.int64), (reg & np.uint64(0xffffffff)).astype(np.int64)], axis=1).reshape(-1, 2)


def oracle_dust_minier(xy, reg):
    a = np.ascontiguousarray(xy, dtype=np.uint64).copy()
    r = np.ascontiguousarray(reg, dtype=np.uint64)
    n = oracle().wmo_dust_minier(a.ctypes.data_as(_u64p), len(a), r.ctypes.data_as(_u64p), len(r))
    return a[:n].copy()


def ref_dust_minier(xy, seq: bytes, T):
    a = np.ascontiguousarray(xy, dtype=np.uint64).copy()
    n = ref().ref_dust_minier(a.ctypes.data_as(_u64p), len(a), seq, len(seq), T)
    return a[:n].copy()


def emul_dust_minier(xy, reg):
    a = np.ascontiguousarray(xy, dtype=np.uint64).copy()
    r = np.ascontiguousarray(reg, dtype=np.uint64)
    n = emul().wmt_dust_squeeze_dev(a.ctypes.data_as(_u64p), len(a), r.ctypes.data_as(_u64p), len(r))
    return a[:n].copy()


def acgt(rng, n):
    """n random bases as bytes (one byte per base)."""
    return np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=n)].tobytes()


def _mutate(rng, s: bytearray, rate):
    for i in np.nonzero(rng.random(len(s)) < rate)[0]:
        s[i] = b"ACGT"[int(rng.integers(0, 4))]
    return s


def crafted_sequences():
    """Homopolymers; di- and trinucleotide repeats with errors; N runs at every offset of a repeat; IUPAC, lowercase and U;
    lengths 0-2, W-1, W, W+1 and around them; repeats next to random sequence."""
    rng = np.random.default_rng(11)
    rand = lambda n: acgt(rng, n)  # noqa: E731
    out = [b"", b"A", b"AC", b"ACG", b"AAA", b"A" * 63, b"A" * 64, b"A" * 65, b"CA" * 31 + b"C", b"CAG" * 21 + b"C", b"CAG" * 22,
           b"A" * 300, b"G" * 2000, b"AC" * 500, b"ACG" * 400, b"AATG" * 300, b"ACGTA" * 200]
    for unit in (b"AC", b"CAG", b"AAG", b"GATA"):
        out.append(bytes(_mutate(rng, bytearray(unit * (600 // len(unit))), 0.05)))
        out.append(rand(200) + bytes(_mutate(rng, bytearray(unit * 100), 0.02)) + rand(200))
    rep = b"CA" * 60
    for off in range(0, 70, 3):  # an N run at every offset of a repeat, and runs of several lengths
        out.append(rep[:off] + b"N" * (1 + off % 5) + rep[off:])
    out.append(b"N" * 10 + b"A" * 100 + b"N" + b"A" * 100 + b"NN")
    out.append(b"acacacacacacacacacacacacacacacacacac" + b"RYKMSWacgu" * 6 + b"uuuuuuuuuuuuuuuuuuuuuu" + b"TTTTnTTTTTT" * 8)
    out.append(b"\x00\x01\x02\x03" * 40)  # bytes 0..3 are bases in seq_nt4_table
    for n in (61, 62, 63, 64, 65, 66, 127, 128, 129):
        out.append(b"AT" * (n // 2) + b"A" * (n % 2))
    return out


def random_sequences(seed, n, lo=0, hi=4000):
    """Random sequences with planted microsatellites and tandem repeats (mutated), N runs and lowercase stretches."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        L = int(rng.integers(lo, hi))
        s = bytearray(acgt(rng, L))
        for _ in range(int(rng.integers(0, 6))):
            if L < 10:
                break
            u = int(rng.integers(1, 12))
            unit = acgt(rng, u)
            span = int(rng.integers(10, min(L, 400) + 1))
            at = int(rng.integers(0, L - span + 1))
            s[at:at + span] = _mutate(rng, bytearray((unit * (span // u + 1))[:span]), float(rng.choice([0, 0.01, 0.05, 0.15])))
        if L > 20 and rng.random() < 0.3:
            at = int(rng.integers(0, L - 5))
            s[at:at + int(rng.integers(1, 5))] = b"N" * len(s[at:at + int(rng.integers(1, 5))])
        if L > 20 and rng.random() < 0.3:
            at = int(rng.integers(0, L - 20))
            s[at:at + 20] = bytes(s[at:at + 20]).lower()
        out.append(bytes(s))
    return out


def case_set():
    return crafted_sequences() + random_sequences(5, 150, hi=3000)
