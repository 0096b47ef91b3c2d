"""Homopolymer-compressed minimizers (-H) without a GPU: the oracle's HPC sketch and -H index against the digests of the
reference's own (oracle/ref_harness_hpc.cpp), and the bit functions of the device's compaction front end (csrc/hpc.cuh)
against a byte-per-base restatement."""
import ctypes as C
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hpc_lib as H  # noqa: E402
import make_golden  # noqa: E402

HPC_MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "hpc_manifest.json")))


def _sketch_set():
    return H.crafted_sequences() + H.random_sequences(7, 80)


@pytest.mark.parametrize("bloom", [False, True])
@pytest.mark.parametrize("w", [1, 10, 50, 255])
@pytest.mark.parametrize("k", [14, 15, 16, 19, 28])
def test_oracle_hpc_sketch_matches_reference(k, w, bloom):
    seqs = _sketch_set()
    kmers = H.hpc_kmers(seqs, k, 200, seed=k) if bloom else np.zeros(0, dtype=np.uint64)
    ob = H.HpcBloom(kmers) if bloom else None
    got = [H.oracle_sketch_hpc(s, w, k, i, ob) for i, s in enumerate(seqs)]
    spans = np.concatenate(got)[:, 0] & np.uint64(0xff)
    assert (spans > np.uint64(k)).any()
    ref = lambda: tuple(H.ref_sketch_hpc(s, w, k, i, kmers) for i, s in enumerate(seqs))  # noqa: E731
    H.assert_ref(f"hpc_sketch_k{k}_w{w}_{'bloom' if bloom else 'plain'}", tuple(got), ref)


def test_hpc_sketch_reaches_the_corners():
    """The crafted set really holds what it is meant to: a span >= 256 that is dropped, and runs cut at a slice end."""
    s = H.crafted_sequences()[1]  # a 300-bp run
    code, pos = H.hpc_compress(s)
    assert len(code) < len(s) and pos[-1] == len(s) - 1
    run_end = s.index(b"G" * 300) + 299
    assert run_end in pos
    full = H.oracle_sketch_hpc(s, 1, 15)  # w = 1: every valid k-mer of span < 256 is a minimizer
    assert len(full) and not (full[:, 0] & np.uint64(0xff) >= np.uint64(256)).any()
    # the 15 k-mers that contain the run cover more than 255 bases: none of them is a minimizer
    j = int(np.searchsorted(pos, run_end))
    y = (full[:, 1] & np.uint64(0xffffffff)) >> np.uint64(1)
    assert not np.isin(pos[j:j + 15], y).any() and np.isin(pos[j + 15:j + 30], y).any()


@pytest.mark.parametrize("name", ["hpc_clr", "hpc_ont_small"])
def test_oracle_hpc_index_matches_reference(name, tmp_path):
    """The flattened -H index of the reference (mm_idx_reader_read with MM_I_HPC) is the oracle's index of its HPC sketches."""
    from winnowmap_b200.mapper import make_options
    ref, _, _ = make_golden.make_hpc_inputs(name, str(tmp_path))
    io, _ = make_options(make_golden.HPC_CASES[name]["preset"])
    recs = make_golden.read_fasta(ref)
    got = H.oracle_index_hpc([(n, s.encode()) for n, s in recs], io.k, io.w, H.HpcBloom([]))
    H.assert_ref(f"hpc_index_{name}", got, lambda: H.ref_index_hpc(ref, None, io.k, io.w))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hpc") / "hpc_emul.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include",
                           os.path.join(ROOT, "tests", "hostsim", "hpc_emul.cpp"), "-o", so])
    L = C.CDLL(so)
    L.wmt_hpc_ends.restype = C.c_long
    L.wmt_hpc_ends.argtypes = [C.c_char_p, C.c_long, C.c_void_p, C.c_int, C.c_void_p]
    return L


def test_compaction_bits_match_byte_restatement(emul):
    """Slices at every offset of the 32-base groups, with runs and N crossing group and slice boundaries."""
    seqs = H.crafted_sequences() + H.random_sequences(3, 300, lo=1, hi=400)
    rng = np.random.default_rng(5)
    pool, off = bytearray(), [0]
    for s in seqs:  # slices start at arbitrary offsets, some inside a run that continues from the previous slice
        pool += s
        off.append(len(pool))
        if rng.random() < 0.3:
            pool += s[-1:] * int(rng.integers(1, 5))
            off.append(len(pool))
    off = np.array(off, dtype=np.int64)
    out = np.zeros(len(pool) + 1, dtype=np.int32)
    n = emul.wmt_hpc_ends(bytes(pool), len(pool), off.ctypes.data, len(off) - 1, out.ctypes.data)
    exp = np.concatenate([H.hpc_compress(bytes(pool[off[i]:off[i + 1]]))[1] for i in range(len(off) - 1)])
    assert n == len(exp) and np.array_equal(out[:n], exp)


@pytest.fixture(scope="module")
def hostsim(tmp_path_factory):
    """The product's host orchestration on the oracle backend with an HPC index (tests/hostsim/hpc_backend.cpp)."""
    d, cs = os.path.join(ROOT, "tests", "hostsim"), os.path.join(ROOT, "winnowmap_b200", "csrc")
    so = str(tmp_path_factory.mktemp("hpc_hostsim") / "libwm_hostsim_hpc.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
                           f"-I{os.environ.get('CUDA_HOME', '/usr/local/cuda')}/include", os.path.join(d, "hpc_backend.cpp"),
                           os.path.join(d, "kernel_emul.cpp")] + [os.path.join(cs, f) for f in ("host_map.cpp", "host_align.cpp", "host_glue.cpp", "host_io.cpp", "host_format.cpp")] +
                          ["-x", "c", os.path.join(ROOT, "oracle", "wm_oracle.c"), os.path.join(ROOT, "oracle", "wm_oracle_hpc.c"),
                           "-o", so, "-lz", "-lm", "-lpthread"], stderr=subprocess.DEVNULL)
    L = C.CDLL(so)
    L.wmt_map_file.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    return L


@pytest.mark.parametrize("name", sorted(HPC_MANIFEST))
def test_host_pipeline_matches_hpc_golden(hostsim, name, tmp_path):
    """The product's host orchestration on the oracle-backed backend: pins the HPC branch of adjust_minier without a GPU.
    (The stage-1 divergence estimate, which averages the spans, does not reach this version's output: only stage-1
    chains carry it, and the printed records are made again in stage 2.)"""
    m = HPC_MANIFEST[name]
    ref, reads, wfile = make_golden.make_hpc_inputs(name, str(tmp_path))
    assert make_golden.md5(ref) == m["ref_md5"] and make_golden.md5(reads) == m["reads_md5"]
    out = str(tmp_path / "o.paf")
    rc = hostsim.wmt_map_file(ref.encode(), wfile.encode() if wfile else None, m["params"]["preset"].encode(), reads.encode(), out.encode(), 8)
    assert rc == 0
    exp = gzip.open(os.path.join(ROOT, "tests", "golden", name + ".paf.gz")).read()
    got = open(out, "rb").read()
    if got != exp:
        for i, (x, y) in enumerate(zip(exp.split(b"\n"), got.split(b"\n"))):
            assert x == y, f"line {i}: exp {x[:200]!r} got {y[:200]!r}"
        raise AssertionError("line count differs")
