#!/usr/bin/env python
"""Cost of homopolymer-compressed minimizers (-H) on one GPU, against the plain path, on bench-shaped ONT reads:

  1. the sketch stage alone (wm_bench_sketch: CUDA-event time of wm_sketch_run / wm_sketch_run_hpc on reads already packed
     on the device), plain and HPC, k = 15, w = 50;
  2. Mapper end to end (index build excluded), -x map-ont with -H against without, on a tandem-rich reference, in Mbase/s
     of wall time, alternating the two arms.

Prints the card's name and power limit with the numbers, and one JSON line at the end.  Everything it writes goes to a
temporary directory."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_data  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, plim = [s.strip() for s in out.split(",")]
        return name, plim
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mbases", type=float, default=32.0, help="read bases (Mbase)")
    ap.add_argument("--ref-mbases", type=float, default=20.0, help="reference length (Mbase)")
    ap.add_argument("--reps", type=int, default=5, help="timed sketch calls per arm")
    ap.add_argument("--rounds", type=int, default=2, help="alternating end-to-end rounds per arm")
    a = ap.parse_args()
    from winnowmap_b200 import kernels, lib
    from winnowmap_b200.mapper import Mapper
    L = lib()
    L.wm_bench_sketch.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.POINTER(C.c_int64), C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.POINTER(C.c_double)]
    name, plim = card()
    print(f"card: {name}, power limit {plim}", flush=True)
    rng = np.random.default_rng(7)
    contigs = gen_data.make_ref(rng, int(a.ref_mbases * 1e6), 1, True)
    n50 = 10000
    n_reads = max(1, int(a.mbases * 1e6 / (n50 * 0.8)))
    recs = gen_data.make_reads(np.random.default_rng(8), contigs, n_reads, n50, 0.05, min_len=1000)
    seqs = [bytes(s) for _, s in recs]
    n_bases = sum(len(s) for s in seqs)
    print(f"{len(seqs)} reads, {n_bases / 1e6:.1f} Mbase; reference {a.ref_mbases:.0f} Mbase with tandem arrays", flush=True)
    res = dict(card=name, power_limit=plim, n_bases=n_bases)
    # 1. sketch stage
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    buf = b"".join(seqs)
    bloom = kernels.Bloom(np.zeros(0, dtype=np.uint64))
    for hpc in (0, 1, 0, 1):
        ms = C.c_double()
        rc = L.wm_bench_sketch(bloom.h, len(seqs), buf, off.ctypes.data_as(C.POINTER(C.c_int64)), 50, 15, hpc, a.reps, C.byref(ms))
        assert rc == 0
        key = "sketch_ms_hpc" if hpc else "sketch_ms_plain"
        res.setdefault(key, []).append(round(ms.value, 3))
        print(f"sketch {'HPC  ' if hpc else 'plain'}: {ms.value:8.2f} ms  ({n_bases / ms.value / 1e3:.0f} Mbase/s)", flush=True)
    # 2. end to end
    with tempfile.TemporaryDirectory() as td:
        ref, reads = os.path.join(td, "ref.fa"), os.path.join(td, "reads.fa")
        gen_data.write_fasta(ref, contigs)
        gen_data.write_fasta(reads, recs)
        mappers = {hpc: Mapper(ref, None, preset="map-ont", hpc=bool(hpc)) for hpc in (0, 1)}
        for r in range(a.rounds + 1):  # round 0 warms both arms up
            for hpc in (0, 1):
                out = os.path.join(td, f"out{hpc}.paf")
                t0 = time.perf_counter()
                mappers[hpc].map_file(reads, out)
                dt = time.perf_counter() - t0
                if r == 0:
                    continue
                key = "e2e_mbase_s_hpc" if hpc else "e2e_mbase_s_plain"
                res.setdefault(key, []).append(round(n_bases / dt / 1e6, 2))
                print(f"map-ont {'-H' if hpc else '  '}: {dt:7.2f} s  {n_bases / dt / 1e6:7.2f} Mbase/s", flush=True)
        for mp in mappers.values():
            mp.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
