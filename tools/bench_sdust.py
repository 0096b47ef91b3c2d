#!/usr/bin/env python
"""Cost of SDUST low-complexity masking (-T) on one GPU, on tandem-rich ONT reads:

  1. the SDUST kernel alone (wm_bench_sdust: CUDA-event time of wm_sdust_run on reads already packed on the device), T = 20;
  2. the seed stage of a whole mapping run (MapStats t_seed: sketch, SDUST, seed lookup, sort and chaining of every wave), with
     -T 20 against without;
  3. Mapper end to end (index build excluded), -x map-ont -c with -T 20 against without, in Mbase/s of wall time, alternating
     the two arms after a warm-up round of each.

Prints the card's name, power limit and SM clocks (the maximum, the application clock and the clock read right after each
timed piece of work) with the numbers, and one JSON line at the end.  Everything it writes goes to a
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


def smi(fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={fields}", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    return [x.strip() for x in out.split(",")]


def card():
    """name, power limit, max SM clock and application (target) SM clock of GPU 0"""
    try:
        return smi("name,power.limit,clocks.max.sm,clocks.applications.graphics")
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"


def sm_clock():
    """the SM clock in effect now (read right after GPU work, so it is the clock under load)"""
    try:
        return smi("clocks.sm")[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mbases", type=float, default=32.0, help="read bases (Mbase)")
    ap.add_argument("--ref-mbases", type=float, default=20.0, help="reference length (Mbase)")
    ap.add_argument("--T", type=int, default=20, help="SDUST threshold")
    ap.add_argument("--reps", type=int, default=5, help="timed SDUST runs")
    ap.add_argument("--rounds", type=int, default=2, help="alternating end-to-end rounds per arm")
    a = ap.parse_args()
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import Mapper
    L = lib()
    L.wm_bench_sdust.argtypes = [C.c_int, C.c_char_p, C.POINTER(C.c_int64), C.c_int, C.c_int, C.POINTER(C.c_double)]
    name, plim, clk, app_clk = card()
    print(f"card: {name}, power limit {plim}, max SM clock {clk}, application SM clock {app_clk}", flush=True)
    rng = np.random.default_rng(7)
    contigs = gen_data.make_ref(rng, int(a.ref_mbases * 1e6), 1, True)
    n50 = 10000
    n_reads = max(1, int(a.mbases * 1e6 / (n50 * 0.8)))
    recs = gen_data.make_reads(np.random.default_rng(8), contigs, n_reads, n50, 0.05, min_len=1000)
    seqs = [bytes(s) for _, s in recs]
    n_bases = sum(len(s) for s in seqs)
    print(f"{len(seqs)} reads, {n_bases / 1e6:.1f} Mbase; reference {a.ref_mbases:.0f} Mbase with tandem arrays", flush=True)
    res = dict(card=name, power_limit=plim, max_sm_clock=clk, application_sm_clock=app_clk, n_bases=n_bases, T=a.T, sm_clock_under_load=[])
    # 1. the kernel alone, over the whole reads
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    buf = b"".join(seqs)
    for _ in range(2):
        ms = C.c_double()
        assert L.wm_bench_sdust(len(seqs), buf, off.ctypes.data_as(C.POINTER(C.c_int64)), a.T, a.reps, C.byref(ms)) == 0
        res.setdefault("sdust_kernel_ms", []).append(round(ms.value, 3))
        res["sm_clock_under_load"].append(sm_clock())
        print(f"SDUST kernel: {ms.value:8.2f} ms  ({n_bases / ms.value / 1e3:.0f} Mbase/s)  SM clock {res['sm_clock_under_load'][-1]}", flush=True)
    # 2 and 3. whole runs
    with tempfile.TemporaryDirectory() as td:
        ref, reads = os.path.join(td, "ref.fa"), os.path.join(td, "reads.fa")
        gen_data.write_fasta(ref, contigs)
        gen_data.write_fasta(reads, recs)
        mappers = {T: Mapper(ref, None, preset="map-ont", sdust_thres=T) for T in (0, a.T)}
        for r in range(a.rounds + 1):  # round 0 warms both arms up
            for T in (0, a.T):
                out = os.path.join(td, f"out{T}.paf")
                mappers[T].reset_stats()
                t0 = time.perf_counter()
                mappers[T].map_file(reads, out)
                dt = time.perf_counter() - t0
                if r == 0:
                    continue
                t_seed = mappers[T].stats()["t_seed"]
                res["sm_clock_under_load"].append(sm_clock())
                res.setdefault(f"e2e_mbase_s_T{T}", []).append(round(n_bases / dt / 1e6, 2))
                res.setdefault(f"t_seed_s_T{T}", []).append(round(t_seed, 3))
                print(f"map-ont -c -T {T:3d}: {dt:7.2f} s  {n_bases / dt / 1e6:7.2f} Mbase/s  seed stage {t_seed:6.2f} s", flush=True)
        res["paf_lines_T0"], res["paf_lines_T"] = (sum(1 for _ in open(os.path.join(td, f"out{T}.paf"))) for T in (0, a.T))
        for mp in mappers.values():
            mp.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
