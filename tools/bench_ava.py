#!/usr/bin/env python
"""All-vs-all read overlaps (-X) on one GPU: a synthetic ONT read set mapped against itself.

  1. Mapper.map_file end to end (index build excluded), -x map-ont -X without and with -c, in Mbase/s of wall time;
  2. the seed stage with the seed filter against without it: the same mapping options without the filter bits are
     -P --no-long-join (-X is -D -P --no-long-join --dual=no).  Reported per arm: the wall time of the seed calls of the
     orchestrator (each ends in a device synchronise; the `t_seed` statistic), the anchors in the chains the seed stage
     returns (`n_chained`) and the kernel launches;
  3. optionally the reference binary's own -X run on the same files (oracle/_ref/winnowmap, when build() made it).

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
from bench_hpc import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mbases", type=float, default=20.0, help="read bases (Mbase)")
    ap.add_argument("--genome-mbases", type=float, default=5.0, help="length of the genome the reads come from (Mbase)")
    ap.add_argument("--rounds", type=int, default=2, help="timed rounds per arm, after one warm-up round")
    ap.add_argument("--ref-threads", type=int, default=0, help="threads of the reference's run (0: skip it)")
    a = ap.parse_args()
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import F_ALL_CHAINS, F_NO_LJOIN, Mapper
    L = lib()
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    name, plim = card()
    print(f"card: {name}, power limit {plim}", flush=True)
    genome = gen_data.make_ref(np.random.default_rng(7), int(a.genome_mbases * 1e6), 1, False)
    n50 = 12000
    n_reads = max(2, int(a.mbases * 1e6 / (n50 * 0.8)))
    recs = gen_data.make_reads(np.random.default_rng(8), genome, n_reads, n50, 0.05, min_len=2000)
    n_bases = sum(len(s) for _, s in recs)
    print(f"{len(recs)} reads, {n_bases / 1e6:.1f} Mbase from a {a.genome_mbases:.0f} Mbase genome (coverage {n_bases / a.genome_mbases / 1e6:.1f})", flush=True)
    res = dict(card=name, power_limit=plim, n_reads=len(recs), n_bases=n_bases)
    with tempfile.TemporaryDirectory() as td:
        reads = os.path.join(td, "reads.fa")
        gen_data.write_fasta(reads, recs)
        arms = {
            "X": Mapper(reads, None, preset="map-ont", cigar=False, all_vs_all=True),
            "X_c": Mapper(reads, None, preset="map-ont", all_vs_all=True),
            "P_noljoin": Mapper(reads, None, preset="map-ont", cigar=False),  # -X without the seed filter
        }
        arms["P_noljoin"].mo.flag |= F_ALL_CHAINS | F_NO_LJOIN
        for r in range(a.rounds + 1):  # round 0 warms every arm up
            for key, mp in arms.items():
                out = os.path.join(td, f"{key}.paf")
                mp.reset_stats()
                L.wm_prof_reset()
                t0 = time.perf_counter()
                mp.map_file(reads, out)
                dt = time.perf_counter() - t0
                prof = (C.c_double * 13)()
                L.wm_prof_get(prof)
                st = mp.stats()
                if r == 0:
                    continue
                n_lines = sum(1 for _ in open(out, "rb"))
                row = dict(mbase_s=round(n_bases / dt / 1e6, 2), t_seed_s=round(st["t_seed"], 3), n_chained=int(st["n_chained"]),
                           launches=int(prof[0]), lines=n_lines)
                res.setdefault(key, []).append(row)
                print(f"{key:10s} {dt:7.2f} s  {row['mbase_s']:7.2f} Mbase/s  seed {row['t_seed_s']:6.3f} s  chained anchors {row['n_chained']}"
                      f"  launches {row['launches']}  lines {n_lines}", flush=True)
        for mp in arms.values():
            mp.close()
        refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
        if a.ref_threads > 0 and os.path.exists(refbin):
            t0 = time.perf_counter()
            subprocess.run([refbin, "-t", str(a.ref_threads), "-x", "map-ont", "-X", reads, reads], stdout=subprocess.DEVNULL,
                           stderr=subprocess.DEVNULL, check=True)
            dt = time.perf_counter() - t0
            res["reference_X"] = dict(threads=a.ref_threads, cpus=os.cpu_count(), s=round(dt, 2), mbase_s=round(n_bases / dt / 1e6, 3))
            print(f"reference -X, {a.ref_threads} threads: {dt:7.2f} s  {n_bases / dt / 1e6:7.3f} Mbase/s", flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
