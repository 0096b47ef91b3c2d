#!/usr/bin/env python
"""--heap-sort=yes on one GPU: what the heap replay costs in the seed stage and in a whole mapping run.

  1. The seed stage alone (wm_seed_batch) on the crafted index of tests/heap_lib.py: one giant task (one query hash copied 2600
     times, > 10^5 anchors), one task whose heap lies in global memory and 2000 window-sized tasks cut from tandem reads, with
     and without heap sort.  Reported: tasks and anchors replayed, clocks of the merging lane per replayed anchor, the clocks of
     the giant task alone, and the wall time of the call (index upload included, the same in both arms).
  2. Mapper.map_file with and without heap_sort on the heap_tandem read set of tools/make_golden.py (300 ONT-like reads of
     2-20 kb from a short-unit tandem reference, -x map-ont -c) and all-vs-all on the same reads (-x map-ont -X -c).  Reported:
     Mbase/s, the seed stage's time (MapStats.t_seed) and the replay counters, alternating the arms over --rounds rounds after a
     warm-up round.

Prints one JSON object.  The card, its power limit and SM clock are read with nvidia-smi's query (read-only)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(("name", "power_limit", "sm_clock_now", "sm_clock_max"), [x.strip() for x in q.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def seed_stage():
    import heap_lib as H
    from winnowmap_b200 import kernels
    from test_gpu_heap import _big_tasks
    ix = H.Index()
    rng = np.random.default_rng(5)
    big = _big_tasks()
    windows = []
    for r in range(2000):
        s = ix.seqs[r % 4]
        st = int(rng.integers(0, len(s) - 2000))
        windows.append((ol_sketch(s[st:st + 2000]), 2000))
    out = {}
    for name, tasks in (("giant", [(big[1][1], big[1][2])]), ("global_heap", [(big[2][1], big[2][2])]), ("windows", windows)):
        row = {}
        for heap in (False, True):
            kernels.seed_heap_stats(reset=True)
            kernels.seed_batch(ix.keys, ix.pos_off, ix.pos, tasks, 5000, heap=heap)  # warm-up
            kernels.seed_heap_stats(reset=True)
            t0 = time.perf_counter()
            res = kernels.seed_batch(ix.keys, ix.pos_off, ix.pos, tasks, 5000, heap=heap)
            dt = time.perf_counter() - t0
            st = kernels.seed_heap_stats()
            row["heap" if heap else "sorted"] = dict(wall_ms=round(dt * 1e3, 2), anchors=int(sum(len(r[0]) for r in res)), **st)
        h = row["heap"]
        h["clocks_per_replayed_anchor"] = round(h["clocks"] / max(h["anchors"], 1), 1)
        out[name] = row
    return out


def ol_sketch(seq):
    import heap_lib as H
    import oracle_lib as ol
    return ol.oracle_sketch(seq, H.W, H.K, 0, None)


def mapping(rounds):
    import make_golden
    from winnowmap_b200 import kernels
    from winnowmap_b200.mapper import Mapper
    tmp = tempfile.mkdtemp(prefix="wm_bench_heap_")
    ref, reads = make_golden.make_heap_inputs("tandem", tmp)
    n_bases = sum(len(line.strip()) for line in open(reads) if not line.startswith(">"))
    out = {}
    for name, target, kw in (("ont_tandem", ref, {}), ("ava_tandem", reads, dict(all_vs_all=True))):
        mps = {hs: Mapper(target, None, preset="map-ont", heap_sort=hs, **kw) for hs in (False, True)}
        res = {False: [], True: []}
        for r in range(rounds + 1):
            for hs in (False, True):
                mp = mps[hs]
                mp.reset_stats()
                kernels.seed_heap_stats(reset=True)
                t0 = time.perf_counter()
                mp.map_file(reads, os.path.join(tmp, "o.paf"))
                dt = time.perf_counter() - t0
                if r:
                    res[hs].append(dict(mbase_s=round(n_bases / dt / 1e6, 3), t_seed_s=round(mp.stats()["t_seed"], 3), **kernels.seed_heap_stats()))
        for mp in mps.values():
            mp.close()
        out[name] = {"sorted" if not hs else "heap": v for hs, v in res.items()}
    out["bases"] = n_bases
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info(), seed_stage=seed_stage(), mapping=mapping(a.rounds), gpu_after=gpu_info())))


if __name__ == "__main__":
    main()
