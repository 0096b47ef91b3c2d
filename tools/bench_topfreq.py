#!/usr/bin/env python
"""Times the -W list counted on the GPU (wm_topfreq, wm_index_build_topfreq) on the bench's tandem-repeat reference.

The reference is bench.py's: seed 1005, gen_data.make_ref with tandem arrays, one contig per 250 Mbp, 500 Mbp unless
WM_TOPFREQ_REF_LEN says otherwise (3000000000: a human-sized reference, to show that the partitions hold).  Reports:
  - wm_topfreq for k = 15 and k = 19: host clock around one call (which ends in a device synchronise), after a warm-up call;
  - the CPU stand-in (tools/wm_tools.c on all host threads, k = 15) for comparison;
  - wm_index_build_opt from the stand-in's file against wm_index_build_topfreq, alternated over two rounds;
  - the peak device memory in use during the calls (sampled every 5 ms);
  - the card's name and power limit, read in the same run.
Prints one JSON line."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_data  # noqa: E402
from winnowmap_b200.mapper import Mapper, _setup, make_options  # noqa: E402
from winnowmap_b200 import lib  # noqa: E402

REF_LEN = int(os.environ.get("WM_TOPFREQ_REF_LEN", 500_000_000))


class PeakMem:
    def __init__(self, L):
        self.L, self.used, self.stop = L, 0.0, False
        f, t = C.c_double(), C.c_double()
        L.wm_device_mem(C.byref(f), C.byref(t))
        self.base = t.value - f.value
        self.th = threading.Thread(target=self.run, daemon=True)
        self.th.start()

    def run(self):
        f, t = C.c_double(), C.c_double()
        while not self.stop:
            self.L.wm_device_mem(C.byref(f), C.byref(t))
            self.used = max(self.used, t.value - f.value)
            time.sleep(0.005)

    def close(self):
        self.stop = True
        self.th.join()
        return self.used - self.base


def main():
    L = _setup(lib())
    L.wm_device_mem.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    res = {"ref_len": REF_LEN, "gpu": gpu[0] if gpu else None}
    with tempfile.TemporaryDirectory() as td:
        t0 = time.time()
        contigs = gen_data.make_ref(np.random.default_rng(1005), REF_LEN, max(1, round(REF_LEN / 250_000_000)), True)
        ref = os.path.join(td, "ref.fa")
        gen_data.write_fasta(ref, contigs)
        res["gen_s"] = round(time.time() - t0, 1)
        t0 = time.time()
        wfile = os.path.join(td, "rep.txt")
        n_sd, thr_sd = gen_data.write_top_kmers(wfile, contigs, 15, 0.9998)
        res["stand_in_k15_s"] = round(time.time() - t0, 2)
        res["stand_in_k15"] = {"n": n_sd, "threshold": thr_sd, "host_threads": os.cpu_count()}
        del contigs
        peak = PeakMem(L)
        for k in (15, 19):
            thr = C.c_uint64(0)
            L.wm_topfreq(ref.encode(), k, 0.9998, None, None, 0, C.byref(thr), 0)  # warm-up
            t0 = time.time()
            n = L.wm_topfreq(ref.encode(), k, 0.9998, None, None, 0, C.byref(thr), 0)
            res[f"wm_topfreq_k{k}_s"] = round(time.time() - t0, 3)
            res[f"wm_topfreq_k{k}"] = {"n": n, "threshold": thr.value}
        res["peak_device_mem_topfreq_gb"] = round(peak.close() / 1e9, 2)
        io, _ = make_options("map-ont")
        rounds = {"file": [], "topfreq": []}
        peak = PeakMem(L)
        for _ in range(2):
            for kind in ("file", "topfreq"):
                t0 = time.time()
                mp = Mapper(ref, wfile) if kind == "file" else Mapper(ref, distinct=0.9998)
                L.wm_device_synchronize()
                rounds[kind].append(round(time.time() - t0, 2))
                if kind == "topfreq":
                    st = mp.stats()
                    res["index_topfreq_stats"] = {k: st[k] for k in ("n_topfreq", "topfreq_threshold", "t_topfreq", "t_index")}
                mp.close()
        res["peak_device_mem_index_gb"] = round(peak.close() / 1e9, 2)
        res["index_build_file_s"], res["index_build_topfreq_s"] = rounds["file"], rounds["topfreq"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
