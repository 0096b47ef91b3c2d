#!/usr/bin/env python
"""Times multi-part indexes (-I) and the -f selection on one GPU.

A tandem-enriched reference (gen_data.make_ref with tandem arrays, seed 1005, four contigs) of WM_PARTS_REF_LEN bases (1 Gbase
by default), indexed whole and cut into 2 and 4 parts (-I just below a half and a quarter of it: parts end at contig
boundaries), with the -W list counted on the GPU (distinct=0.9998).  ONT-like reads (seed 2005, N50 10 kb, 5 % error,
WM_PARTS_READ_BASES bases, 40 Mbase by default).  Reports, per configuration:
  - the index build time (host clock around the constructor, which ends in a device synchronise);
  - the map rate of wm_map_file, part-major and merged (--split-prefix), in read bases per second, after a warm-up pass;
  - the peak device memory in use over the build and the passes (sampled every 5 ms), against the single index;
and for the single index and for each part of the 4-part index the time of wm_idx_cal_max_occ (each call a new f, so nothing
is cached) against numpy's introselect (np.partition, the host nth_element) over the same counts, both the mean of 5 calls.
The card's name and power limit are read in the same run.  Prints one JSON line."""
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import gen_data  # noqa: E402
from winnowmap_b200 import lib  # noqa: E402
from winnowmap_b200.mapper import Mapper, _setup  # noqa: E402

REF_LEN = int(os.environ.get("WM_PARTS_REF_LEN", 1_000_000_000))
READ_BASES = int(os.environ.get("WM_PARTS_READ_BASES", 40_000_000))


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


def counts_of(L, ctx):
    """The occurrence count of every key of one index, from its fan-out blob (header: n_seq, names bytes, S words, n_keys)."""
    n = L.wm_idx_blob_size(ctx)
    buf = np.empty(n, np.uint8)
    L.wm_idx_blob_write(ctx, buf.ctypes.data)
    h = buf[:64].view(np.uint64)
    n_seq, names, s_words, n_keys = (int(x) for x in h[2:6])
    pad8 = lambda x: (x + 7) & ~7  # noqa: E731
    o = 64 + pad8(n_seq * 4) + n_seq * 8 + pad8(names) + pad8(s_words * 4) + n_keys * 8
    pos_off = buf[o:o + (n_keys + 1) * 8].view(np.uint64)
    return np.diff(pos_off).astype(np.uint32)


def time_select(L, part, counts, reps=5):
    dev, host = [], []
    for i in range(reps):
        f = 0.0002 + 1e-7 * i  # a new f each call: the per-f cache does not answer
        t0 = time.perf_counter()
        v = L.wm_idx_cal_max_occ(part, f)
        dev.append(time.perf_counter() - t0)
        rank = int((1.0 - np.float32(f).item()) * len(counts))
        t0 = time.perf_counter()
        w = int(np.partition(counts, rank)[rank]) + 1
        host.append(time.perf_counter() - t0)
        assert v == w, (v, w)
    return {"n_keys": len(counts), "device_ms": round(1e3 * np.mean(dev), 2), "host_nth_element_ms": round(1e3 * np.mean(host), 2)}


def main():
    L = _setup(lib())
    L.wm_device_mem.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.wm_idx_blob_size.argtypes = [C.c_void_p]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    res = {"ref_len": REF_LEN, "read_bases": READ_BASES, "gpu": gpu[0] if gpu else None}
    with tempfile.TemporaryDirectory() as td:
        t0 = time.time()
        contigs = gen_data.make_ref(np.random.default_rng(1005), REF_LEN, 4, True)
        ref, reads = os.path.join(td, "ref.fa"), os.path.join(td, "reads.fa")
        gen_data.write_fasta(ref, contigs)
        rng = np.random.default_rng(2005)
        n_reads = max(1, READ_BASES // 9000)
        recs = gen_data.make_reads(rng, contigs, n_reads, 10000, 0.05, min_len=1000)
        gen_data.write_fasta(reads, recs)
        res["read_bases"] = int(sum(len(s) for _, s in recs))
        del contigs, recs
        res["gen_s"] = round(time.time() - t0, 1)
        configs = {"1": None, "2": REF_LEN // 2 - 1, "4": REF_LEN // 4 - 1}
        for name, part_bases in configs.items():
            peak = PeakMem(L)
            t0 = time.time()
            kw = {} if part_bases is None else {"part_bases": part_bases}
            mp = Mapper(ref, preset="map-ont", distinct=0.9998, **kw)
            L.wm_device_synchronize()
            r = {"n_parts": mp.n_parts, "build_s": round(time.time() - t0, 2)}
            out = os.path.join(td, "out.paf")
            for mode, split in (("part_major", False), ("merged", True)):
                if part_bases is None and mode == "part_major":
                    mode = "single"
                mp.mo.split_prefix = b"x" if split else None
                mp.map_file(reads, out)  # warm-up
                t0 = time.time()
                mp.map_file(reads, out)
                dt = time.time() - t0
                r[f"{mode}_s"] = round(dt, 2)
                r[f"{mode}_mbase_per_s"] = round(res["read_bases"] / dt / 1e6, 1)
            r["peak_device_mem_gb"] = round(peak.close() / 1e9, 2)
            if part_bases is None:
                r["cal_max_occ"] = time_select(L, mp.ctx, counts_of(L, mp.ctx))
            elif name == "4":
                r["cal_max_occ_parts"] = [time_select(L, L.wm_idx_part(mp.ctx, i), counts_of(L, L.wm_idx_part(mp.ctx, i))) for i in range(mp.n_parts)]
            mp.close()
            res[f"parts_{name}"] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
