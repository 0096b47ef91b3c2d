#!/usr/bin/env python
"""Ad-hoc GPU-vs-reference comparison on a generated dataset (used for tuning / robustness checks on the GPU box):
   python tools/run_compare.py --len 3400000 --tandem --reads 600 --n50 12000 [--preset map-ont]
prints both mapping times and whether the PAF outputs are byte-identical (needs oracle/_ref/winnowmap).
With --cli the same argv (-t, -x, -W, --cli-args, ref, reads) goes to the reference and to winnowmap_b200/winnowmap-b200, run
from the dataset's directory with relative file names, and the Python API's Mapper.map_file is timed on the same run:
   python tools/run_compare.py --len 20000000 --tandem --reads 2000 --n50 30000 --cli --cli-args "-c"  (or "-a")"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

import gen_data  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--len", type=int, default=3_400_000)
    ap.add_argument("--contigs", type=int, default=1)
    ap.add_argument("--tandem", action="store_true")
    ap.add_argument("--reads", type=int, default=600)
    ap.add_argument("--n50", type=int, default=12000)
    ap.add_argument("--err", type=float, default=0.05)
    ap.add_argument("--preset", default="map-ont")
    ap.add_argument("-k", type=int, default=15)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--out", default="/tmp/wm_cmp")
    ap.add_argument("--repeat", action="store_true", help="map a second time and report the warm timing")
    ap.add_argument("--cli", action="store_true", help="compare the command lines: the reference's and winnowmap-b200")
    ap.add_argument("--cli-args", default="-c", help="output options of --cli (split on spaces)")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    rng = np.random.default_rng(1005)
    contigs = gen_data.make_ref(rng, a.len, a.contigs, a.tandem)
    ref, reads, wf = [os.path.join(a.out, x) for x in ("ref.fa", "reads.fa", "rep.txt")]
    gen_data.write_fasta(ref, contigs)
    n, thr = gen_data.write_top_kmers(wf, contigs, a.k, 0.9998)
    recs = gen_data.make_reads(np.random.default_rng(2005), contigs, a.reads, a.n50, a.err, min_len=1000)
    gen_data.write_fasta(reads, recs)
    nb = sum(len(s) for _, s in recs)
    print(f"dataset: {a.len} bp ref, {a.reads} reads, {nb / 1e6:.1f} Mbase, -W list {n} k-mers (> {thr})", flush=True)
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if a.cli:
        return compare_cli(a, refbin, nb)
    t0 = time.time()
    with open(os.path.join(a.out, "ref.paf"), "wb") as f:
        subprocess.run([refbin, "-t", str(a.threads), "-c", "-x", a.preset, "-W", wf, ref, reads], stdout=f, stderr=subprocess.DEVNULL, check=True)
    t_ref = time.time() - t0
    from winnowmap_b200.mapper import Mapper
    t0 = time.time()
    mp = Mapper(ref, wf, preset=a.preset, cigar=True)
    t_idx = time.time() - t0
    t0 = time.time()
    mp.map_file(reads, os.path.join(a.out, "gpu.paf"))
    t_gpu = time.time() - t0
    t_warm = None
    if a.repeat:  # steady state: buffers allocated, CUDA context warm
        from winnowmap_b200 import lib
        if os.environ.get("WM_TIMING"):
            print("--- first pass timers ---", file=sys.stderr, flush=True)
            lib().wm_dump_timers()
        t0 = time.time()
        mp.map_file(reads, os.path.join(a.out, "gpu2.paf"))
        t_warm = time.time() - t0
    st = mp.stats()
    same = open(os.path.join(a.out, "ref.paf"), "rb").read() == open(os.path.join(a.out, "gpu.paf"), "rb").read()
    print(f"reference (index+map, {a.threads} threads): {t_ref:.2f}s | gpu index {t_idx:.2f}s map {t_gpu:.2f}s ({nb / t_gpu / 1e6:.1f} Mbase/s) | identical: {same}")
    if t_warm is not None:
        print(f"gpu map, second pass (warm): {t_warm:.2f}s ({nb / t_warm / 1e6:.1f} Mbase/s)")
    print({k: round(v, 3) for k, v in st.items()})
    if os.environ.get("WM_TIMING"):
        from winnowmap_b200 import lib
        lib().wm_dump_timers()


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def compare_cli(a, refbin, nb):
    argv = ["-t", str(a.threads), "-x", a.preset, "-W", "rep.txt"] + a.cli_args.split() + ["ref.fa", "reads.fa"]
    exe = os.path.join(ROOT, "winnowmap_b200", "winnowmap-b200")
    times, outs = {}, {}
    for name, binary in (("reference", refbin), ("winnowmap-b200", exe)):
        t0 = time.time()
        outs[name] = subprocess.run([binary] + argv, cwd=a.out, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout
        times[name] = time.time() - t0
    from winnowmap_b200.mapper import Mapper
    t0 = time.time()
    mp = Mapper(os.path.join(a.out, "ref.fa"), os.path.join(a.out, "rep.txt"), preset=a.preset, cigar=True, sam="-a" in a.cli_args.split(),
                n_threads=a.threads)
    mp.map_file(os.path.join(a.out, "reads.fa"), os.path.join(a.out, "api.out"))
    mp.close()
    t_api = time.time() - t0
    print(f"GPU: {gpu_name()}")
    print(f"argv: winnowmap {' '.join(argv)}")
    print(f"reference {times['reference']:.2f}s | winnowmap-b200 {times['winnowmap-b200']:.2f}s (index + map, process start to exit) | "
          f"Mapper index + map_file {t_api:.2f}s | identical: {outs['reference'] == outs['winnowmap-b200']} | {nb / 1e6:.1f} Mbase")


if __name__ == "__main__":
    main()
