"""Junction annotation (--junc-bed) in spliced base-level alignment: the transcriptome of tools/bench_splice.py mapped with
-x splice -c, with and without a BED of all its transcripts.  Reports
  junc_kernel_ms   the annotation kernel's CUDA-event time over one profiled run, and its share of the DP fill's time there
  mbase_s          map_file throughput with and without the BED, two alternated rounds after one warm-up run of each
  gpu              the card name and power limit, read in this call.
Prints one JSON line."""
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
import make_golden  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome", type=int, default=5_000_000)
    ap.add_argument("--genes", type=int, default=150)
    ap.add_argument("--reads", type=int, default=3000)
    ap.add_argument("--threads", type=int, default=min(32, os.cpu_count() or 1))
    a = ap.parse_args()
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import Mapper, _setup
    L = _setup(lib())
    L.wm_prof_enable.argtypes = [C.c_int]
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    td = tempfile.mkdtemp(prefix="wm_bench_junc_")
    rng = np.random.default_rng(61)  # the transcriptome of tools/bench_splice.py at these sizes
    layout = []
    contigs, tx = gen_data.make_transcriptome(rng, a.genome, a.genes, n_contigs=4, long_introns=8, long_genes=20, layout=layout)
    recs = gen_data.make_spliced_reads(rng, contigs, tx, a.reads, 0.06, a.reads // 20, a.reads // 200)
    ref, reads, wfile, bed = (os.path.join(td, x) for x in ("ref.fa", "reads.fa", "rep.txt", "tx.bed"))
    gen_data.write_fasta(ref, contigs)
    gen_data.write_fasta(reads, recs)
    gen_data.write_top_kmers(wfile, contigs, 15, 0.9998)
    with open(bed, "w") as f:
        for n, ch, sd, ex in layout:
            f.write(make_golden._bed12(n, ch, sd, ex, 0) + "\n")
    bases = sum(len(r[1]) for r in recs)
    mps = {False: Mapper(ref, wfile, preset="splice", cigar=True, spliced_alignment=True, n_threads=a.threads),
           True: Mapper(ref, wfile, preset="splice", cigar=True, spliced_alignment=True, n_threads=a.threads, junc_bed=bed)}
    o3 = (C.c_double * 3)()
    # one profiled run with the BED: the annotation kernel against the DP fill
    L.wm_prof_enable(1); L.wm_prof_reset(); L.wm_junc_stats(o3, 1)
    mps[True].map_file(reads, os.path.join(td, "p.paf"))
    prof = (C.c_double * 13)(); L.wm_prof_get(prof); L.wm_junc_stats(o3, 1)
    L.wm_prof_enable(0)
    junc_ms, fill_ms = o3[2], prof[1]
    rates = {False: [], True: []}
    for rnd in range(3):  # round 0 warms up
        for with_bed in (False, True):
            t0 = time.perf_counter()
            mps[with_bed].map_file(reads, os.path.join(td, f"o{int(with_bed)}.paf"))
            dt = time.perf_counter() - t0
            if rnd > 0:
                rates[with_bed].append(bases / dt / 1e6)
    same = open(os.path.join(td, "o0.paf"), "rb").read() == open(os.path.join(td, "o1.paf"), "rb").read()
    for m in mps.values():
        m.close()
    print(json.dumps(dict(gpu=gpu_info(), reads=len(recs), mbases=bases / 1e6, intervals=sum(len(x[3]) - 1 for x in layout),
                          junc_launches=o3[0], junc_windows=o3[1], junc_kernel_ms=round(junc_ms, 3), dp_fill_ms=round(fill_ms, 3),
                          junc_share_of_fill=round(junc_ms / fill_ms, 5) if fill_ms > 0 else None,
                          mbase_s_without_bed=[round(x, 2) for x in rates[False]], mbase_s_with_bed=[round(x, 2) for x in rates[True]],
                          outputs_differ=not same)))


if __name__ == "__main__":
    main()
