#!/usr/bin/env python
"""Spliced mapping (-x splice -W, no base alignment) on a generated transcriptome (tools/gen_data.py make_transcriptome).

  python tools/bench_splice.py [--genome 20000000] [--genes 600] [--reads 20000] [--threads N] [--align c|a]

Prints one line per figure:
  map_file        Mapper.map_file rate over the whole read set, after a warm-up on a slice of it (GPU required; no CPU fallback)
  chain_kernels   the chaining class's kernel time over that run, from the library's per-class CUDA events (wm_prof_get)
  giant_tasks     on the host, for a sample of reads: the stage-2 seed hits of each read (the oracle's sketch and index lookup on the
                  same -W filter), how many tasks exceed the giant-task size (2048 anchors) and how many of their anchors have a
                  window (src/chain.c:49-55) that reaches more than 4096 anchors back, below the tile kernel's ring
  reference       the reference binary (oracle/_ref/winnowmap, when built) on the same inputs and thread count
With --align c (or a), the runs are -c (or -a) through Mapper(..., spliced_alignment=True): the DP is ksw_exts2 on the GPU;
map_file then also reports the number of DP and ll jobs, and the reference line whether the outputs are byte-identical (SAM:
but for the @PG line).
Everything is written to a temporary directory."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen_data  # noqa: E402

TILE_MIN, RING = 2048, 4096


def window_starts(x, max_dist_x, min_dist_x, max_iter):
    """st[i] of src/chain.c:49-55 in closed form (csrc/chain_dev.cuh wm_chain_window_start)."""
    i = np.arange(len(x))
    lb = lambda d: np.searchsorted(x, np.where(x >= np.uint64(d), x - np.uint64(d), np.uint64(0)), side="left")  # first s: x[s] + d >= x[i]
    lb_max, lb_min = lb(max_dist_x), lb(min_dist_x)
    return np.maximum(lb_max, np.minimum(i - max_iter, lb_min)), i


def giant_stats(ref_fa, reads, wfile, n_sample, io, mo):
    import oracle_lib as ol
    kmers = [ln.split()[0] for ln in open(wfile)]
    bloom = ol.OracleBloom([ol.oracle().wmo_encode_kmer(k.encode(), len(k)) for k in kmers]) if kmers else None
    mz = np.concatenate([ol.oracle_sketch(s.tobytes(), io.w, io.k, rid, bloom) for rid, (_, s) in enumerate(gen_data.read_fasta(ref_fa))])
    idx = ol.OracleIndex(mz)
    max_gap_ref = mo.max_gap_ref if mo.max_gap_ref > 0 else mo.max_gap
    n_tasks = n_giant = n_anchors_giant = n_deep = 0
    for _, s in reads[:n_sample]:
        mv = ol.oracle_sketch(s.tobytes(), io.w, io.k, 0, bloom)
        a, _, _ = idx.seed_hits(mv, len(s), mo.mid_occ)
        n_tasks += 1
        if len(a) <= TILE_MIN:
            continue
        n_giant += 1
        n_anchors_giant += len(a)
        # both strands form one sorted array, as in the mapper (bit 63 of x is the strand)
        st, i = window_starts(np.ascontiguousarray(a[:, 0], dtype=np.uint64), max_gap_ref, min(mo.min_gap_ref, max_gap_ref), mo.max_chain_iter)
        n_deep += int((st < i - RING).sum())
    return n_tasks, n_giant, n_anchors_giant, n_deep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome", type=int, default=20_000_000)
    ap.add_argument("--genes", type=int, default=600)
    ap.add_argument("--reads", type=int, default=20000)
    ap.add_argument("--threads", type=int, default=min(32, os.cpu_count() or 1))
    ap.add_argument("--sample", type=int, default=400)
    ap.add_argument("--align", choices=("c", "a"), default=None)
    a = ap.parse_args()
    from winnowmap_b200 import lib
    from winnowmap_b200.mapper import Mapper
    td = tempfile.mkdtemp(prefix="wm_bench_splice_")
    rng = np.random.default_rng(61)
    contigs, tx = gen_data.make_transcriptome(rng, a.genome, a.genes, n_contigs=4, long_introns=8, long_genes=20)
    recs = gen_data.make_spliced_reads(rng, contigs, tx, a.reads, 0.06, a.reads // 20, a.reads // 200)
    ref, reads, wfile, warm = (os.path.join(td, x) for x in ("ref.fa", "reads.fa", "rep.txt", "warm.fa"))
    gen_data.write_fasta(ref, contigs)
    gen_data.write_fasta(reads, recs)
    gen_data.write_fasta(warm, recs[:1000])
    gen_data.write_top_kmers(wfile, contigs, 15, 0.9998)
    bases = sum(len(s) for _, s in recs)
    print(f"inputs: genome {a.genome / 1e6:.1f} Mbase, {len(tx)} transcripts, {len(recs)} reads, {bases / 1e6:.1f} Mbase", flush=True)
    L = lib()
    L.wm_prof_get.argtypes = [C.POINTER(C.c_double)]
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip()
        print(f"device: {smi}")
    except Exception:
        print("device: nvidia-smi unavailable")
    mp = Mapper(ref, wfile, preset="splice", cigar=a.align is not None, sam=a.align == "a", n_threads=a.threads, spliced_alignment=True)
    out = os.path.join(td, "out.paf")
    mp.map_file(warm, os.path.join(td, "warm.paf"))
    mp.reset_stats()
    L.wm_prof_enable(1); L.wm_prof_reset()
    t0 = time.perf_counter()
    mp.map_file(reads, out)
    t = time.perf_counter() - t0
    prof = (C.c_double * 13)(); L.wm_prof_get(prof)
    L.wm_prof_enable(0)
    n_lines = sum(1 for _ in open(out))
    st = mp.stats()
    print(f"map_file: {t:.2f} s, {bases / t / 1e6:.2f} Mbase/s, {n_lines} output lines"
          + (f", {int(st['n_dp_jobs'])} DP jobs, {int(st['n_ll_jobs'])} ll jobs, DP rounds {st['t_dp']:.2f} s" if a.align else ""))
    ms_sum, ms_uni, n_l = prof[1 + 6], prof[2 + 6], prof[3 + 6]
    print(f"chain_kernels: {ms_uni if ms_uni > 0 else ms_sum:.1f} ms over {int(n_l)} launches ({ms_sum:.1f} ms summed over launches)")
    n_tasks, n_giant, n_ag, n_deep = giant_stats(ref, recs, wfile, a.sample, mp.io, mp.mo)
    print(f"giant_tasks: {n_giant} of {n_tasks} sampled reads have more than {TILE_MIN} anchors; {n_deep} of their {n_ag} anchors have "
          f"a window reaching more than {RING} anchors back")
    mp.close()
    refbin = os.path.join(ROOT, "oracle", "_ref", "winnowmap")
    if os.path.exists(refbin):
        t0 = time.perf_counter()
        got = subprocess.run([refbin, "-t", str(a.threads), "-x", "splice"] + (["-" + a.align] if a.align else []) + ["-W", wfile, ref, reads],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True).stdout
        tr = time.perf_counter() - t0
        print(f"reference: {tr:.2f} s, {bases / tr / 1e6:.2f} Mbase/s with {a.threads} threads (index build included)")
        if a.align:
            import make_golden
            mine = open(out, "rb").read()
            same = make_golden.sam_without_pg(mine) == make_golden.sam_without_pg(got) if a.align == "a" else mine == got
            print(f"identical: {same}")
    else:
        print("reference: oracle/_ref/winnowmap not built")


if __name__ == "__main__":
    main()
