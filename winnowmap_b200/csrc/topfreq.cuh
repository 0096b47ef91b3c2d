// The repetitive k-mer list of -W computed on the device (topfreq.cu): what `meryl count k=K` followed by
// `meryl print greater-than distinct=D` lists for a FASTA (ext/meryl/src/meryl/merylOp-nextMer.C:103-115), as the canonical
// codes encodeKmer (reference src/index.c:362-376) gives each line of such a list.
//
// The two device functions below read a packed pool (pkseq.cuh) and compile on the host as well (tests/hostsim/topfreq_emul.cpp).
#pragma once
#include "pkseq.cuh"

// canonical code of the k bases from base b (the smaller of the forward and reverse-complement codes, first base in the high
// bits: encodeKmer's value for that spelling); false when one of the k bases is ambiguous
__device__ __forceinline__ bool wm_tf_kmer(const uint32_t *__restrict__ pk, const uint32_t *__restrict__ nm, int64_t b, int k, uint64_t *code)
{
	uint64_t fw, rv;
	wm_pk_kmer(wm_pk_window(pk, b), k, &fw, &rv);
	*code = fw < rv ? fw : rv;
	return (wm_pk_nwindow(nm, b) & (uint32_t)((1ULL << k) - 1)) == 0;
}

// Bit j of the result: the k-mer at base p0 + j (p0 a multiple of 32) lies inside one task and has no ambiguous base.  The
// tasks are consecutive slices of the pool, task t = bases [off[t], off[t + 1]), off[n_tasks] = n_bases: a k-mer never spans
// two sequences.
__device__ __forceinline__ uint32_t wm_tf_valid32(const uint32_t *__restrict__ nm, const int64_t *__restrict__ off, int n_tasks, int k, int64_t p0)
{
	const int64_t n_bases = off[n_tasks];
	int lo = 0, hi = n_tasks; // the last task with off[t] <= p0
	while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (off[m] <= p0) lo = m; else hi = m; }
	int t = lo;
	int64_t end = off[t + 1];
	// ambiguity flags of bases p0 .. p0 + 63: a k-mer starting in the first 32 ends by base 58 (k <= 28)
	const uint64_t amb = (uint64_t)wm_pk_nwindow(nm, p0) | (uint64_t)wm_pk_nwindow(nm, p0 + 32) << 32, km = (1ULL << k) - 1;
	uint32_t v = 0;
	for (int j = 0; j < 32 && p0 + j < n_bases; ++j) {
		while (p0 + j >= end) end = off[++t + 1];
		if (p0 + j + k <= end && (amb >> j & km) == 0) v |= 1u << j;
	}
	return v;
}

#ifndef WM_HOST_EMUL
#include <vector>
#include <cuda_runtime.h>

// one packed pool: n_tasks sequences, task t = bases [d_off[t], d_off[t + 1]) (device array of n_tasks + 1 offsets)
struct wm_tf_group { const uint32_t *pk, *nm; const int64_t *d_off; int n_tasks; };
// the list: canonical codes ascending, their counts, the threshold they are above, the number of distinct k-mers counted
struct wm_tf_list { std::vector<uint64_t> codes; std::vector<uint32_t> counts; uint64_t threshold; int64_t n_distinct; };
// counts the canonical k-mers of every task of the groups (1 <= k <= 28) and selects those above the meryl threshold for
// `distinct`; all scratch is freed on return
void wm_topfreq_dev(const std::vector<wm_tf_group> &groups, int k, double distinct, wm_tf_list *out, cudaStream_t st);
#endif
