/* TEST INFRASTRUCTURE ONLY: the -W list restated in plain C, the oracle of the device's wm_topfreq for every k.
 * What `meryl count k=K` followed by `meryl print greater-than distinct=D` selects:
 *   1. every canonical k-mer of every sequence (a k-mer never spans two sequences, any base outside ACGTacgt breaks it;
 *      canonical: the smaller of the forward and reverse-complement codes, A0 C1 G2 T3, first base in the high bits, as
 *      encodeKmer, src/index.c:362-376), collected and sorted; runs are the counts;
 *   2. ext/meryl/src/meryl/merylOp-nextMer.C:103-115: nKmersTarget = (uint64)(D * numDistinct); the count values that
 *      occur, ascending, accumulate their occurrences; the threshold is the first value at which the sum is >= the target;
 *   3. the k-mers whose count is greater than the threshold (greater-than), ascending.
 * Compiled by the tests themselves (tests/topfreq_lib.py); nothing in the product links it. */
#include <stdint.h>
#include <stdlib.h>

static int cmp_u64(const void *a, const void *b)
{
	const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
	return x < y ? -1 : x > y;
}

static int base_code(unsigned char c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; }
}

/* seq: the sequences concatenated, sequence i = seq[off[i] .. off[i + 1]).  Returns the list's length (-1: out of memory);
 * up to cap entries into kmers / counts; the threshold into *threshold and the number of distinct k-mers into *n_distinct. */
int64_t wm_oracle_topfreq(const char *seq, const int64_t *off, int n_seq, int k, double distinct, uint64_t *kmers, uint32_t *counts, int64_t cap,
                          uint64_t *threshold, int64_t *n_distinct)
{
	const uint64_t mask = k < 32 ? (1ULL << 2 * k) - 1 : ~0ULL, shift = 2 * (uint64_t)(k - 1);
	uint64_t *all = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(off[n_seq] + 1));
	int64_t n = 0, i, j, nd = 0, m = 0;
	if (!all) return -1;
	for (i = 0; i < n_seq; ++i) { /* 1. collect */
		uint64_t fw = 0, rv = 0; int l = 0;
		for (j = off[i]; j < off[i + 1]; ++j) {
			const int c = base_code((unsigned char)seq[j]);
			if (c > 3) { l = 0; continue; }
			fw = (fw << 2 | (uint64_t)c) & mask;
			rv = rv >> 2 | (uint64_t)(3 - c) << shift;
			if (++l >= k) all[n++] = fw < rv ? fw : rv;
		}
	}
	qsort(all, (size_t)n, sizeof(uint64_t), cmp_u64);
	/* runs: code all[r], count cnt[r] */
	uint64_t *cnt = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(n + 1)), *vals = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(n + 1));
	if (!cnt || !vals) { free(all); free(cnt); free(vals); return -1; }
	for (i = 0; i < n; i = j) {
		for (j = i; j < n && all[j] == all[i]; ++j) {}
		all[nd] = all[i], cnt[nd] = (uint64_t)(j - i), ++nd;
	}
	/* 2. the histogram of counts (values that occur, ascending) and meryl's rule */
	for (i = 0; i < nd; ++i) vals[i] = cnt[i];
	qsort(vals, (size_t)nd, sizeof(uint64_t), cmp_u64);
	const uint64_t target = (uint64_t)(distinct * (double)nd);
	uint64_t thr = 0, acc = 0;
	for (i = 0; i < nd; i = j) {
		for (j = i; j < nd && vals[j] == vals[i]; ++j) {}
		acc += (uint64_t)(j - i); /* histogramOccurrences of value vals[i] */
		if (acc >= target) { thr = vals[i]; break; }
	}
	/* 3. select */
	for (i = 0; i < nd; ++i)
		if (cnt[i] > thr) { if (m < cap) kmers[m] = all[i], counts[m] = (uint32_t)cnt[i]; ++m; }
	*threshold = thr, *n_distinct = nd;
	free(all); free(cnt); free(vals);
	return m;
}
