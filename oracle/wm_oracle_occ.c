/* TEST INFRASTRUCTURE ONLY.  A plain-C restatement of mm_idx_cal_max_occ (reference src/index.c:173-194) over the
 * occurrence counts of an index's keys (a singleton counts 1): INT32_MAX for f <= 0, else the k-th smallest count plus one
 * with k = (uint32_t)((1. - f) * n).  Where k reaches n the reference reads past its array; this returns -1 there. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int cmp_u32(const void *a, const void *b)
{
	const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
	return x < y ? -1 : x > y;
}

int32_t wm_oracle_cal_max_occ(const uint32_t *counts, int64_t n, float f)
{
	uint32_t k, v, *a;
	if (f <= 0.) return INT32_MAX;
	k = (uint32_t)((1. - f) * (size_t)n);
	if ((int64_t)k >= n) return -1;
	a = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
	memcpy(a, counts, sizeof(uint32_t) * (size_t)n);
	qsort(a, (size_t)n, sizeof(uint32_t), cmp_u32); /* any order statistic of a sorted copy is the selection's */
	v = a[k];
	free(a);
	return (int32_t)(v + 1);
}
