/* TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
 *
 * The junction annotation of one DP target window (mm_idx_bed_junc, reference src/index.c:780-803), restated from what it
 * computes: for the window [st, en) of one sequence whose intervals a[0..n) are sorted by start, byte p of s is 0 but for
 *   bit 1 / 2  at the first / last base of every + strand interval inside the window,
 *   bit 8 / 4  at the first / last base of every - strand interval inside the window,
 * where "inside" is st <= a.st and a.en <= en, and intervals without a strand mark nothing.  Returns the index of the first
 * interval with a.st >= st (n when there is none).  The record layout is that of mm_idx_intv1_t. */
#include <stdint.h>
#include <string.h>

typedef struct {
	int32_t st, en, max;
	int32_t score:30, strand:2;
} wmo_intv1_t;

int wmo_bed_junc(const wmo_intv1_t *a, int n, int32_t st, int32_t en, uint8_t *s)
{
	int first = n, i;
	memset(s, 0, (size_t)(en - st));
	for (i = 0; i < n; ++i)
		if (a[i].st >= st) { if (i < first) first = i; }
	for (i = 0; i < n; ++i) {
		if (a[i].st < st || a[i].en > en || a[i].strand == 0) continue;
		if (a[i].strand > 0) s[a[i].st - st] |= 1, s[a[i].en - 1 - st] |= 2;
		else s[a[i].st - st] |= 8, s[a[i].en - 1 - st] |= 4;
	}
	return first;
}

/* the same bytes in reverse order (mm_seq_rev after the left extension's call, src/align.c:693-694) */
int wmo_bed_junc_rev(const wmo_intv1_t *a, int n, int32_t st, int32_t en, uint8_t *s)
{
	const int r = wmo_bed_junc(a, n, st, en, s);
	int32_t i, l = en - st;
	for (i = 0; i < l >> 1; ++i) { const uint8_t t = s[i]; s[i] = s[l - 1 - i]; s[l - 1 - i] = t; }
	return r;
}
