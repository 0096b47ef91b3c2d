// TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
//
// Symmetric DUST (SDUST; Morgulis et al., J. Comput. Biol. 13:1028, 2006) as Winnowmap 2.03 runs it with -T, restated in plain
// C from the algorithm, and the minimizer squeeze that follows it in the mapper.  The tests pin both against the reference's own
// functions (oracle/ref_harness_sdust.cpp) and the device code against these.
//
// The scan keeps a window of the last W - 2 triplets of the sequence and, for its "valid suffix" (the longest suffix in which no
// triplet occurs more than 2T/10 times), the triplet counts cv and the score rv = sum over triplets of C(cv, 2); rw is the same
// score over the whole window.  Whenever rw * 10 > L * T, every suffix of the window that reaches past the valid suffix is scored
// and the "perfect" ones (score * 10 > T * length, and no smaller score ratio than any perfect interval they contain) are
// recorded in P, which is kept sorted by descending start, then ascending finish.  Intervals of P that fall out of the window
// are merged into the result.  A base outside ACGT ends a piece: the intervals still pending are flushed; the window itself,
// its counts and scores carry over into the next piece, as in the reference.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { int start, finish, r, l; } wmo_perf_t;

typedef struct {
	int W, T;
	int *win; int head, n; // ring of triplets, oldest at head
	int L, rw, rv, cw[64], cv[64];
	wmo_perf_t *P; int nP, mP;
	uint64_t *res; long n_res, m_res;
	int max_nP; // the largest P seen (tests size the device's list with it)
} wmo_sdust_t;

static inline int wmo_sd_nt4(unsigned char c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2;
	             case 'T': case 't': case 'U': case 'u': return 3; default: return c < 4 ? c : 4; }
}

static inline int wmo_sd_at(const wmo_sdust_t *s, int i) { return s->win[(s->head + i) % (s->W - 2)]; }

static void wmo_sd_emit(wmo_sdust_t *s, int st, int fi)
{
	if (s->n_res && st <= (int)(uint32_t)s->res[s->n_res - 1]) { // touches or overlaps the last region: extend it
		const int f = (int)(uint32_t)s->res[s->n_res - 1];
		s->res[s->n_res - 1] = (s->res[s->n_res - 1] >> 32) << 32 | (uint32_t)(f > fi ? f : fi);
		return;
	}
	if (s->n_res == s->m_res) s->m_res = s->m_res ? 2 * s->m_res : 16, s->res = (uint64_t*)realloc(s->res, s->m_res * sizeof(uint64_t));
	s->res[s->n_res++] = (uint64_t)st << 32 | (uint32_t)fi;
}

// the last (leftmost) interval of P goes to the result once it starts before the window; then every interval that does is dropped
static void wmo_sd_flush(wmo_sdust_t *s, int wstart)
{
	if (s->nP == 0 || s->P[s->nP - 1].start >= wstart) return;
	wmo_sd_emit(s, s->P[s->nP - 1].start, s->P[s->nP - 1].finish);
	while (s->nP > 0 && s->P[s->nP - 1].start < wstart) --s->nP;
}

static void wmo_sd_push(wmo_sdust_t *s, int t)
{
	const int cap = s->W - 2;
	if (s->n >= cap) { // the oldest triplet leaves the window, and the valid suffix if it reaches that far
		const int o = s->win[s->head];
		s->head = (s->head + 1) % cap, --s->n;
		s->rw -= --s->cw[o];
		if (s->L > s->n) --s->L, s->rv -= --s->cv[o];
	}
	s->win[(s->head + s->n) % cap] = t, ++s->n;
	++s->L;
	s->rw += s->cw[t]++;
	s->rv += s->cv[t]++;
	if (s->cv[t] * 10 > 2 * s->T) { // t is too frequent in the valid suffix: cut the suffix just past its oldest occurrence there
		int o;
		do {
			o = wmo_sd_at(s, s->n - s->L);
			s->rv -= --s->cv[o];
			--s->L;
		} while (o != t);
	}
}

static void wmo_sd_perfect(wmo_sdust_t *s, int wstart)
{
	int c[64], r = s->rv, best_r = 0, best_l = 0;
	memcpy(c, s->cv, sizeof(c));
	for (int i = s->n - s->L - 1; i >= 0; --i) { // suffixes longer than the valid one, shortest first
		const int t = wmo_sd_at(s, i);
		r += c[t]++;
		const int l = s->n - i - 1;
		if (r * 10 <= s->T * l) continue;
		int j = 0;
		for (; j < s->nP && s->P[j].start >= i + wstart; ++j) // the intervals this one contains; the best ratio among them
			if (best_r == 0 || s->P[j].r * best_l > best_r * s->P[j].l) best_r = s->P[j].r, best_l = s->P[j].l;
		if (best_r != 0 && r * best_l < best_r * l) continue;
		best_r = r, best_l = l;
		if (s->nP == s->mP) s->mP = s->mP ? 2 * s->mP : 16, s->P = (wmo_perf_t*)realloc(s->P, s->mP * sizeof(wmo_perf_t));
		memmove(s->P + j + 1, s->P + j, (s->nP - j) * sizeof(wmo_perf_t));
		++s->nP;
		s->P[j].start = i + wstart, s->P[j].finish = s->n + 2 + wstart, s->P[j].r = r, s->P[j].l = l;
		if (s->nP > s->max_nP) s->max_nP = s->nP;
	}
}

// The low-complexity regions of seq[0, len) as start << 32 | end, sorted and disjoint (at most max_out written); returns their
// number.  *max_nP (may be 0) receives the largest size the perfect-interval list reached.
long wmo_sdust(const char *seq, int len, int T, int W, uint64_t *out, long max_out, int *max_nP)
{
	wmo_sdust_t s;
	memset(&s, 0, sizeof(s));
	s.W = W, s.T = T;
	s.win = (int*)malloc(sizeof(int) * (W > 2 ? W - 2 : 1));
	for (int i = 0, l = 0, t = 0; i <= len; ++i) {
		const int b = i < len ? wmo_sd_nt4((unsigned char)seq[i]) : 4;
		if (b < 4) {
			++l, t = (t << 2 | b) & 63;
			if (l < 3) continue;
			const int wstart = (l > W ? l - W : 0) + (i + 1 - l);
			wmo_sd_flush(&s, wstart);
			wmo_sd_push(&s, t);
			if (s.rw * 10 > s.L * T) wmo_sd_perfect(&s, wstart);
		} else { // end of a piece: everything pending goes out, the window start advancing one base per interval
			int wstart = (l - W + 1 > 0 ? l - W + 1 : 0) + (i + 1 - l);
			while (s.nP) wmo_sd_flush(&s, wstart++);
			l = t = 0;
		}
	}
	const long n = s.n_res;
	memcpy(out, s.res, sizeof(uint64_t) * (n < max_out ? n : max_out));
	if (max_nP) *max_nP = s.max_nP;
	free(s.win); free(s.P); free(s.res);
	return n;
}

// The minimizers (x, y pairs of mm_sketch, position order) that keep at most half of their span [pos - span + 1, pos] outside
// the regions `reg` (wmo_sdust): kept in place, order preserved; returns their number.  T <= 0 keeps all.
long wmo_dust_minier(uint64_t *xy, long n, const uint64_t *reg, long n_reg)
{
	long k = 0, u = 0;
	for (long j = 0; j < n; ++j) {
		const int32_t pos = (int32_t)((uint32_t)xy[2 * j + 1] >> 1), span = (int32_t)(xy[2 * j] & 0xff);
		const int32_t s = pos - (span - 1), e = s + span;
		while (u < n_reg && (int32_t)(uint32_t)reg[u] <= s) ++u; // regions that end before the span never come back
		int32_t l = 0;
		for (long v = u; v < n_reg && (int32_t)(reg[v] >> 32) < e; ++v) {
			const int32_t rs = (int32_t)(reg[v] >> 32), re = (int32_t)(uint32_t)reg[v];
			l += (e < re ? e : re) - (s > rs ? s : rs);
		}
		if (l <= span >> 1) xy[2 * k] = xy[2 * j], xy[2 * k + 1] = xy[2 * j + 1], ++k;
	}
	return k;
}
