/* TEST INFRASTRUCTURE ONLY.  mm_chain_dp with is_cdna = 1 (src/chain.c:15-167, n_segs == 1): the chaining of spliced
 * mapping.  The same restatement as wmo_chain_dp of wm_oracle.c, link it with, except for the gap cost (chain.c:69-77): a gap
 * longer on the reference than on the query costs min(c_lin, c_log), any other c_lin + c_log / 2.
 * a_xy is modified (re-ordered chains are written to b_xy).  Returns n_u. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint64_t x, y; } wmo128_t;
void wmo_radix_sort_128x(wmo128_t *beg, long n); /* wm_oracle.c */
void wmo_radix_sort_64(uint64_t *beg, long n);

static inline int wmo_ilog2_32(uint32_t v)
{ /* chain.c:8-20: floor(log2(v)) for v > 0 */
	int r = 0;
	while (v >>= 1) ++r;
	return r;
}

int wmo_chain_dp_cdna(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc,
                      float gap_scale, long n, uint64_t *a_xy, uint64_t *u_out, uint64_t *b_xy, long *n_b)
{
	wmo128_t *a = (wmo128_t*)a_xy, *b = (wmo128_t*)b_xy, *w;
	int32_t k, *f, *p, *t, *v, n_u, n_v;
	int64_t i, j, st = 0;
	uint64_t *u, *u2, sum_qspan = 0;
	float avg_qspan;
	*n_b = 0;
	if (n == 0) return 0;
	f = (int32_t*)malloc(n * 4); p = (int32_t*)malloc(n * 4);
	t = (int32_t*)calloc(n, 4); v = (int32_t*)malloc(n * 4);
	for (i = 0; i < n; ++i) sum_qspan += a[i].y >> 32 & 0xff;
	avg_qspan = (float)sum_qspan / n; /* chain.c:41-42 */
	for (i = 0; i < n; ++i) { /* chain.c:45-90 */
		uint64_t ri = a[i].x;
		int64_t max_j = -1;
		int32_t qi = (int32_t)a[i].y, q_span = a[i].y >> 32 & 0xff;
		int32_t max_f = q_span, n_skip = 0, min_d;
		while (st < i && ri > a[st].x + max_dist_x) ++st;
		if (i - st > max_iter)
			while (i - st > max_iter && ri > a[st].x + min_dist_x) ++st;
		for (j = i - 1; j >= st; --j) {
			int64_t dr = ri - a[j].x;
			int32_t dq = qi - (int32_t)a[j].y, dd, sc, log_dd, gap_cost;
			if (dr == 0 || dq <= 0) continue;
			if (dq > max_dist_y || dq > max_dist_x) continue;
			dd = dr > dq ? dr - dq : dq - dr;
			if (dd > bw) continue;
			min_d = dq < dr ? dq : dr;
			sc = min_d > q_span ? q_span : dq < dr ? dq : dr;
			log_dd = dd ? wmo_ilog2_32(dd) : 0;
			{ /* chain.c:69-76 with is_cdna and sidi == sidj (so dr != 0 here) */
				int c_lin = (int)(dd * .01 * avg_qspan), c_log = log_dd;
				if (dr > dq) gap_cost = c_lin < c_log ? c_lin : c_log; /* an intron: longer on the reference */
				else gap_cost = c_lin + (c_log >> 1);
			}
			sc -= (int)((double)gap_cost * gap_scale + .499);
			sc += f[j];
			if (sc > max_f) {
				max_f = sc, max_j = j;
				if (n_skip > 0) --n_skip;
			} else if (t[j] == i) {
				if (++n_skip > max_skip) break;
			}
			if (p[j] >= 0) t[p[j]] = i;
		}
		f[i] = max_f, p[i] = max_j;
		v[i] = max_j >= 0 && v[max_j] > max_f ? v[max_j] : max_f;
	}
	/* chain.c:92-116 */
	memset(t, 0, n * 4);
	for (i = 0; i < n; ++i) if (p[i] >= 0) t[p[i]] = 1;
	for (i = n_u = 0; i < n; ++i) if (t[i] == 0 && v[i] >= min_sc) ++n_u;
	if (n_u == 0) { free(f); free(p); free(t); free(v); return 0; }
	u = (uint64_t*)malloc(n_u * 8);
	for (i = n_u = 0; i < n; ++i)
		if (t[i] == 0 && v[i] >= min_sc) {
			j = i;
			while (j >= 0 && f[j] < v[j]) j = p[j];
			if (j < 0) j = i;
			u[n_u++] = (uint64_t)f[j] << 32 | j;
		}
	wmo_radix_sort_64(u, n_u);
	for (i = 0; i < n_u >> 1; ++i) { uint64_t tt = u[i]; u[i] = u[n_u - i - 1], u[n_u - i - 1] = tt; }
	/* chain.c:118-135 */
	memset(t, 0, n * 4);
	for (i = n_v = k = 0; i < n_u; ++i) {
		int32_t n_v0 = n_v, k0 = k;
		j = (int32_t)u[i];
		do { v[n_v++] = j; t[j] = 1; j = p[j]; } while (j >= 0 && t[j] == 0);
		if (j < 0) {
			if (n_v - n_v0 >= min_cnt) u[k++] = u[i] >> 32 << 32 | (n_v - n_v0);
		} else if ((int32_t)(u[i] >> 32) - f[j] >= min_sc) {
			if (n_v - n_v0 >= min_cnt) u[k++] = ((u[i] >> 32) - f[j]) << 32 | (n_v - n_v0);
		}
		if (k0 == k) n_v = n_v0;
	}
	n_u = k;
	/* chain.c:141-147 */
	for (i = 0, k = 0; i < n_u; ++i) {
		int32_t k0 = k, ni = (int32_t)u[i];
		for (j = 0; j < ni; ++j) b[k] = a[v[k0 + (ni - j - 1)]], ++k;
	}
	/* chain.c:149-165 */
	w = (wmo128_t*)malloc((n_u > 0 ? n_u : 1) * sizeof(wmo128_t));
	for (i = k = 0; i < n_u; ++i) { w[i].x = b[k].x, w[i].y = (uint64_t)k << 32 | i; k += (int32_t)u[i]; }
	wmo_radix_sort_128x(w, n_u);
	u2 = (uint64_t*)malloc((n_u > 0 ? n_u : 1) * 8);
	for (i = k = 0; i < n_u; ++i) {
		int32_t jj = (int32_t)w[i].y, nn = (int32_t)u[jj];
		u2[i] = u[jj];
		memcpy(&a[k], &b[w[i].y >> 32], nn * sizeof(wmo128_t));
		k += nn;
	}
	for (i = 0; i < n_u; ++i) u_out[i] = u2[i];
	if (k) memcpy(b, a, k * sizeof(wmo128_t));
	*n_b = k;
	free(f); free(p); free(t); free(v); free(u); free(u2); free(w);
	return n_u;
}
