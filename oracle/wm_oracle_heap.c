/* TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
 *
 * Restatement of seed collection with --heap-sort=yes: collect_matches (src/map.c:97-130), skip_seed (:132-154) and
 * collect_seed_hits_heap (:156-220), written from what they compute.  The occurrence lists of the kept query minimizers are
 * merged through a binary heap keyed on the 64-bit occurrence r.  The heap routines follow the semantics of ksort.h's
 * heapdown / heapmake under the comparison "a before b when a.x > b.x is false ..." spelled out below; the order they leave
 * among equal keys is the whole point, so it is restated step by step rather than replaced by a stable sort.
 *
 * Built with wm_oracle.c (its flattened index, wmo_idx_get) by oracle/build_heap.sh into oracle/libwm_oracle_heap.so. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* wm_oracle.c: hash -> occurrence list (ascending), n */
const uint64_t *wmo_idx_get(const void *ix, uint64_t minier, int *n);

#define WMO_F_NO_DIAG  0x001
#define WMO_F_NO_DUAL  0x002
#define WMO_F_FOR_ONLY 0x100000
#define WMO_F_REV_ONLY 0x200000

typedef struct { uint64_t x, y; } wmo_h128_t;

typedef struct {
	uint32_t n, q_pos, q_span, seg_id, is_tandem;
	const uint64_t *cr;
} wmo_match_t;

/* Sift the element at i down a heap of n entries whose root holds the smallest x.  The walk goes to the left child, takes the
 * right one instead only when the left is strictly greater, and stops at the first child strictly greater than the sinking
 * element: equal children move up past it. */
static void wmo_heap_down(wmo_h128_t *h, long i, long n)
{
	wmo_h128_t tmp = h[i];
	long k = i;
	while ((k = 2 * k + 1) < n) {
		if (k != n - 1 && h[k].x > h[k + 1].x) ++k;
		if (h[k].x > tmp.x) break;
		h[i] = h[k];
		i = k;
	}
	h[i] = tmp;
}

/* Bottom-up construction: every inner node from the last one to the root is sifted down */
static void wmo_heap_make(wmo_h128_t *h, long n)
{
	long i;
	for (i = n / 2 - 1; i >= 0; --i) wmo_heap_down(h, i, n);
}

/* skip_seed: 1 drops the occurrence; *is_self marks a forward hit of a read against itself off the diagonal */
static int wmo_skip(int64_t flag, uint64_t r, const wmo_match_t *q, const char *qname, int qlen, const char *const *names,
                    const uint32_t *seq_len, int *is_self)
{
	*is_self = 0;
	if (qname && (flag & (WMO_F_NO_DIAG | WMO_F_NO_DUAL))) {
		const uint32_t rid = (uint32_t)(r >> 32);
		const int cmp = strcmp(qname, names[rid]);
		if ((flag & WMO_F_NO_DIAG) && cmp == 0 && (int)seq_len[rid] == qlen) {
			if ((uint32_t)r >> 1 == q->q_pos >> 1) return 1;
			if ((r & 1) == (q->q_pos & 1)) *is_self = 1;
		}
		if ((flag & WMO_F_NO_DUAL) && cmp > 0) return 1;
	}
	if ((flag & WMO_F_FOR_ONLY) && (r & 1) != (q->q_pos & 1)) return 1;
	if ((flag & WMO_F_REV_ONLY) && (r & 1) == (q->q_pos & 1)) return 1;
	return 0;
}

/* Anchors of one query (n_mv minimizers as x, y pairs) into a_xy (at most max_a written; the return value is their number,
 * after the filter), rep_len and the kept minimizers' span << 32 | position in mini_pos.  qname == NULL: a read without a name.
 * names / seq_len: the index's sequences. */
long wmo_collect_seed_hits_heap(const void *ix, int64_t flag, int max_occ, const char *qname, const char *const *names,
                                const uint32_t *seq_len, const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a,
                                int *rep_len_, uint64_t *mini_pos, int *n_mini_pos_)
{
	int rep_st = 0, rep_en = 0, rep_len = 0, n_mini_pos = 0;
	long i, n_m = 0, n_h = 0, n_tot = 0, n_for = 0, n_rev = 0;
	wmo_match_t *m = (wmo_match_t*)malloc(sizeof(wmo_match_t) * (n_mv > 0 ? n_mv : 1));
	wmo_h128_t *h, *rev;
	for (i = 0; i < n_mv; ++i) { /* collect_matches */
		const uint64_t px = mv_xy[2 * i], py = mv_xy[2 * i + 1];
		const uint32_t q_pos = (uint32_t)py, q_span = px & 0xff;
		int t;
		const uint64_t *cr = wmo_idx_get(ix, px >> 8, &t);
		if (t >= max_occ) {
			int en = (q_pos >> 1) + 1, st = en - (int)q_span;
			if (st > rep_en) { rep_len += rep_en - rep_st; rep_st = st, rep_en = en; }
			else rep_en = en;
			continue;
		}
		m[n_m].n = (uint32_t)t, m[n_m].q_pos = q_pos, m[n_m].q_span = q_span, m[n_m].seg_id = (uint32_t)(py >> 32), m[n_m].cr = cr;
		m[n_m].is_tandem = (i > 0 && px >> 8 == mv_xy[2 * (i - 1)] >> 8) || (i < n_mv - 1 && px >> 8 == mv_xy[2 * (i + 1)] >> 8);
		if (mini_pos) mini_pos[n_mini_pos] = (uint64_t)q_span << 32 | q_pos >> 1;
		++n_mini_pos;
		n_tot += t;
		++n_m;
	}
	rep_len += rep_en - rep_st;
	*rep_len_ = rep_len, *n_mini_pos_ = n_mini_pos;
	/* the heap: one entry (first occurrence, match index << 32 | rank in the list) per match with a non-empty list, in order */
	h = (wmo_h128_t*)malloc(sizeof(wmo_h128_t) * (n_m > 0 ? n_m : 1));
	rev = (wmo_h128_t*)malloc(sizeof(wmo_h128_t) * (n_tot > 0 ? n_tot : 1));
	for (i = 0; i < n_m; ++i)
		if (m[i].n > 0) h[n_h].x = m[i].cr[0], h[n_h].y = (uint64_t)i << 32, ++n_h;
	wmo_heap_make(h, n_h);
	while (n_h > 0) {
		const wmo_match_t *q = &m[h[0].y >> 32];
		const uint64_t r = h[0].x;
		const int32_t rpos = (uint32_t)r >> 1;
		int is_self;
		if (!wmo_skip(flag, r, q, qname, qlen, names, seq_len, &is_self)) {
			wmo_h128_t p;
			if ((r & 1) == (q->q_pos & 1)) {
				p.x = (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
				p.y = (uint64_t)q->q_span << 32 | q->q_pos >> 1;
			} else {
				p.x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
				p.y = (uint64_t)q->q_span << 32 | (uint32_t)(qlen - ((q->q_pos >> 1) + 1 - q->q_span) - 1);
			}
			p.y |= (uint64_t)q->seg_id << 48;
			if (q->is_tandem) p.y |= 1ULL << 42;
			if (is_self) p.y |= 1ULL << 43;
			/* forward anchors in pop order; reverse ones kept aside in pop order (the reference fills them from the end and
			 * reverses them afterwards, which gives the same sequence) */
			if (!(p.x >> 63)) { if (n_for < max_a) a_xy[2 * n_for] = p.x, a_xy[2 * n_for + 1] = p.y; ++n_for; }
			else rev[n_rev++] = p;
		}
		if ((uint32_t)h[0].y < q->n - 1) { /* the next occurrence of the same list takes the root */
			++h[0].y;
			h[0].x = m[h[0].y >> 32].cr[(uint32_t)h[0].y];
		} else h[0] = h[--n_h];
		wmo_heap_down(h, 0, n_h);
	}
	for (i = 0; i < n_rev; ++i)
		if (n_for + i < max_a) a_xy[2 * (n_for + i)] = rev[i].x, a_xy[2 * (n_for + i) + 1] = rev[i].y;
	free(m); free(h); free(rev);
	return n_for + n_rev;
}
