// The anchor of one occurrence (shared by the default seed path and the heap merge) and the heap merge itself:
// collect_seed_hits_heap (reference src/map.c:156-220, --heap-sort=yes), replayed on the device for the tasks whose sorted
// anchors hold equal x.  The device code here is also compiled for the host by the emulation tests (tests/hostsim/heap_emul.cpp),
// so it uses no CUDA runtime call.
//
// Why only those tasks.  The heap pops occurrences in ascending 64-bit position r; forward anchors are written in pop order,
// reverse ones from the end and then reversed, so the task's array is [forward anchors in pop order][reverse anchors in pop
// order], ascending in x.  Where no two kept anchors share x, that is the one ascending order, which the tie-exact radix sort
// already produced.  Anchors with equal x (copies of one query hash share an occurrence list; two lists may share a position)
// come out in an order that depends on the whole heap history: ks_heapdown (src/ksort.h:43-53) moves past equal children and
// takes the left one of two equal children.  So those tasks are replayed, pop by pop, with the same comparisons.
#pragma once
#include "seed.cuh"

// One anchor o of src/map.c:183-194 / :236-248 from query minimizer p and occurrence r, and with FILTER, skip_seed
// (src/map.c:132-154) into drop.  qlen[T] and skip[T] are the task's query length and filter bits (WM_SKIP_*, names below the
// read's name) with T the task expression t_expr; td is the minimizer's MM_SEED_TANDEM bit.  A macro rather than a function: the
// default path's wm_seed_expand_kernel is this very text and compiles to the instructions it had before the heap merge shared it.
#define WM_SEED_ANCHOR(FILTER, ix, p, r, qlen, skip, t_expr, td, o, drop) do { \
	const uint32_t q_pos = (uint32_t)(p).y, q_span = (uint32_t)((p).x & 0xff); \
	const int32_t rpos = (uint32_t)(r) >> 1; \
	if (((r) & 1) == (q_pos & 1)) { /* forward strand */ \
		(o).x = ((r) & 0xffffffff00000000ULL) | (uint32_t)rpos; \
		(o).y = (uint64_t)q_span << 32 | q_pos >> 1; \
	} else { /* reverse strand */ \
		(o).x = 1ULL << 63 | ((r) & 0xffffffff00000000ULL) | (uint32_t)rpos; \
		(o).y = (uint64_t)q_span << 32 | (uint32_t)((qlen)[t_expr] - ((q_pos >> 1) + 1 - q_span) - 1); \
	} \
	(o).y |= (uint64_t)((p).y >> 32) << 48; /* MM_SEED_SEG_SHIFT */ \
	if (td) (o).y |= 1ULL << 42;            /* MM_SEED_TANDEM */ \
	if (FILTER) { \
		const int t = (t_expr); \
		const uint2 sk = (skip)[t]; \
		const bool fwd = ((r) & 1) == (q_pos & 1); \
		bool drop_ = false; \
		if (sk.x & (WM_SKIP_NO_DIAG | WM_SKIP_NO_DUAL)) { \
			const uint32_t rid = (uint32_t)((r) >> 32), rank = (ix).name_rank[rid]; \
			/* strcmp(qname, name) == 0 and the sequence is as long as the window (not the read: src/map.c:364, :813) */ \
			if ((sk.x & WM_SKIP_NO_DIAG) && (sk.x & WM_SKIP_NAME_EQ) && rank == sk.y && (int)(ix).seq_len[rid] == (qlen)[t]) { \
				if ((uint32_t)rpos == q_pos >> 1) drop_ = true; /* the diagonal */ \
				else if (fwd) (o).y |= 1ULL << 43;             /* MM_SEED_SELF */ \
			} \
			if ((sk.x & WM_SKIP_NO_DUAL) && rank < sk.y) drop_ = true; /* strcmp(qname, name) > 0 */ \
		} \
		if ((sk.x & WM_SKIP_FOR_ONLY) && !fwd) drop_ = true; \
		if ((sk.x & WM_SKIP_REV_ONLY) && fwd) drop_ = true; \
		(drop) = drop_; \
	} \
} while (0)

// One list of the merge: the query minimizer (mm_match_t's q_pos, q_span, seg_id), its occurrences cr[0 .. n) and its tandem bit
struct wm_heap_list {
	wm128_dev p;
	const uint64_t *cr;
	uint32_t n, tandem;
};
#define WM_HEAP_ENTRY_BYTES (sizeof(wm128_dev) + sizeof(wm_heap_list)) // heap entry + list, per query minimizer of a task

// ks_heapdown with heap_lt(a, b) = a.x > b.x (src/map.c:87, src/ksort.h:43-53): the root holds the smallest x; a child moves up
// unless it is strictly greater than the sinking element, and of two equal children the left one is taken
__device__ __forceinline__ void wm_heap_down(wm128_dev *h, int i, int n)
{
	const wm128_dev tmp = h[i];
	int k = i;
	while ((k = (k << 1) + 1) < n) {
		if (k != n - 1 && h[k].x > h[k + 1].x) ++k;
		if (h[k].x > tmp.x) break;
		h[i] = h[k]; i = k;
	}
	h[i] = tmp;
}

// collect_seed_hits_heap of one task by one warp, written over the task's sorted anchors a[0 .. n) (the same multiset).
// The task's query minimizers are mz[m0 .. m1); cnt[m] is the length of m's occurrence list (0 when it is absent or reaches
// max_occ: collect_matches keeps no match, or one with n = 0, and neither enters the heap), list_off[m] where it starts in
// ix.pos, raw_off[m] the exclusive prefix of cnt (the anchors before the seed filter); qlen and task_skip are the task's query
// length and seed-filter bits (read with FILTER only).  H and L hold one heap entry and one list
// per query minimizer; stage, when not null, gets the task's occurrence lists (raw_off[m1] - raw_off[m0] positions), so that
// the pops read nothing from global memory.  H, L and stage may lie in shared or in global memory.
// Lanes list the matches in match order and stage their occurrences; lane 0 merges.  Returns, on lane 0, the number of anchors
// written; anything but n (or a forward count that disagrees with the sorted slice) means the slice was not this task's.
template <bool FILTER>
__device__ __forceinline__ int64_t wm_heap_replay_task(const wm_idx_dev &ix, const wm128_dev *__restrict__ mz, int64_t m0, int64_t m1,
                                                      const int32_t *__restrict__ cnt, const uint64_t *__restrict__ list_off,
                                                      const uint8_t *__restrict__ tandem, const int64_t *__restrict__ raw_off, int32_t qlen,
                                                      uint2 task_skip, wm128_dev *H, wm_heap_list *L, uint64_t *stage, wm128_dev *a, int64_t n, int lane)
{
	int n_l = 0;
	for (int64_t b = m0; b < m1; b += 32) { // the heap entries (cr[0], i << 32) in match order, as src/map.c:169-175 builds them
		const int64_t m = b + lane;
		const int c = m < m1 ? cnt[m] : 0;
		const unsigned bal = __ballot_sync(0xffffffffu, c > 0);
		if (c > 0) {
			const int j = n_l + __popc(bal & ((1u << lane) - 1u));
			const uint64_t *src = ix.pos + list_off[m];
			const uint64_t *cr = src;
			if (stage) {
				uint64_t *d = stage + (raw_off[m] - raw_off[m0]);
				for (int k = 0; k < c; ++k) d[k] = src[k];
				cr = d;
			}
			wm_heap_list l;
			l.p = mz[m], l.cr = cr, l.n = (uint32_t)c, l.tandem = tandem[m];
			L[j] = l;
			wm128_dev e;
			e.x = cr[0], e.y = (uint64_t)j << 32;
			H[j] = e;
		}
		n_l += __popc(bal);
	}
	__syncwarp();
	int64_t written = 0;
	if (lane == 0) {
		int64_t lo = 0, hi = n; // n_for: the first reverse anchor of the sorted slice
		while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (a[mid].x >> 63) hi = mid; else lo = mid + 1; }
		const int64_t n_for = lo;
		int hs = n_l;
		for (int i = (hs >> 1) - 1; i >= 0; --i) wm_heap_down(H, i, hs); // ks_heapmake
		int64_t f = 0, v = 0;
		while (hs > 0) {
			const wm128_dev top = H[0];
			const uint32_t j = (uint32_t)(top.y >> 32), k = (uint32_t)top.y;
			const wm_heap_list l = L[j];
			wm128_dev o;
			bool drop = false;
			WM_SEED_ANCHOR(FILTER, ix, l.p, top.x, &qlen, &task_skip, 0, l.tandem, o, drop);
			if (k < l.n - 1) { // the list's next occurrence replaces the root (src/map.c:197-203)
				wm128_dev e;
				e.x = l.cr[k + 1], e.y = top.y + 1;
				H[0] = e;
			} else H[0] = H[--hs];
			wm_heap_down(H, 0, hs);
			if (!drop) {
				if (!(o.x >> 63)) { if (f < n_for) a[f] = o; ++f; }
				else { if (n_for + v < n) a[n_for + v] = o; ++v; }
			}
		}
		written = f == n_for ? f + v : -1;
	}
	__syncwarp();
	return written;
}
