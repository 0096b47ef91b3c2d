// Seed lookup and anchor generation on sm_90a: mm_idx_get (reference src/index.c:88-105),
// collect_matches (src/map.c:97-130) and collect_seed_hits (src/map.c:222-254) for a batch of
// sketched query windows, followed by the tie-exact anchor sort (rsort.cuh).
//
// Index layout in HBM (replicated per GPU): sorted unique minimizer hashes `keys`, CSR offsets
// `pos_off` into the occurrence array `pos` (each list ascending, as src/index.c:239 leaves it) and an
// open-addressing hash table key -> key index for O(1) probes.  The bucket/khash structure of the
// reference is an implementation detail; the contract "hash -> (sorted list, n)" is what is kept.
#include <string.h>
#include <vector>
#include <algorithm>
#include "wm_common.cuh"
#include "scan.cuh"
#include "sketch.cuh"
#include "rsort.cuh"
#include "seed.cuh"
#include "seed_heap.cuh"

#define WM_HT_EMPTY 0xffffffffffffffffULL

__device__ __forceinline__ uint64_t wm_ht_mix(uint64_t k)
{
	k ^= k >> 31; k *= 0x9E3779B97F4A7C15ULL; k ^= k >> 29;
	return k;
}

__global__ void wm_ht_fill_kernel(const uint64_t *__restrict__ keys, int64_t n_keys, uint64_t *ht_key, uint32_t *ht_val, uint64_t mask)
{
	int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_keys) return;
	const uint64_t key = keys[i];
	uint64_t slot = wm_ht_mix(key) & mask;
	for (;;) {
		unsigned long long old = atomicCAS((unsigned long long*)&ht_key[slot], (unsigned long long)WM_HT_EMPTY, (unsigned long long)key);
		if (old == WM_HT_EMPTY || old == key) { ht_val[slot] = (uint32_t)i; return; }
		slot = (slot + 1) & mask;
	}
}

// mm_idx_get: returns the number of occurrences and the offset of the list in pos[]
__device__ __forceinline__ int wm_idx_get(const wm_idx_dev &ix, uint64_t minier, uint64_t *off)
{
	uint64_t slot = wm_ht_mix(minier) & ix.ht_mask;
	for (;;) {
		const uint64_t k = ix.ht_key[slot];
		if (k == minier) {
			const uint32_t i = ix.ht_val[slot];
			const uint64_t o = ix.pos_off[i];
			*off = o;
			return (int)(ix.pos_off[i + 1] - o);
		}
		if (k == WM_HT_EMPTY) { *off = 0; return 0; }
		slot = (slot + 1) & ix.ht_mask;
	}
}

// pass 1: one thread per query minimizer
__global__ void wm_seed_lookup_kernel(wm_idx_dev ix, const wm128_dev *__restrict__ mz, const int64_t *__restrict__ mz_off, int n_tasks, int64_t n_mz,
                                      int max_occ, int32_t *__restrict__ n_occ, int32_t *__restrict__ cnt, uint64_t *__restrict__ list_off,
                                      uint8_t *__restrict__ tandem, int32_t *__restrict__ mz_task)
{
	const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (m >= n_mz) return;
	int lo = 0, hi = n_tasks; // task of this minimizer: last t with mz_off[t] <= m
	while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (mz_off[mid] <= m) lo = mid; else hi = mid; }
	const uint64_t h = mz[m].x >> 8;
	uint64_t off;
	const int t = wm_idx_get(ix, h, &off);
	n_occ[m] = t;
	cnt[m] = t >= max_occ ? 0 : t; // src/map.c:111
	list_off[m] = off;
	int td = 0; // src/map.c:121-122
	if (m > mz_off[lo] && mz[m - 1].x >> 8 == h) td = 1;
	if (m < mz_off[lo + 1] - 1 && mz[m + 1].x >> 8 == h) td = 1;
	tandem[m] = (uint8_t)td;
	mz_task[m] = lo;
}

// pass 2: one thread per anchor (src/map.c:233-249).  FILTER: skip_seed (src/map.c:132-154) with the per-task bits of the
// seed filter (skip[t].x: WM_SKIP_* bits, .y: index names less than the read's name); keep[j] = 0 drops the occurrence.  Without
// -D / --dual=no / --for-only / --rev-only skip_seed() never skips: the FILTER = false instance runs and nothing is compacted.
template <bool FILTER>
__global__ void wm_seed_expand_kernel(wm_idx_dev ix, const wm128_dev *__restrict__ mz, int64_t n_mz, const int64_t *__restrict__ a_off,
                                      const uint64_t *__restrict__ list_off, const uint8_t *__restrict__ tandem, const int32_t *__restrict__ mz_task,
                                      const int32_t *__restrict__ qlen, int64_t n_a, wm128_dev *__restrict__ a,
                                      const uint2 *__restrict__ skip, int32_t *__restrict__ keep)
{
	const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n_a) return;
	int64_t lo = 0, hi = n_mz; // last m with a_off[m] <= j
	while (hi - lo > 1) { int64_t mid = (lo + hi) >> 1; if (a_off[mid] <= j) lo = mid; else hi = mid; }
	const wm128_dev p = mz[lo];
	const uint64_t r = ix.pos[list_off[lo] + (uint64_t)(j - a_off[lo])];
	wm128_dev o;
	bool drop = false;
	WM_SEED_ANCHOR(FILTER, ix, p, r, qlen, skip, mz_task[lo], tandem[lo], o, drop);
	if (FILTER) keep[j] = drop ? 0 : 1;
	a[j] = o;
}

// the seed filter's compaction, stable (the kept anchors keep their order, as collect_seed_hits writes them, so the tie-exact
// sort sees what radix_sort_128x sees): one thread per anchor, then one per task offset, which moves to its rank among the kept
__global__ void wm_seed_compact_kernel(const wm128_dev *__restrict__ a_raw, const int32_t *__restrict__ keep, const int64_t *__restrict__ keep_off,
                                       int64_t n_a, int64_t *__restrict__ task_a_off, int n_tasks, wm128_dev *__restrict__ a)
{
	const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (j < n_a) {
		if (keep[j]) a[keep_off[j]] = a_raw[j];
	} else if (j - n_a <= n_tasks) {
		const int t = (int)(j - n_a);
		task_a_off[t] = keep_off[task_a_off[t]];
	}
}

// pass 3: one thread per task: rep_len (src/map.c:106-127), kept-minimizer count, anchor offsets
__global__ void wm_seed_task_kernel(const wm128_dev *__restrict__ mz, const int64_t *__restrict__ mz_off, const int64_t *__restrict__ a_off,
                                    const int32_t *__restrict__ n_occ, int max_occ, int n_tasks, int32_t *__restrict__ rep_len,
                                    int32_t *__restrict__ n_mini_pos, int64_t *__restrict__ task_a_off, uint32_t *__restrict__ mini_pos)
{
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t > n_tasks) return;
	if (t == n_tasks) { task_a_off[t] = a_off[mz_off[t]]; return; }
	int rep_st = 0, rep_en = 0, rl = 0, nk = 0;
	for (int64_t m = mz_off[t]; m < mz_off[t + 1]; ++m) {
		const uint32_t q_pos = (uint32_t)mz[m].y, q_span = (uint32_t)(mz[m].x & 0xff);
		if (n_occ[m] >= max_occ) {
			int en = (int)(q_pos >> 1) + 1, st = en - (int)q_span;
			if (st > rep_en) { rl += rep_en - rep_st; rep_st = st, rep_en = en; }
			else rep_en = en;
			mini_pos[m] = q_pos >> 1;
		} else { ++nk; mini_pos[m] = (q_pos >> 1) | 0x80000000u; }
	}
	rl += rep_en - rep_st;
	rep_len[t] = rl, n_mini_pos[t] = nk;
	task_a_off[t] = a_off[mz_off[t]];
}

// tie-exact radix_sort_128x of each task's anchors (src/map.c:252)
__global__ void wm_anchor_sort_small_kernel(wm128_dev *__restrict__ a, const int64_t *__restrict__ off, int n_arr, const int32_t *__restrict__ ids)
{
	int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_arr) return;
	if (ids) t = ids[t];
	const int64_t n = off[t + 1] - off[t];
	if (n <= WM_RS_MIN_SIZE) wm_rs_insertsort(a + off[t], a + off[t] + n);
}

// One warp per array of more than 64 anchors.  Arrays of up to smem_cap anchors are staged in shared
// memory, where the serial cycle-leader walk of lane 0 runs at shared-memory instead of L2 latency.
__global__ void __launch_bounds__(32)
wm_anchor_sort_big_kernel(wm128_dev *__restrict__ a, const int64_t *__restrict__ off, const int32_t *__restrict__ big_ids, int n_big,
                          wm_rs_range *__restrict__ wl_all, int smem_cap)
{
	extern __shared__ __align__(16) unsigned char wm_sort_smem[];
	__shared__ wm_rs_warp_ws W;
	__shared__ __align__(8) uint64_t mbar;
	const int lane = threadIdx.x;
	uint32_t phase = 0;
	if (lane == 0) wm_mbar_init(&mbar, 1);
	__syncwarp();
	for (int i = blockIdx.x; i < n_big; i += gridDim.x) {
		const int t = big_ids[i];
		const int64_t base = off[t];
		const int n = (int)(off[t + 1] - base);
		wm_rs_range *wl = wl_all + (base >> 6) + t;
		wm128_dev *g = a + base;
		if (n <= smem_cap) {
			// the array into its shared-memory stage and back with bulk-asynchronous copies (16-byte elements: always aligned)
			wm128_dev *s = (wm128_dev*)wm_sort_smem;
			const uint32_t bytes = (uint32_t)n * (uint32_t)sizeof(wm128_dev);
			if (lane == 0) { wm_mbar_expect_tx(&mbar, bytes); wm_bulk_g2s(s, g, bytes, &mbar); }
			wm_mbar_wait(&mbar, phase); phase ^= 1;
			wm_radix_sort_warp(s, n, &W, wl, lane);
			__syncwarp();
			if (lane == 0) { wm_bulk_s2g(g, s, bytes); wm_bulk_s2g_wait(); } // (the stage is reused by the next array)
			__syncwarp();
		} else wm_radix_sort_warp(g, n, &W, wl, lane);
	}
}

// ---- giant arrays (a read inside a tandem array: 10^4..10^5 anchors) ----
// One CTA per array.  The permutation walk of a radix pass (ksort.h:126-138) is a serial chain, but only a thin one has to
// stay serial: every slot is written once, and *the j-th element to arrive in a bucket ejects that bucket's j-th misplaced
// element* (the bucket's own elements in between shift one slot to the right).  So a pass is done in three steps: all threads
// list the misplaced slots and their elements' digits (wm_gs_token_classify); thread 0 walks over digits and per-bucket arrival
// counters only, recording each element's arrival index (wm_gs_token_walk), while three feeder warps stream every bucket's
// upcoming digits into a shared-memory FIFO (wm_gs_token_feed), so the walker never waits for global memory; all threads move
// the 16-byte elements to the slots the records imply (wm_gs_token_place).  Passes with exactly two non-empty buckets need no
// walk at all (wm_gs_two_bucket_pass).  Sub-buckets that need another big pass go back on the array's work list; the smaller
// ones are sorted by the four warps in parallel (staged in shared memory, rsort.cuh); the <= 64-element ones by one thread each.
#define WM_GS_THREADS 128
#define WM_GS_F 128 // digit FIFO depth per bucket (bytes, power of two)
// WM_GS_STAGE: sub-ranges up to this many elements are sorted by one warp in shared memory.  Two instantiations: <2048>
// (143 KB of shared memory, one CTA per SM) for the giant arrays and <512> (47 KB, four CTAs per SM) for the medium ones,
// of which there are thousands per wave.
template <int WM_GS_STAGE>
struct wm_gs_sm {
	int B[256], E[256];            // bucket bounds of the current pass
	int ptr[256];                  // per bucket: list rank of the next misplaced slot an arrival ejects (walker)
	int filled[256];               // digits loaded so far, per bucket (feeders)
	int hist[256];
	int n_big, n_small, next_small, walk_done;
	union {
		struct { int A[256], moff[257]; } tok; // phase 1, token pass: arrivals before each bucket's turn, list offsets
		wm_rs_warp_ws W[4];                    // phase 2
	} v;
	wm_rs_range swl[4][40];        // per-warp work list of phase 2 (disjoint sub-ranges of > 64 elements of a <= 2048-element range)
	uint64_t mbar[4];              // per-warp mbarriers of the bulk copies that stage a sub-range
	uint32_t mbar_phase[4];
	union alignas(16) { // (bulk copies land in `stage`: 16-byte aligned)
		uint8_t fifo[256][WM_GS_F];
		wm128_dev stage[4][WM_GS_STAGE];
	} u;
};

// ---- a pass with exactly two non-empty buckets, in closed form ----
// The walk of ksort.h:126-138 over two buckets A (lower digit, region [beg, mid)) and B ([mid, end)) does this: let
// p_1 < .. < p_m be the positions of A's region that hold B-elements and q_1 < .. < q_m those of B's region that hold
// A-elements.  Cycle j picks up the element at p_j, drops it at B's write pointer and pushes the B-elements it finds there
// one slot to the right until it kicks out the A-element at q_j, which lands at p_j.  Hence, with q_0 = mid - 1:
//   A's region: position p_j receives the element of q_j, everything else stays;
//   B's region: position q_{j-1} + 1 receives the element of p_j, the positions up to q_j the element of their left
//               neighbour; everything after q_m stays.
// Both are prefix sums over "is misplaced" flags -- no serial walk.  The strand byte of an anchor array always splits it two
// ways, and the 64 kb byte of the position often does.  tmp / idx: scratch of the array (elements / int32), same indexing as a.
__device__ __forceinline__ int wm_gs_block_excl(bool flag, int *warp_tot, int tid, int *total)
{ // exclusive rank of `flag` among the CTA's 128 threads (4 warps); *total = number of flags set
	const unsigned w = __ballot_sync(0xffffffffu, flag);
	const int lane = tid & 31, wid = tid >> 5;
	if (lane == 0) warp_tot[wid] = __popc(w);
	__syncthreads();
	const int t0 = warp_tot[0], t1 = warp_tot[1], t2 = warp_tot[2], t3 = warp_tot[3];
	__syncthreads();
	*total = t0 + t1 + t2 + t3;
	return __popc(w & ((1u << lane) - 1u)) + (wid > 0 ? t0 : 0) + (wid > 1 ? t1 : 0) + (wid > 2 ? t2 : 0);
}

__device__ void wm_gs_two_bucket_pass(wm128_dev *a, wm128_dev *tmp, int32_t *idx, int beg, int mid, int end, int s, int lo, int *warp_tot, int tid)
{
	int carry = 0, tot;
	for (int base = beg; base < mid; base += WM_GS_THREADS) { // the list p_j (idx[beg ..))
		const int t = base + tid;
		const bool flag = t < mid && (int)(a[t].x >> s & 255) != lo;
		const int r = carry + wm_gs_block_excl(flag, warp_tot, tid, &tot);
		if (flag) idx[beg + r] = t;
		carry += tot;
	}
	const int m = carry;
	__syncthreads();
	carry = 0;
	for (int base = mid; base < end; base += WM_GS_THREADS) { // the list q_j (idx[mid ..)) and B's region
		const int t = base + tid;
		wm128_dev e; e.x = e.y = 0;
		if (t < end) e = a[t];
		const bool flag = t < end && (int)(e.x >> s & 255) == lo;
		const int c = carry + wm_gs_block_excl(flag, warp_tot, tid, &tot); // A-elements in [mid, t)
		if (flag) idx[mid + c] = t;
		if (t < end) {
			wm128_dev v = e;
			if (c < m) {
				wm128_dev left; left.x = left.y = 0;
				if (t > mid) left = a[t - 1];
				v = (t == mid || (int)(left.x >> s & 255) == lo) ? a[idx[beg + c]] : left;
			}
			tmp[t] = v;
		}
		carry += tot;
	}
	__syncthreads();
	carry = 0;
	for (int base = beg; base < mid; base += WM_GS_THREADS) { // A's region
		const int t = base + tid;
		wm128_dev e; e.x = e.y = 0;
		if (t < mid) e = a[t];
		const bool flag = t < mid && (int)(e.x >> s & 255) != lo;
		const int j = carry + wm_gs_block_excl(flag, warp_tot, tid, &tot);
		if (t < mid) tmp[t] = flag ? a[idx[mid + j]] : e;
		carry += tot;
	}
	__syncthreads();
	for (int t = beg + tid; t < end; t += WM_GS_THREADS) a[t] = tmp[t];
	__syncthreads();
}

// ---- any other pass: the token walk ----
// Bucket k's region is [B[k], E[k]); a slot is misplaced when its element's digit is not k.  lst / dig / rec: the misplaced slots
// in position order (bucket k's are lst[moff[k] .. moff[k + 1])), their elements' digits and the walk's records, all indexed by
// the list rank; the same scratch as the closed form (tmp, idx) plus two per-anchor arrays.  When the pass has at most
// sizeof(S->u) misplaced slots, the digits are also kept in shared memory (the `u` union is free in phase 1) and the walk reads
// them there directly; bigger passes stream them to the walker through per-bucket FIFOs.
//
// classify (all threads): the list, the digits and moff[]; returns the number of misplaced slots.  Each thread's slot grows by
// WM_GS_THREADS per round, so the bucket that holds it is found by a cursor that only moves forward.
template <typename sm_t>
__device__ int wm_gs_token_classify(sm_t *S, const wm128_dev *a, int32_t *lst, uint8_t *dig, int beg, int end, int s, int tid)
{
	int *moff = S->v.tok.moff;
	uint8_t *dsm = (uint8_t*)&S->u;
	for (int k = tid; k < 256; k += WM_GS_THREADS) moff[k] = 0;
	__syncthreads();
	int carry = 0, tot, kk = 0, n_own = 0; // n_own: this thread's misplaced slots in bucket kk's region, not yet counted in moff[kk]
	for (int base = beg; base < end; base += WM_GS_THREADS) {
		const int t = base + tid;
		int d = 0;
		if (t < end) {
			while (S->E[kk] <= t) { if (n_own) { atomicAdd(&moff[kk], n_own); n_own = 0; } ++kk; }
			d = (int)(a[t].x >> s & 255);
		}
		const bool mis = t < end && d != kk;
		const int r = carry + wm_gs_block_excl(mis, S->hist, tid, &tot);
		if (mis) {
			lst[r] = t; dig[r] = (uint8_t)d; ++n_own;
			if (r < (int)sizeof(S->u)) dsm[r] = (uint8_t)d;
		}
		carry += tot;
	}
	if (n_own) atomicAdd(&moff[kk], n_own);
	__syncthreads();
	if (tid < 32) { // counts -> exclusive offsets, in place; every bucket's walk pointer and FIFO fill start at its offset
		const int lane = tid;
		int cnt[8], sum = 0;
		#pragma unroll
		for (int k = 0; k < 8; ++k) { cnt[k] = moff[lane * 8 + k]; sum += cnt[k]; }
		int incl = sum;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { int t2 = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t2; }
		int acc = incl - sum;
		#pragma unroll
		for (int k = 0; k < 8; ++k) { moff[lane * 8 + k] = acc; S->ptr[lane * 8 + k] = acc; S->filled[lane * 8 + k] = acc; acc += cnt[k]; }
		if (lane == 31) moff[256] = acc;
		if (lane == 0) S->walk_done = 0;
	}
	__syncthreads();
	return carry;
}

// walk (thread 0), following ksort.h:126-138 on digits alone.  ptr[t] is the list rank of bucket t's next misplaced slot not yet
// ejected.  Bucket k's turn opens one cycle for each of its misplaced slots that no earlier arrival has ejected (A[k] were); a
// step moves the element in hand into bucket t (p = ptr[t]++), which ejects the element of t's misplaced slot p, whose digit is
// the next t.  The cycle closes when that digit is k: the ejected element goes to the slot q the cycle opened.  rec[] gets, per
// list rank, p for an arrival (the ejected slot's rank; the arrival index is p - moff[t]) and ~q for the element closing a cycle.
// A bucket's digits are consumed strictly in list order (arrivals before its turn, cycle openings during it).
//
// ... with every digit in shared memory (dsm): two dependent shared-memory loads per step, no waiting
template <typename sm_t, bool DBG>
__device__ void wm_gs_token_walk_resident(sm_t *S, int32_t *rec, unsigned long long &n_steps)
{
	int *ptr = S->ptr, *A = S->v.tok.A;
	const int *moff = S->v.tok.moff;
	const uint8_t *dsm = (const uint8_t*)&S->u;
	asm volatile("" : "+l"(rec)); // keep the pointer in registers (the loop re-derived it from the parameter bank on every step)
	for (int k = 0; k < 256; ++k) {
		const int q0 = ptr[k], qe = moff[k + 1];
		A[k] = q0 - moff[k];
		for (int q = q0; q < qe; ++q) {
			int t = dsm[q], g = q; // g: list rank of the element in hand
			if (DBG) ++n_steps;
			for (;;) {
				const int p = ptr[t];
				ptr[t] = p + 1;
				const int t2 = dsm[p];
				rec[g] = p;
				g = p;
				if (DBG) ++n_steps;
				if (t2 == k) { rec[p] = ~q; break; }
				t = t2;
			}
		}
	}
}

// ... or through FIFOs: the digit of rank p of bucket t, once the feeders have put it into the FIFO; then frees its FIFO slot
// (ptr[t] = p + 1).  Both loads are in one volatile asm so that the digit is read after the poll of `filled`, and the store after both.
template <bool DBG>
__device__ __forceinline__ int wm_gs_fifo_next(int *filled, const uint8_t *fifo, int *ptr, int t, int p, unsigned long long &n_wait)
{
	const uint32_t pf = (uint32_t)__cvta_generic_to_shared(filled + t), pd = (uint32_t)__cvta_generic_to_shared(fifo + t * WM_GS_F + (p & (WM_GS_F - 1)));
	uint32_t f, d;
	for (;;) {
		asm volatile("ld.volatile.shared.u32 %0, [%2];\n\tld.volatile.shared.u8 %1, [%3];" : "=r"(f), "=r"(d) : "r"(pf), "r"(pd));
		if ((int)f > p) break;
		if (DBG) ++n_wait;
	}
	*(volatile int*)&ptr[t] = p + 1;
	return (int)d;
}

template <typename sm_t, bool DBG>
__device__ void wm_gs_token_walk_fifo(sm_t *S, int32_t *rec, unsigned long long &n_steps, unsigned long long &n_wait)
{
	int *ptr = S->ptr, *A = S->v.tok.A, *filled = S->filled;
	const int *moff = S->v.tok.moff;
	const uint8_t *fifo = &S->u.fifo[0][0];
	asm volatile("" : "+l"(rec));
	for (int k = 0; k < 256; ++k) {
		const int q0 = ptr[k], qe = moff[k + 1];
		A[k] = q0 - moff[k];
		for (int q = q0; q < qe; ++q) {
			int t = wm_gs_fifo_next<DBG>(filled, fifo, ptr, k, q, n_wait), g = q;
			if (DBG) ++n_steps;
			for (;;) {
				const int p = ptr[t];
				const int t2 = wm_gs_fifo_next<DBG>(filled, fifo, ptr, t, p, n_wait);
				rec[g] = p; // (after the FIFO read: its address must not hold up the chain)
				g = p;
				if (DBG) ++n_steps;
				if (t2 == k) { rec[p] = ~q; break; }
				t = t2;
			}
		}
	}
}

// feed (warps 1-3, buckets tid - 32, + 96, + 192): keep every bucket's FIFO up to WM_GS_F digits ahead of the walker
template <typename sm_t>
__device__ void wm_gs_token_feed(sm_t *S, const uint8_t *dig, int tid)
{
	const int *moff = S->v.tok.moff;
	volatile int *ptr = S->ptr; volatile int *done = &S->walk_done;
	for (;;) {
		bool any = false, fed = false;
		for (int k = tid - 32; k < 256; k += WM_GS_THREADS - 32) {
			const int fl = S->filled[k], qe = moff[k + 1];
			if (fl >= qe) continue;
			any = true;
			const int pending = fl - ptr[k];   // loaded, not yet taken by the walker
			int room = WM_GS_F - pending;
			if (room > qe - fl) room = qe - fl;
			if (room > 32) room = 32;
			if (room >= WM_GS_F / 4 || (room > 0 && (room == qe - fl || pending < WM_GS_F / 4))) { // refill in batches unless the FIFO runs low
				const uint8_t *src = dig + fl;
				uint8_t r[32];
				#pragma unroll
				for (int m = 0; m < 32; ++m) if (m < room) r[m] = src[m];
				#pragma unroll
				for (int m = 0; m < 32; ++m) if (m < room) S->u.fifo[k][(fl + m) & (WM_GS_F - 1)] = r[m];
				__threadfence_block();
				*(volatile int*)&S->filled[k] = fl + room;
				fed = true;
			}
		}
		if (!any || *done) break;
		// nothing to load right now: do not hammer shared memory with polls (the walker's own loads queue behind them)
		if (!fed) __nanosleep(256);
	}
}

// place (all threads): the j-th arrival in bucket t (record p = moff[t] + j) lands at the start of t's run j (B[t], or one past
// t's (j-1)-th misplaced slot); the element closing the cycle opened at rank q lands at slot lst[q]; an own element of bucket t
// moves one slot to the right when an arrival ended its run r (the misplaced slots of t before it), r < A[t], and stays otherwise.
template <typename sm_t>
__device__ void wm_gs_token_place(sm_t *S, wm128_dev *a, wm128_dev *tmp, const int32_t *lst, const int32_t *rec, int beg, int end, int s, int tid)
{
	const int *A = S->v.tok.A, *moff = S->v.tok.moff;
	int carry = 0, tot, kk = 0;
	for (int base = beg; base < end; base += WM_GS_THREADS) {
		const int t = base + tid;
		wm128_dev e; e.x = e.y = 0;
		int d = 0;
		if (t < end) { while (S->E[kk] <= t) ++kk; e = a[t]; d = (int)(e.x >> s & 255); }
		const bool mis = t < end && d != kk;
		const int r = carry + wm_gs_block_excl(mis, S->hist, tid, &tot);
		if (t < end) {
			int dst;
			if (mis) {
				const int p = rec[r];
				dst = p < 0 ? lst[~p] : p == moff[d] ? S->B[d] : lst[p - 1] + 1;
			} else dst = r - moff[kk] < A[kk] ? t + 1 : t;
			tmp[dst] = e;
		}
		carry += tot;
	}
	__syncthreads();
	for (int t = beg + tid; t < end; t += WM_GS_THREADS) a[t] = tmp[t];
	__syncthreads();
}

template <int WM_GS_STAGE, bool WM_GS_DBG>
__global__ void __launch_bounds__(WM_GS_THREADS)
wm_anchor_sort_giant_kernel(wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ ids, int n_arr,
                            wm_rs_range *__restrict__ wl_all, unsigned long long *dbg, wm128_dev *__restrict__ tmp_all, int32_t *__restrict__ idx_all,
                            int32_t *__restrict__ rec_all, uint8_t *__restrict__ dig_all, int two_min)
{
	// tmp_all / idx_all / rec_all / dig_all: scratch of the passes, indexed like a_all (the closed form uses the first two); two_min:
	// ranges of at least this many elements take the closed form when their pass has two non-empty buckets (0: never)
	// dbg (tuning aid, WM_SORT_DEBUG=1): clocks spent by thread 0 in [0] histograms, [1] token walks, [2] sub-bucket dispatch + tiny
	// sorts, [3] phase 2, [7] the parallel parts of the passes (closed form, classify, place); [4] walker steps, [5] walker waits
	// (polls of an empty FIFO), [6] / [8] elements in closed-form / token passes
	long long t_dbg = dbg ? clock64() : 0;
	unsigned long long n_steps_dbg = 0, n_wait_dbg = 0;
#define WM_GS_LAP(i) do { if (dbg && tid == 0) { const long long t2 = clock64(); atomicAdd(dbg + (i), (unsigned long long)(t2 - t_dbg)); t_dbg = t2; } } while (0)
	extern __shared__ __align__(16) unsigned char wm_gs_smem[];
	typedef wm_gs_sm<WM_GS_STAGE> sm_t;
	sm_t *S = (sm_t*)wm_gs_smem;
	if (threadIdx.x < 4) { wm_mbar_init(&S->mbar[threadIdx.x], 1); S->mbar_phase[threadIdx.x] = 0; }
	__syncthreads();
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	for (int ai = blockIdx.x; ai < n_arr; ai += gridDim.x) {
		const int task = ids[ai];
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		wm128_dev *a = a_all + base;
		// work lists in global memory (the array's slice of wl_all: n / 64 + 1 entries): big ranges grow from the front,
		// small ones from the back
		wm_rs_range *wl = wl_all + (base >> 6) + task;
		const int wl_cap = (n >> 6) + 1;
		if (tid == 0) { S->n_big = 0, S->n_small = 0; wm_rs_range r; r.beg = 0, r.end = n, r.s = 56; wl[0] = r; S->n_big = 1; }
		__syncthreads();
		// ---- phase 1: big passes, one at a time ----
		for (;;) {
			if (S->n_big == 0) break;
			__syncthreads();
			wm_rs_range R = wl[S->n_big - 1];
			__syncthreads();
			if (tid == 0) --S->n_big;
			int beg = R.beg, end = R.end, s = R.s;
			bool single; int n_nz = 0, lo_digit = 0;
			for (;;) { // histogram of byte s >> 3; identity passes (one bucket holds everything) are skipped (ksort.h:121-125)
				for (int k = tid; k < 256; k += WM_GS_THREADS) S->hist[k] = 0;
				__syncthreads();
				for (int i = beg + tid; i < end; i += WM_GS_THREADS) atomicAdd(&S->hist[a[i].x >> s & 255], 1);
				__syncthreads();
				single = false; n_nz = 0; lo_digit = -1;
				for (int k = 0; k < 256; ++k) { // (uniform: every thread scans the same table)
					const int h = S->hist[k];
					if (h == end - beg) single = true;
					if (h > 0) { ++n_nz; if (lo_digit < 0) lo_digit = k; }
				}
				if (!single || s == 0) break;
				s = s > 8 ? s - 8 : 0;
				__syncthreads();
			}
			WM_GS_LAP(0);
			if (single) { __syncthreads(); continue; } // all keys equal down to the last byte: nothing moves
			if (wid == 0) { // bucket bounds: exclusive prefix over 256 counts
				int cnt[8], sum = 0;
				#pragma unroll
				for (int k = 0; k < 8; ++k) { cnt[k] = S->hist[lane * 8 + k]; sum += cnt[k]; }
				int incl = sum;
				#pragma unroll
				for (int o = 1; o < 32; o <<= 1) { int t2 = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t2; }
				int acc = beg + incl - sum;
				#pragma unroll
				for (int k = 0; k < 8; ++k) { S->B[lane * 8 + k] = acc; acc += cnt[k]; S->E[lane * 8 + k] = acc; }
			}
			__syncthreads();
			if (n_nz == 2 && two_min > 0 && end - beg >= two_min) { // two buckets: the pass in closed form, by all threads
				wm_gs_two_bucket_pass(a, tmp_all + base, idx_all + base, beg, S->E[lo_digit], end, s, lo_digit, S->hist, tid);
				if (WM_GS_DBG && tid == 0) atomicAdd(dbg + 6, (unsigned long long)(end - beg));
			} else { // any other pass: the token walk
				int32_t *lst = idx_all + base + beg, *rec = rec_all + base + beg;
				uint8_t *dig = dig_all + base + beg;
				const int n_mis = wm_gs_token_classify(S, a, lst, dig, beg, end, s, tid);
				WM_GS_LAP(7);
				if (n_mis > 0) {
					if (n_mis <= (int)sizeof(S->u)) { if (tid == 0) wm_gs_token_walk_resident<sm_t, WM_GS_DBG>(S, rec, n_steps_dbg); }
					else if (tid == 0) { wm_gs_token_walk_fifo<sm_t, WM_GS_DBG>(S, rec, n_steps_dbg, n_wait_dbg); *(volatile int*)&S->walk_done = 1; }
					else if (wid > 0) wm_gs_token_feed(S, dig, tid);
					__syncthreads();
					WM_GS_LAP(1);
					wm_gs_token_place(S, a, tmp_all + base, lst, rec, beg, end, s, tid);
				}
				if (WM_GS_DBG && tid == 0) atomicAdd(dbg + 8, (unsigned long long)(end - beg));
			}
			WM_GS_LAP(7);
			// sub-buckets (ksort.h:140-145)
			if (s > 0) {
				const int ns = s > 8 ? s - 8 : 0;
				for (int k = tid; k < 256; k += WM_GS_THREADS) {
					const int cb = S->B[k], ce = S->E[k], sz = ce - cb;
					if (sz > WM_GS_STAGE) { const int q = atomicAdd(&S->n_big, 1); wm_rs_range r; r.beg = cb, r.end = ce, r.s = ns; wl[q] = r; }
					else if (sz > WM_RS_MIN_SIZE) { const int q = atomicAdd(&S->n_small, 1); wm_rs_range r; r.beg = cb, r.end = ce, r.s = ns; wl[wl_cap - 1 - q] = r; }
					else if (sz > 1) wm_rs_insertsort(a + cb, a + ce);
				}
			}
			__syncthreads();
		}
		WM_GS_LAP(2);
		// ---- phase 2: the small ranges, one warp each, staged in shared memory ----
		if (tid == 0) S->next_small = 0;
		__syncthreads();
		{
			wm128_dev *st = S->u.stage[wid];
			uint32_t ph2 = S->mbar_phase[wid]; // the warp's barrier survives from array to array: remember its phase
			for (;;) {
				int q = 0;
				if (lane == 0) q = atomicAdd(&S->next_small, 1);
				q = __shfl_sync(0xffffffffu, q, 0);
				if (q >= S->n_small) break;
				const wm_rs_range R = wl[wl_cap - 1 - q];
				const int m = R.end - R.beg;
				const uint32_t bytes = (uint32_t)m * (uint32_t)sizeof(wm128_dev);
				if (lane == 0) { wm_mbar_expect_tx(&S->mbar[wid], bytes); wm_bulk_g2s(st, a + R.beg, bytes, &S->mbar[wid]); }
				wm_mbar_wait(&S->mbar[wid], ph2); ph2 ^= 1;
				wm_radix_sort_warp_from(st, m, R.s, &S->v.W[wid], S->swl[wid], lane);
				__syncwarp();
				if (lane == 0) { wm_bulk_s2g(a + R.beg, st, bytes); wm_bulk_s2g_wait(); }
				__syncwarp();
			}
			if (lane == 0) S->mbar_phase[wid] = ph2;
		}
		__syncthreads();
		WM_GS_LAP(3);
	}
	if (dbg && tid == 0) { atomicAdd(dbg + 4, n_steps_dbg); atomicAdd(dbg + 5, n_wait_dbg); }
#undef WM_GS_LAP
}

// WM_SORT_DEBUG=1: the counters of one launch of the CTA kernels (see wm_anchor_sort_giant_kernel), on stderr; frees dbg
#define WM_GS_DBG_BYTES (16 * sizeof(unsigned long long))
static void wm_gs_debug_report(unsigned long long *dbg, int n_arrays, cudaStream_t st)
{
	unsigned long long h[16];
	WM_CUDA_CHECK(cudaStreamSynchronize(st));
	WM_CUDA_CHECK(cudaMemcpy(h, dbg, WM_GS_DBG_BYTES, cudaMemcpyDeviceToHost));
	fprintf(stderr, "[sort-debug] arrays=%d clocks: hist %llu walk %llu parallel %llu dispatch %llu phase2 %llu | walker steps %llu wait polls %llu"
	        " | elements in token passes %llu closed-form passes %llu\n", n_arrays, h[0], h[1], h[7], h[2], h[3], h[4], h[5], h[8], h[6]);
	cudaFree(dbg);
}

// sort n_arr arrays (device); h_off is the host copy of the offsets
void wm_anchor_sort_run(wm_seed_ws *ws, wm128_dev *d_a, const int64_t *d_off, const int64_t *h_off, int n_arr, cudaStream_t st, const int32_t *only, int n_only)
{ // only != null: just the arrays only[0 .. n_only) of the n_arr
	if (n_arr <= 0 || (only && n_only <= 0)) return;
	std::vector<int32_t> big, small_ids;
	if (only) {
		for (int q = 0; q < n_only; ++q) { const int i = only[q]; if (h_off[i + 1] - h_off[i] > WM_RS_MIN_SIZE) big.push_back(i); else if (h_off[i + 1] - h_off[i] > 1) small_ids.push_back(i); }
	} else for (int i = 0; i < n_arr; ++i) if (h_off[i + 1] - h_off[i] > WM_RS_MIN_SIZE) big.push_back(i);
	if (getenv("WM_DP_STATS")) {
		int64_t mx = 0, n_2k = 0, n_10k = 0;
		for (int i = 0; i < n_arr; ++i) { int64_t n = h_off[i + 1] - h_off[i]; mx = n > mx ? n : mx; n_2k += n > 2560; n_10k += n > 10240; }
		fprintf(stderr, "[sort-stats] arrays=%d big=%d >2560:%ld >10240:%ld max=%ld total=%ld\n", n_arr, (int)big.size(), (long)n_2k, (long)n_10k, (long)mx, (long)h_off[n_arr]);
	}
	if (!only) { wm_count_launch(); wm_anchor_sort_small_kernel<<<(n_arr + 127) / 128, 128, 0, st>>>(d_a, d_off, n_arr, 0); }
	else if (!small_ids.empty()) {
		int32_t *d_small = (int32_t*)ws->small_ids.need(sizeof(int32_t) * small_ids.size());
		WM_CUDA_CHECK(wm_memcpy_async(d_small, small_ids.data(), sizeof(int32_t) * small_ids.size(), cudaMemcpyHostToDevice, st));
		wm_count_launch(); wm_anchor_sort_small_kernel<<<(unsigned)((small_ids.size() + 127) / 128), 128, 0, st>>>(d_a, d_off, (int)small_ids.size(), d_small);
		wm_stream_sync(st); // small_ids is a local
	}
	WM_CUDA_CHECK(cudaGetLastError());
	if (!big.empty()) {
		// three launches by size class: the shared-memory stage of the array sets the occupancy
		static int cap_m_env = -1; // WM_SORT_GIANT_MIN: arrays above this many anchors go to the <2048> instantiation (default: none --
		// measured on the tandem workload: everything on the light <512> instantiation, four CTAs per SM, is 10 % faster end to end)
		if (cap_m_env < 0) { const char *e = getenv("WM_SORT_GIANT_MIN"); cap_m_env = e && atoi(e) >= 2048 ? atoi(e) : (1 << 30); } // (above 13312 only with the walker kernels: the single-warp kernel stages the array in 208 KB)
		static int giant = -1, medium_coop = -1; // WM_SORT_GIANT=0 / WM_SORT_MEDIUM=0: the single-warp kernels (kept for comparison)
		if (giant < 0) { const char *e = getenv("WM_SORT_GIANT"); giant = (e && *e == '0') ? 0 : 1; e = getenv("WM_SORT_MEDIUM"); medium_coop = (e && *e == '0') ? 0 : 1; }
		const int cap_s = 2048, cap_m = medium_coop || cap_m_env < 13312 ? cap_m_env : 13312; // 32 KB and up to 208 KB of anchors
		WM_CUDA_CHECK(cudaFuncSetAttribute(wm_anchor_sort_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (cap_m < 13312 ? cap_m : 13312) * (int)sizeof(wm128_dev)));
		std::stable_sort(big.begin(), big.end(), [&](int x, int y) { return h_off[x + 1] - h_off[x] > h_off[y + 1] - h_off[y]; });
		size_t n_l = 0, n_m = 0;
		while (n_l < big.size() && h_off[big[n_l] + 1] - h_off[big[n_l]] > cap_m) ++n_l;
		while (n_l + n_m < big.size() && h_off[big[n_l + n_m] + 1] - h_off[big[n_l + n_m]] > cap_s) ++n_m;
		const size_t n_s = big.size() - n_l - n_m;
		int32_t *d_big = (int32_t*)ws->big_ids.need(sizeof(int32_t) * big.size());
		wm_rs_range *d_wl = (wm_rs_range*)ws->rs_stacks.need(sizeof(wm_rs_range) * (size_t)((h_off[n_arr] >> 6) + n_arr + 2));
		WM_CUDA_CHECK(wm_memcpy_async(d_big, big.data(), sizeof(int32_t) * big.size(), cudaMemcpyHostToDevice, st));
		static int two_min = -1; // WM_SORT_TWO_MIN: ranges of at least this many anchors take the closed form when their pass has two buckets (0: never)
		if (two_min < 0) { const char *e = getenv("WM_SORT_TWO_MIN"); two_min = e ? atoi(e) : 512; }
		// scratch of the passes of the CTA kernels, per anchor: one element (tmp), the misplaced slots (idx), the token walk's records
		// (int32) and digits (bytes)
		wm128_dev *d_tmp = 0; int32_t *d_idx = 0, *d_rec = 0; uint8_t *d_dig = 0;
		if (n_l || n_m) {
			const size_t na = (size_t)h_off[n_arr] + 1;
			d_tmp = (wm128_dev*)ws->sort_tmp.need(sizeof(wm128_dev) * na);
			d_idx = (int32_t*)ws->sort_idx.need(sizeof(int32_t) * na);
			d_rec = (int32_t*)ws->sort_tok.need((sizeof(int32_t) + 1) * na);
			d_dig = (uint8_t*)(d_rec + na);
		}
		if (n_l) {
			wm_count_launch();
			if (giant) {
				typedef wm_gs_sm<2048> sm_t;
				static bool attr_set = false;
				if (!attr_set) {
					WM_CUDA_CHECK(cudaFuncSetAttribute(wm_anchor_sort_giant_kernel<2048, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(sm_t)));
					WM_CUDA_CHECK(cudaFuncSetAttribute(wm_anchor_sort_giant_kernel<2048, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(sm_t)));
					attr_set = true;
				}
				unsigned long long *dbg = 0;
				if (getenv("WM_SORT_DEBUG")) { WM_CUDA_CHECK(cudaMalloc((void**)&dbg, WM_GS_DBG_BYTES)); WM_CUDA_CHECK(cudaMemset(dbg, 0, WM_GS_DBG_BYTES)); }
				static int giant_ctas = -1; // WM_SORT_GIANT_CTAS
				if (giant_ctas < 0) { const char *e = getenv("WM_SORT_GIANT_CTAS"); giant_ctas = e && atoi(e) > 0 ? atoi(e) : wm_sm_count(); } // one CTA per SM
				const unsigned g_l = (unsigned)(n_l < (size_t)giant_ctas ? n_l : (size_t)giant_ctas);
				if (dbg) wm_anchor_sort_giant_kernel<2048, true><<<g_l, WM_GS_THREADS, sizeof(sm_t), st>>>(d_a, d_off, d_big, (int)n_l, d_wl, dbg, d_tmp, d_idx, d_rec, d_dig, two_min);
				else wm_anchor_sort_giant_kernel<2048, false><<<g_l, WM_GS_THREADS, sizeof(sm_t), st>>>(d_a, d_off, d_big, (int)n_l, d_wl, 0, d_tmp, d_idx, d_rec, d_dig, two_min);
				if (dbg) {
					wm_gs_debug_report(dbg, (int)n_l, st);
				}
			} else wm_anchor_sort_big_kernel<<<(unsigned)n_l, 32, 0, st>>>(d_a, d_off, d_big, (int)n_l, d_wl, 0);
		}
		if (n_m) {
			wm_count_launch();
			if (medium_coop) { // thousands of arrays per wave: the light instantiation, four CTAs per SM
				typedef wm_gs_sm<512> sm_t;
				static bool attr_set = false;
				if (!attr_set) {
					WM_CUDA_CHECK(cudaFuncSetAttribute(wm_anchor_sort_giant_kernel<512, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(sm_t)));
					WM_CUDA_CHECK(cudaFuncSetAttribute(wm_anchor_sort_giant_kernel<512, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(sm_t)));
					attr_set = true;
				}
				unsigned long long *dbg = 0;
				if (getenv("WM_SORT_DEBUG")) { WM_CUDA_CHECK(cudaMalloc((void**)&dbg, WM_GS_DBG_BYTES)); WM_CUDA_CHECK(cudaMemset(dbg, 0, WM_GS_DBG_BYTES)); }
				static int med_ctas = -1; // WM_SORT_MEDIUM_CTAS: resident CTAs of the medium class (47 KB of shared memory each)
				if (med_ctas < 0) { const char *e = getenv("WM_SORT_MEDIUM_CTAS"); med_ctas = e && atoi(e) > 0 ? atoi(e) : 4 * wm_sm_count(); } // four CTAs per SM
				const unsigned g_m = (unsigned)(n_m < (size_t)med_ctas ? n_m : (size_t)med_ctas);
				if (dbg) {
					wm_anchor_sort_giant_kernel<512, true><<<g_m, WM_GS_THREADS, sizeof(sm_t), st>>>(d_a, d_off, d_big + n_l, (int)n_m, d_wl, dbg, d_tmp, d_idx, d_rec, d_dig, two_min);
					wm_gs_debug_report(dbg, (int)n_m, st);
				} else wm_anchor_sort_giant_kernel<512, false><<<g_m, WM_GS_THREADS, sizeof(sm_t), st>>>(d_a, d_off, d_big + n_l, (int)n_m, d_wl, 0, d_tmp, d_idx, d_rec, d_dig, two_min);
			} else wm_anchor_sort_big_kernel<<<(unsigned)n_m, 32, cap_m * sizeof(wm128_dev), st>>>(d_a, d_off, d_big + n_l, (int)n_m, d_wl, cap_m);
		}
		if (n_s) { wm_count_launch(); wm_anchor_sort_big_kernel<<<(unsigned)n_s, 32, cap_s * sizeof(wm128_dev), st>>>(d_a, d_off, d_big + n_l + n_m, (int)n_s, d_wl, cap_s); }
		WM_CUDA_CHECK(cudaGetLastError());
	}
}

// ---- --heap-sort=yes: collect_seed_hits_heap for the tasks whose sorted anchors tie (seed_heap.cuh) ----
// tie scan: one thread per sorted anchor; the first thread to see a[j].x == a[j - 1].x inside task t lists t
__global__ void wm_seed_tie_scan_kernel(const wm128_dev *__restrict__ a, const int64_t *__restrict__ task_a_off, int n_tasks, int64_t n_a,
                                        int32_t *__restrict__ flag, int32_t *__restrict__ ids, int32_t *__restrict__ n_ids)
{
	const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n_a || j == 0) return;
	if (a[j].x != a[j - 1].x) return;
	int lo = 0, hi = n_tasks; // the task holding j: last t with task_a_off[t] <= j
	while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (task_a_off[mid] <= j) lo = mid; else hi = mid; }
	if (j == task_a_off[lo]) return; // the previous anchor belongs to another task
	if (atomicCAS(&flag[lo], 0, 1) == 0) ids[atomicAdd(n_ids, 1)] = lo;
}

// counters of the replay, summed over all launches on a device (wm_seed_heap_stats): tasks, anchors, clocks of the merging
// lane, tasks whose heap lay in global memory, tasks whose replay disagreed with their sorted slice
__device__ unsigned long long g_wm_heap_stat[5];

// heap replay: one warp per listed task.  A task takes this launch when its heap, lists and staged occurrences need at most
// smem_bytes (small launch: min_bytes 0) or more than min_bytes (large launch: heap and lists in shared memory when they fit,
// the occurrences too when those fit as well; else both in global memory, heap_g / list_g at the task's minimizer offsets).
template <bool FILTER>
__global__ void __launch_bounds__(32)
wm_seed_heap_kernel(wm_idx_dev ix, const wm128_dev *__restrict__ mz, const int64_t *__restrict__ mz_off, const int32_t *__restrict__ cnt,
                    const uint64_t *__restrict__ list_off, const uint8_t *__restrict__ tandem, const int64_t *__restrict__ raw_off,
                    const int32_t *__restrict__ qlen, const uint2 *__restrict__ skip, const int32_t *__restrict__ ids, const int32_t *__restrict__ n_ids,
                    const int64_t *__restrict__ task_a_off, wm128_dev *__restrict__ a, wm128_dev *heap_g, wm_heap_list *list_g,
                    int64_t smem_bytes, int64_t min_bytes)
{
	extern __shared__ __align__(16) unsigned char wm_heap_smem[];
	const int lane = threadIdx.x, n_t = *n_ids;
	for (int i = blockIdx.x; i < n_t; i += gridDim.x) {
		const int t = ids[i];
		const int64_t m0 = mz_off[t], m1 = mz_off[t + 1], nm = m1 - m0, n_raw = raw_off[m1] - raw_off[m0];
		const int64_t hl = nm * (int64_t)WM_HEAP_ENTRY_BYTES, need = hl + n_raw * (int64_t)sizeof(uint64_t);
		if (min_bytes == 0 ? need > smem_bytes : need <= min_bytes) continue; // the other launch's task
		wm128_dev *H; wm_heap_list *L; uint64_t *stage = 0;
		const bool in_smem = hl <= smem_bytes;
		if (in_smem) {
			H = (wm128_dev*)wm_heap_smem, L = (wm_heap_list*)(H + nm);
			if (need <= smem_bytes) stage = (uint64_t*)(L + nm);
		} else H = heap_g + m0, L = list_g + m0;
		const int64_t base = task_a_off[t], n = task_a_off[t + 1] - base;
		const long long c0 = clock64();
		const int64_t w = wm_heap_replay_task<FILTER>(ix, mz, m0, m1, cnt, list_off, tandem, raw_off, qlen[t], FILTER ? skip[t] : make_uint2(0, 0),
		                                              H, L, stage, a + base, n, lane);
		if (lane == 0) {
			atomicAdd(&g_wm_heap_stat[0], 1ULL); atomicAdd(&g_wm_heap_stat[1], (unsigned long long)n);
			atomicAdd(&g_wm_heap_stat[2], (unsigned long long)(clock64() - c0));
			if (!in_smem) atomicAdd(&g_wm_heap_stat[3], 1ULL);
			if (w != n) atomicAdd(&g_wm_heap_stat[4], 1ULL);
		}
		__syncwarp();
	}
}

#define WM_HEAP_SMEM_SMALL (24 << 10)  // the small launch: up to nine CTAs per SM
#define WM_HEAP_SMEM_LARGE (200 << 10) // the large launch: one CTA per SM

// after the seed pass of heap sort: lists the tasks with ties and replays them.  h_mz_off: host copy of mz_off.
static void wm_seed_heap_run(wm_seed_ws *ws, const wm_idx_dev &ix, const wm128_dev *d_mz, const int64_t *d_mz_off, const int64_t *h_mz_off,
                             int n_tasks, const int32_t *d_qlen, const uint2 *d_skip, wm128_dev *d_a, const int64_t *d_task_a_off, cudaStream_t st)
{
	const int64_t n_a = ws->n_a;
	if (n_a < 2) return;
	int32_t *d_flag = (int32_t*)ws->heap_flag.need(sizeof(int32_t) * (n_tasks + 1));
	int32_t *d_ids = (int32_t*)ws->heap_ids.need(sizeof(int32_t) * (n_tasks + 1));
	WM_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, sizeof(int32_t) * (n_tasks + 1), st)); // d_flag[n_tasks]: the list's length
	wm_count_launch(); wm_seed_tie_scan_kernel<<<(unsigned)((n_a + 255) / 256), 256, 0, st>>>(d_a, d_task_a_off, n_tasks, n_a, d_flag, d_ids, d_flag + n_tasks);
	WM_CUDA_CHECK(cudaGetLastError());
	int64_t max_nm = 0; // the heap in global memory: only for tasks whose heap and lists outgrow the large launch's shared memory
	for (int t = 0; t < n_tasks; ++t) max_nm = std::max(max_nm, h_mz_off[t + 1] - h_mz_off[t]);
	wm128_dev *heap_g = 0; wm_heap_list *list_g = 0;
	if (max_nm * (int64_t)WM_HEAP_ENTRY_BYTES > WM_HEAP_SMEM_LARGE) {
		heap_g = (wm128_dev*)ws->heap_g.need(sizeof(wm128_dev) * (h_mz_off[n_tasks] + 1));
		list_g = (wm_heap_list*)ws->heap_l.need(sizeof(wm_heap_list) * (h_mz_off[n_tasks] + 1));
	}
	static bool attr_set = false;
	if (!attr_set) {
		WM_CUDA_CHECK(cudaFuncSetAttribute(wm_seed_heap_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, WM_HEAP_SMEM_LARGE));
		WM_CUDA_CHECK(cudaFuncSetAttribute(wm_seed_heap_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, WM_HEAP_SMEM_LARGE));
		attr_set = true;
	}
	const int sms = wm_sm_count();
	const int64_t *d_raw = (const int64_t*)ws->a_off.p;
	const int32_t *d_cnt = (const int32_t*)ws->cnt.p;
	const uint64_t *d_loff = (const uint64_t*)ws->list_off.p;
	const uint8_t *d_td = (const uint8_t*)ws->tandem.p;
	const unsigned g_s = (unsigned)std::min(n_tasks, 9 * sms), g_l = (unsigned)std::min(n_tasks, sms);
	for (int cls = 0; cls < 2; ++cls) {
		const int64_t smem = cls == 0 ? WM_HEAP_SMEM_SMALL : WM_HEAP_SMEM_LARGE, min_b = cls == 0 ? 0 : WM_HEAP_SMEM_SMALL;
		const unsigned g = cls == 0 ? g_s : g_l;
		wm_count_launch();
		if (d_skip) wm_seed_heap_kernel<true><<<g, 32, smem, st>>>(ix, d_mz, d_mz_off, d_cnt, d_loff, d_td, d_raw, d_qlen, d_skip, d_ids, d_flag + n_tasks,
		                                                           d_task_a_off, d_a, heap_g, list_g, smem, min_b);
		else wm_seed_heap_kernel<false><<<g, 32, smem, st>>>(ix, d_mz, d_mz_off, d_cnt, d_loff, d_td, d_raw, d_qlen, 0, d_ids, d_flag + n_tasks,
		                                                     d_task_a_off, d_a, heap_g, list_g, smem, min_b);
		WM_CUDA_CHECK(cudaGetLastError());
	}
}

// stats of the replay on the current device: o[0..4] = g_wm_heap_stat (see above); reset: zero them
extern "C" void wm_seed_heap_stats(double *o, int reset)
{
	unsigned long long h[5];
	WM_CUDA_CHECK(cudaMemcpyFromSymbol(h, g_wm_heap_stat, sizeof(h)));
	for (int i = 0; i < 5; ++i) o[i] = (double)h[i];
	if (reset) { memset(h, 0, sizeof(h)); WM_CUDA_CHECK(cudaMemcpyToSymbol(g_wm_heap_stat, h, sizeof(h))); }
}

// a replay that disagreed with its task's sorted slice cannot happen; if one did, the anchors are wrong and must not pass
void wm_seed_heap_check(void)
{
	unsigned long long bad = 0;
	WM_CUDA_CHECK(cudaMemcpyFromSymbol(&bad, g_wm_heap_stat, sizeof(bad), 4 * sizeof(unsigned long long)));
	if (bad) {
		fprintf(stderr, "[ERROR] winnowmap-b200: the heap merge of %llu seed task(s) disagreed with their sorted anchors\n", bad);
		exit(1);
	}
}

// Collect sorted anchors for all sketched tasks.  Inputs are the outputs of wm_sketch_run.
// On return: ws->a (anchors), ws->task_a_off (device, n_tasks+1), ws->rep_len, ws->n_mini_pos, ws->mini_pos;
// h_task_a_off (host, n_tasks+1) receives the anchor offsets.
void wm_seed_run(wm_seed_ws *ws, const wm_idx_dev &ix, const wm128_dev *d_mz, const int64_t *d_mz_off, int64_t n_mz, int n_tasks,
                 const int32_t *d_qlen, int max_occ, int64_t *h_task_a_off, cudaStream_t st, const uint2 *d_skip, bool heap)
{ // d_skip: the seed filter's bits per task, or null when no task filters (then no filter kernel runs); heap: --heap-sort=yes
	for (int i = 0; i <= n_tasks; ++i) h_task_a_off[i] = 0;
	int64_t *d_task_a_off = (int64_t*)ws->task_a_off.need(sizeof(int64_t) * (n_tasks + 1));
	int32_t *d_rep = (int32_t*)ws->rep_len.need(sizeof(int32_t) * (n_tasks + 1));
	int32_t *d_nmp = (int32_t*)ws->n_mini_pos.need(sizeof(int32_t) * (n_tasks + 1));
	WM_CUDA_CHECK(cudaMemsetAsync(d_task_a_off, 0, sizeof(int64_t) * (n_tasks + 1), st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_rep, 0, sizeof(int32_t) * (n_tasks + 1), st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_nmp, 0, sizeof(int32_t) * (n_tasks + 1), st));
	ws->n_a = 0;
	if (n_tasks <= 0) return;
	int32_t *d_nocc = (int32_t*)ws->n_occ.need(sizeof(int32_t) * (n_mz + 1));
	int32_t *d_cnt = (int32_t*)ws->cnt.need(sizeof(int32_t) * (n_mz + 1));
	uint64_t *d_loff = (uint64_t*)ws->list_off.need(sizeof(uint64_t) * (n_mz + 1));
	uint8_t *d_td = (uint8_t*)ws->tandem.need(n_mz + 1);
	int32_t *d_mtask = (int32_t*)ws->mz_task.need(sizeof(int32_t) * (n_mz + 1));
	int64_t *d_aoff = (int64_t*)ws->a_off.need(sizeof(int64_t) * (n_mz + 2));
	int64_t *d_tmp = (int64_t*)ws->scan_tmp.need(sizeof(int64_t) * wm_scan_tmp_elems(n_mz));
	uint32_t *d_mpos = (uint32_t*)ws->mini_pos.need(sizeof(uint32_t) * (n_mz + 1));
	if (n_mz > 0) {
		wm_count_launch(); wm_seed_lookup_kernel<<<(unsigned)((n_mz + 127) / 128), 128, 0, st>>>(ix, d_mz, d_mz_off, n_tasks, n_mz, max_occ, d_nocc, d_cnt, d_loff, d_td, d_mtask);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	wm_exclusive_scan(d_cnt, n_mz, d_aoff, d_tmp, st);
	int64_t n_a = 0;
	WM_CUDA_CHECK(wm_memcpy_async(&n_a, d_aoff + n_mz, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	ws->n_a = n_a;
	wm128_dev *d_a = (wm128_dev*)ws->a.need(sizeof(wm128_dev) * (n_a + 1)); // (with the filter: the bound before it)
	const bool filter = d_skip && n_a > 0;
	if (filter) {
		// the anchors before compaction and their keep flags go to the sort's per-anchor scratch (sort_tmp, sort_idx: dead until the
		// sort below, and sized for at least these n_a anchors there); only the scan of the flags takes a buffer of its own
		wm128_dev *d_raw = (wm128_dev*)ws->sort_tmp.need(sizeof(wm128_dev) * (n_a + 1));
		int32_t *d_keep = (int32_t*)ws->sort_idx.need(sizeof(int32_t) * (n_a + 1));
		int64_t *d_koff = (int64_t*)ws->keep_off.need(sizeof(int64_t) * (n_a + 1));
		wm_count_launch(); wm_seed_expand_kernel<true><<<(unsigned)((n_a + 127) / 128), 128, 0, st>>>(ix, d_mz, n_mz, d_aoff, d_loff, d_td, d_mtask, d_qlen, n_a, d_raw, d_skip, d_keep);
		WM_CUDA_CHECK(cudaGetLastError());
		wm_count_launch(); wm_seed_task_kernel<<<(n_tasks + 1 + 127) / 128, 128, 0, st>>>(d_mz, d_mz_off, d_aoff, d_nocc, max_occ, n_tasks, d_rep, d_nmp, d_task_a_off, d_mpos);
		WM_CUDA_CHECK(cudaGetLastError());
		int64_t *d_tmp2 = (int64_t*)ws->scan_tmp.need(sizeof(int64_t) * wm_scan_tmp_elems(std::max(n_mz, n_a)));
		wm_exclusive_scan(d_keep, n_a, d_koff, d_tmp2, st);
		wm_count_launch(); wm_seed_compact_kernel<<<(unsigned)((n_a + n_tasks + 1 + 127) / 128), 128, 0, st>>>(d_raw, d_keep, d_koff, n_a, d_task_a_off, n_tasks, d_a);
		WM_CUDA_CHECK(cudaGetLastError());
	} else {
		if (n_a > 0) {
			wm_count_launch(); wm_seed_expand_kernel<false><<<(unsigned)((n_a + 127) / 128), 128, 0, st>>>(ix, d_mz, n_mz, d_aoff, d_loff, d_td, d_mtask, d_qlen, n_a, d_a, 0, 0);
			WM_CUDA_CHECK(cudaGetLastError());
		}
		wm_count_launch(); wm_seed_task_kernel<<<(n_tasks + 1 + 127) / 128, 128, 0, st>>>(d_mz, d_mz_off, d_aoff, d_nocc, max_occ, n_tasks, d_rep, d_nmp, d_task_a_off, d_mpos);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	WM_CUDA_CHECK(wm_memcpy_async(h_task_a_off, d_task_a_off, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	ws->n_a = h_task_a_off[n_tasks];
	wm_anchor_sort_run(ws, d_a, d_task_a_off, h_task_a_off, n_tasks, st);
	if (heap) {
		std::vector<int64_t> h_mz_off(n_tasks + 1);
		WM_CUDA_CHECK(wm_memcpy_async(h_mz_off.data(), d_mz_off, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyDeviceToHost, st));
		wm_stream_sync(st);
		wm_seed_heap_run(ws, ix, d_mz, d_mz_off, h_mz_off.data(), n_tasks, d_qlen, d_skip, d_a, d_task_a_off, st);
	}
}

// ---- index upload ----
void wm_idx_dev_build_ht(wm_idx_dev *ix, cudaStream_t st)
{
	uint64_t cap = 1024;
	while (cap < (uint64_t)ix->n_keys * 2) cap <<= 1;
	uint64_t *hk = wm_dev_alloc<uint64_t>(cap);
	uint32_t *hv = wm_dev_alloc<uint32_t>(cap);
	WM_CUDA_CHECK(cudaMemsetAsync(hk, 0xff, cap * 8, st));
	if (ix->n_keys > 0) {
		wm_count_launch(); wm_ht_fill_kernel<<<(unsigned)((ix->n_keys + 255) / 256), 256, 0, st>>>(ix->keys, ix->n_keys, hk, hv, cap - 1);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	ix->ht_key = hk, ix->ht_val = hv, ix->ht_mask = cap - 1;
}

// ---- C ABI: standalone tie-exact sort (for the parity tests) ----
extern "C" int wm_radix_sort_128x_batch(int n_arr, wm128_dev *a, const int64_t *off)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] wm_radix_sort_128x_batch: no CUDA device visible; winnowmap-b200 has no CPU fallback\n");
		exit(1);
	}
	if (n_arr <= 0) return 0;
	const int64_t n = off[n_arr];
	wm128_dev *d_a = wm_dev_alloc<wm128_dev>(n + 1);
	int64_t *d_off = wm_dev_alloc<int64_t>(n_arr + 1);
	WM_CUDA_CHECK(cudaMemcpy(d_a, a, sizeof(wm128_dev) * n, cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_off, off, sizeof(int64_t) * (n_arr + 1), cudaMemcpyHostToDevice));
	wm_seed_ws ws;
	wm_anchor_sort_run(&ws, d_a, d_off, off, n_arr, 0);
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	WM_CUDA_CHECK(cudaMemcpy(a, d_a, sizeof(wm128_dev) * n, cudaMemcpyDeviceToHost));
	ws.release();
	cudaFree(d_a); cudaFree(d_off);
	return 0;
}

// ---- C ABI: the seed stage alone (lookup, anchors, seed filter, tie-exact sort and, with heap, the heap merge), on an index given
// as arrays, for the parity tests ----
extern "C" int wm_seed_batch(int64_t n_keys, const uint64_t *keys, const uint64_t *pos_off, const uint64_t *pos, int n_seq,
                             const uint32_t *seq_len, const uint32_t *name_rank, int n_tasks, const uint64_t *mz_xy, const int64_t *mz_off,
                             const int32_t *qlen, const uint32_t *skip, int max_occ, int heap, uint64_t **a_xy, int64_t **a_off,
                             int32_t *rep_len, int32_t *n_mini_pos, uint32_t *mini_pos)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] wm_seed_batch: no CUDA device visible; winnowmap-b200 has no CPU fallback\n");
		exit(1);
	}
	*a_off = (int64_t*)calloc(n_tasks + 1, sizeof(int64_t));
	*a_xy = (uint64_t*)malloc(16);
	if (n_tasks <= 0) return 0;
	const int64_t n_mz = mz_off[n_tasks], n_pos = pos_off[n_keys];
	wm_idx_dev ix;
	memset(&ix, 0, sizeof(ix));
	ix.n_keys = n_keys, ix.n_seq = (uint32_t)n_seq;
	uint64_t *d_keys = wm_dev_alloc<uint64_t>(n_keys + 1), *d_poff = wm_dev_alloc<uint64_t>(n_keys + 1), *d_pos = wm_dev_alloc<uint64_t>(n_pos + 1);
	uint32_t *d_len = wm_dev_alloc<uint32_t>(n_seq + 1), *d_rank = wm_dev_alloc<uint32_t>(n_seq + 1);
	if (n_keys > 0) WM_CUDA_CHECK(cudaMemcpy(d_keys, keys, sizeof(uint64_t) * n_keys, cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_poff, pos_off, sizeof(uint64_t) * (n_keys + 1), cudaMemcpyHostToDevice));
	if (n_pos > 0) WM_CUDA_CHECK(cudaMemcpy(d_pos, pos, sizeof(uint64_t) * n_pos, cudaMemcpyHostToDevice));
	if (n_seq > 0) {
		WM_CUDA_CHECK(cudaMemcpy(d_len, seq_len, sizeof(uint32_t) * n_seq, cudaMemcpyHostToDevice));
		WM_CUDA_CHECK(cudaMemcpy(d_rank, name_rank, sizeof(uint32_t) * n_seq, cudaMemcpyHostToDevice));
	}
	ix.keys = d_keys, ix.pos_off = d_poff, ix.pos = d_pos, ix.seq_len = d_len, ix.name_rank = d_rank;
	wm_idx_dev_build_ht(&ix, 0);
	wm128_dev *d_mz = wm_dev_alloc<wm128_dev>(n_mz + 1);
	int64_t *d_mzoff = wm_dev_alloc<int64_t>(n_tasks + 1);
	int32_t *d_qlen = wm_dev_alloc<int32_t>(n_tasks);
	uint2 *d_skip = skip ? wm_dev_alloc<uint2>(n_tasks) : 0;
	if (n_mz > 0) WM_CUDA_CHECK(cudaMemcpy(d_mz, mz_xy, sizeof(wm128_dev) * n_mz, cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_mzoff, mz_off, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_qlen, qlen, sizeof(int32_t) * n_tasks, cudaMemcpyHostToDevice));
	if (skip) WM_CUDA_CHECK(cudaMemcpy(d_skip, skip, sizeof(uint2) * n_tasks, cudaMemcpyHostToDevice));
	wm_seed_ws ws;
	wm_seed_run(&ws, ix, d_mz, d_mzoff, n_mz, n_tasks, d_qlen, max_occ, *a_off, 0, d_skip, heap != 0);
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	if (heap) wm_seed_heap_check();
	const int64_t n_a = (*a_off)[n_tasks];
	free(*a_xy);
	*a_xy = (uint64_t*)malloc(sizeof(wm128_dev) * (n_a + 1));
	if (n_a > 0) WM_CUDA_CHECK(cudaMemcpy(*a_xy, ws.a.p, sizeof(wm128_dev) * n_a, cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(rep_len, ws.rep_len.p, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(n_mini_pos, ws.n_mini_pos.p, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost));
	if (n_mz > 0) WM_CUDA_CHECK(cudaMemcpy(mini_pos, ws.mini_pos.p, sizeof(uint32_t) * n_mz, cudaMemcpyDeviceToHost));
	ws.release();
	cudaFree(d_keys); cudaFree(d_poff); cudaFree(d_pos); cudaFree(d_len); cudaFree(d_rank); cudaFree((void*)ix.ht_key); cudaFree((void*)ix.ht_val);
	cudaFree(d_mz); cudaFree(d_mzoff); cudaFree(d_qlen); cudaFree(d_skip);
	return 0;
}
