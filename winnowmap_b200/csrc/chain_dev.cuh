// Device functions of the chaining forward pass (mm_chain_dp, reference src/chain.c:45-90), shared by the kernels in
// chain.cu and by the CPU emulation harness of the tests (tests/hostsim/kernel_emul.cpp compiles this header for the host).
#pragma once
#include <limits.h>
#include "wm_common.cuh"
#include "sketch.cuh"
#include "chain.cuh"
#include "rsort.cuh"

__device__ __forceinline__ int wm_warp_incl_max(int v, int lane)
{
	#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		int t = __shfl_up_sync(0xffffffffu, v, o);
		if (lane >= o) v = max(v, t);
	}
	return v;
}

// score of predecessor j for anchor i (src/chain.c:61-84); false when j is not a candidate.  CDNA: the gap cost of is_cdna
// (src/chain.c:69-77 with n_segs == 1): a gap longer on the reference than on the query (an intron) costs min(c_lin, c_log)
template <bool CDNA = false>
__device__ __forceinline__ bool wm_chain_score(const wm128_dev aj, uint64_t ri, int32_t qi, int32_t q_span, const wm_chain_params &P, double avg_d, double scale_d, int *sc_out)
{
	const int64_t dr = (int64_t)(ri - aj.x);
	const int32_t dq = qi - (int32_t)aj.y;
	if (dr == 0 || dq <= 0) return false;
	if (dq > P.max_dist_y || dq > P.max_dist_x) return false;
	const int32_t dd = (int32_t)(dr > dq ? dr - dq : dq - dr);
	if (dd > P.bw) return false;
	const int32_t min_d = dq < dr ? dq : (int32_t)dr;
	int sc = min_d > q_span ? q_span : min_d;
	const int log_dd = dd ? 31 - __clz(dd) : 0;
	const int c_lin = (int)__dmul_rn(__dmul_rn((double)dd, .01), avg_d);
	const int gap_cost = CDNA && dr > dq ? (c_lin < log_dd ? c_lin : log_dd) : c_lin + (log_dd >> 1);
	sc -= (int)__dadd_rn(__dmul_rn((double)gap_cost, scale_d), .499);
	*sc_out = sc;
	return true;
}

// replay of the n_skip arithmetic (src/chain.c:85-88) over one 32-predecessor chunk: R = lanes that set a new
// maximum, K = lanes that hit a t[j]==i mark without setting one.  Returns the lane at which the reference
// leaves the loop (32 = it does not).
__device__ __forceinline__ int wm_chain_replay(unsigned R, unsigned K, int *n_skip_io, int max_skip)
{
	int n_skip = *n_skip_io, brk = 32;
	if (K == 0) {
		n_skip -= __popc(R); if (n_skip < 0) n_skip = 0;
	} else {
		unsigned ev = R | K;
		while (ev) {
			const int l = __ffs(ev) - 1;
			ev &= ev - 1;
			if (R >> l & 1) { if (n_skip > 0) --n_skip; }
			else if (++n_skip > max_skip) { brk = l; break; }
		}
	}
	*n_skip_io = n_skip;
	return brk;
}

// one warp, one task
template <bool CDNA = false>
__device__ void wm_chain_fill_warp(const wm128_dev *__restrict__ a, int n, const wm_chain_params &P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int lane)
{
	const unsigned FULL = 0xffffffffu;
	// avg_qspan (src/chain.c:41-42)
	unsigned long long sum = 0;
	for (int i = lane; i < n; i += 32) { sum += a[i].y >> 32 & 0xff; t[i] = 0; }
	for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
	const float avg_qspan = __fdiv_rn(__ull2float_rn(sum), __ll2float_rn((long long)n));
	const double avg_d = (double)avg_qspan, scale_d = (double)P.gap_scale;
	__syncwarp();
	int st = 0;
	for (int i = 0; i < n; ++i) {
		const uint64_t ri = a[i].x;
		const int32_t qi = (int32_t)a[i].y, q_span = (int32_t)(a[i].y >> 32 & 0xff);
		while (st < i && ri > a[st].x + (uint64_t)(int64_t)P.max_dist_x) ++st;
		if (i - st > P.max_iter) // the relaxed window of Winnowmap (src/chain.c:52-55)
			while (i - st > P.max_iter && ri > a[st].x + (uint64_t)(int64_t)P.min_dist_x) ++st;
		int max_f = q_span, max_j = -1, n_skip = 0;
		for (int jb = i - 1; jb >= st; jb -= 32) {
			const int j = jb - lane;
			bool cand = false;
			int sc = INT_MIN, pj = -1;
			if (j >= st && wm_chain_score<CDNA>(a[j], ri, qi, q_span, P, avg_d, scale_d, &sc)) {
				sc += f[j]; pj = p[j]; cand = true;
			}
			if (cand && pj >= 0) t[pj] = i; // src/chain.c:87 (only indices below every j still to be visited)
			__syncwarp();
			const bool marked = cand && t[j] == i;
			const int incl = wm_warp_incl_max(cand ? sc : INT_MIN, lane);
			int excl = __shfl_up_sync(FULL, incl, 1);
			if (lane == 0) excl = INT_MIN;
			excl = max(excl, max_f);
			const bool rec = cand && sc > excl;
			const unsigned R = __ballot_sync(FULL, rec), K = __ballot_sync(FULL, marked && !rec);
			const int brk = wm_chain_replay(R, K, &n_skip, P.max_skip);
			const unsigned Rv = brk < 32 ? (R & ((1u << brk) - 1u)) : R;
			if (Rv) {
				const int top = 31 - __clz(Rv);
				max_f = __shfl_sync(FULL, sc, top);
				max_j = jb - top;
			}
			if (brk < 32) break;
		}
		if (lane == 0) {
			f[i] = max_f, p[i] = max_j;
			const int vj = max_j >= 0 ? v[max_j] : INT_MIN;
			v[i] = (max_j >= 0 && vj > max_f) ? vj : max_f; // src/chain.c:89
		}
		__syncwarp();
	}
}


// ---- second formulation: dense candidates -------------------------------------------------------------------
// Only candidates (predecessors that pass the three `continue`s of src/chain.c:61-73) touch the state of the
// reference's inner loop: a non-candidate changes neither max_f nor n_skip nor t[].  So the scan is split: a cheap
// pass tests 32 predecessors per step (one load, a handful of integer operations, one ballot) and appends the
// candidates, in scan order, to a small per-warp list; whenever 32 of them are waiting, they are resolved with the
// exact chunk logic above.  In tandem arrays a window of `max_iter` = 5000 predecessors holds about 10 % candidates,
// so the expensive resolve runs ten times less often.  Early termination (n_skip > max_skip) discards the rest of
// the list; candidates scanned past the break point cost only the cheap test.
#define WM_CHAIN_DENSE_CAP 64

__device__ __forceinline__ bool wm_chain_is_cand(const wm128_dev aj, uint64_t ri, int32_t qi, const wm_chain_params &P)
{ // the predicate of wm_chain_score without the score
	const int64_t dr = (int64_t)(ri - aj.x);
	const int32_t dq = qi - (int32_t)aj.y;
	if (dr == 0 || dq <= 0) return false;
	if (dq > P.max_dist_y || dq > P.max_dist_x) return false;
	const int32_t dd = (int32_t)(dr > dq ? dr - dq : dq - dr);
	return dd <= P.bw;
}

// D: the warp's candidate list (WM_CHAIN_DENSE_CAP entries, shared memory)
template <bool CDNA = false>
__device__ void wm_chain_fill_warp_dense(const wm128_dev *__restrict__ a, int n, const wm_chain_params &P, int32_t *f, int32_t *p, int32_t *t, int32_t *v,
                                         int32_t *D, int lane)
{
	const unsigned FULL = 0xffffffffu;
	unsigned long long sum = 0;
	for (int i = lane; i < n; i += 32) { sum += a[i].y >> 32 & 0xff; t[i] = 0; }
	for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
	const float avg_qspan = __fdiv_rn(__ull2float_rn(sum), __ll2float_rn((long long)n));
	const double avg_d = (double)avg_qspan, scale_d = (double)P.gap_scale;
	__syncwarp();
	int st = 0;
	for (int i = 0; i < n; ++i) {
		const uint64_t ri = a[i].x;
		const int32_t qi = (int32_t)a[i].y, q_span = (int32_t)(a[i].y >> 32 & 0xff);
		while (st < i && ri > a[st].x + (uint64_t)(int64_t)P.max_dist_x) ++st;
		if (i - st > P.max_iter)
			while (i - st > P.max_iter && ri > a[st].x + (uint64_t)(int64_t)P.min_dist_x) ++st;
		int max_f = q_span, max_j = -1, n_skip = 0;
		int cnt = 0;      // candidates waiting in D, in scan order
		int jb = i - 1;   // next predecessor to scan
		bool stop = false;
		while (!stop) {
			// cheap scan until 32 candidates wait or the window is exhausted
			while (cnt < 32 && jb >= st) {
				const int j = jb - lane;
				const bool c = j >= st && wm_chain_is_cand(a[j], ri, qi, P);
				const unsigned m = __ballot_sync(FULL, c);
				if (c) D[cnt + __popc(m & ((1u << lane) - 1u))] = j;
				cnt += __popc(m);
				jb -= 32;
			}
			if (cnt == 0) break;
			__syncwarp();
			// exact resolve of the first min(cnt, 32) candidates: the chunk logic of wm_chain_fill_warp on a dense chunk
			const int m_act = cnt < 32 ? cnt : 32;
			const bool cand = lane < m_act;
			int j = -1, sc = INT_MIN, pj = -1;
			if (cand) {
				j = D[lane];
				wm_chain_score<CDNA>(a[j], ri, qi, q_span, P, avg_d, scale_d, &sc);
				sc += f[j]; pj = p[j];
			}
			if (cand && pj >= 0) t[pj] = i;
			__syncwarp();
			const bool marked = cand && t[j] == i;
			const int incl = wm_warp_incl_max(cand ? sc : INT_MIN, lane);
			int excl = __shfl_up_sync(FULL, incl, 1);
			if (lane == 0) excl = INT_MIN;
			excl = max(excl, max_f);
			const bool rec = cand && sc > excl;
			const unsigned R = __ballot_sync(FULL, rec), K = __ballot_sync(FULL, marked && !rec);
			const int brk = wm_chain_replay(R, K, &n_skip, P.max_skip);
			const unsigned Rv = brk < 32 ? (R & ((1u << brk) - 1u)) : R;
			if (Rv) {
				const int top = 31 - __clz(Rv);
				max_f = __shfl_sync(FULL, sc, top);
				max_j = __shfl_sync(FULL, j, top);
			}
			if (brk < 32) break;
			// drop the resolved candidates
			const int rest = cnt - m_act;
			int keep = 0;
			if (lane < rest) keep = D[lane + 32];
			__syncwarp();
			if (lane < rest) D[lane] = keep;
			cnt = rest;
			if (cnt == 0 && jb < st) stop = true;
		}
		if (lane == 0) {
			f[i] = max_f, p[i] = max_j;
			const int vj = max_j >= 0 ? v[max_j] : INT_MIN;
			v[i] = (max_j >= 0 && vj > max_f) ? vj : max_f; // src/chain.c:89
		}
		__syncwarp();
	}
}

// ---- third formulation: sliding window in shared memory ----------------------------------------------------
// The plain warp loop above is latency bound: every 32-predecessor step waits for two dependent global-memory round
// trips (a[j] / f[j] / p[j], then the t[] marks), and the window start is found with one dependent load per step.
// Here (1) the window start of every anchor is computed beforehand, in parallel (wm_chain_window_start: the serial
// `while` loops of src/chain.c:49-55 have a closed form because a[] is sorted), (2) the last RING anchors' (x, q, f, p,
// t-mark, v) live in a per-warp shared-memory ring, so a step costs shared-memory latency; predecessors older than the
// ring are rare (the scan usually stops after ~100 candidates) and are read from global memory as before, (3) anchors are
// loaded and f / p / v written back 32 at a time, coalesced, and (4) a step examines 64 predecessors: the loads and the
// score arithmetic of both halves are issued together, the order-dependent part (running maximum, n_skip replay) is
// resolved half by half.  Marks t[p[j]] = i written for the second half cannot touch an entry of the first half
// (p[j] < j), so publishing them early does not change which entries the first half sees marked.
//
// st[i] of src/chain.c:49-55.  The reference advances st (which persists across i) while ri > a[st].x + max_dist_x,
// then, if i - st > max_iter, while that still holds and ri > a[st].x + min_dist_x.  Both conditions are monotone in
// st and in i (a[] ascending), so st_i = max(lb(max_dist_x), min(i - max_iter, lb(min_dist_x))) with lb(d) = the first s
// whose a[s].x + d >= ri.
__device__ __forceinline__ int wm_chain_window_start(const wm128_dev *__restrict__ a, int i, const wm_chain_params &P)
{
	const uint64_t ri = a[i].x;
	int lo = 0, hi = i; // first s in [0, i] with !(ri > a[s].x + max_dist_x); s = i always qualifies
	while (lo < hi) { const int m = (lo + hi) >> 1; if (ri > a[m].x + (uint64_t)(int64_t)P.max_dist_x) lo = m + 1; else hi = m; }
	int st = lo;
	if (i - st > P.max_iter) {
		hi = i - P.max_iter; // lo = st: the answer lies in [st, i - max_iter]
		while (lo < hi) { const int m = (lo + hi) >> 1; if (ri > a[m].x + (uint64_t)(int64_t)P.min_dist_x) lo = m + 1; else hi = m; }
		st = lo;
	}
	return st;
}

// per-warp ring of RING anchors (RING a power of two >= 64): 28 bytes per slot
template <int RING> struct wm_chain_ring {
	uint64_t x[RING];
	int32_t q[RING], f[RING], p[RING], t[RING], v[RING];
};

// One warp, one task.  v[] holds st[] on entry (wm_chain_window_start of every anchor) and the peak scores on return.
template <int RING, bool CDNA = false>
__device__ void wm_chain_fill_warp_ring(const wm128_dev *__restrict__ a, int n, const wm_chain_params &P, int32_t *f, int32_t *p, int32_t *t, int32_t *v,
                                        wm_chain_ring<RING> *R, int lane)
{
	const unsigned FULL = 0xffffffffu;
	constexpr int MASK = RING - 1;
	unsigned long long sum = 0;
	for (int i = lane; i < n; i += 32) { sum += a[i].y >> 32 & 0xff; t[i] = 0; }
	for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
	const float avg_qspan = __fdiv_rn(__ull2float_rn(sum), __ll2float_rn((long long)n));
	const double avg_d = (double)avg_qspan, scale_d = (double)P.gap_scale;
	__syncwarp();
	for (int i0 = 0; i0 < n; i0 += 32) {
		// this block's anchors and window starts, one per lane
		const int il = i0 + lane;
		wm128_dev al; al.x = al.y = 0; int stl = 0;
		if (il < n) { al = a[il]; stl = v[il]; }
		const int nb = n - i0 < 32 ? n - i0 : 32;
		for (int k = 0; k < nb; ++k) {
			const int i = i0 + k;
			const uint64_t ri = __shfl_sync(FULL, al.x, k), yi = __shfl_sync(FULL, al.y, k);
			const int st = __shfl_sync(FULL, stl, k);
			const int32_t qi = (int32_t)yi, q_span = (int32_t)(yi >> 32 & 0xff);
			const int ring_lo = i - RING; // anchors [max(0, i - RING), i) are in the ring
			int max_f = q_span, max_j = -1, n_skip = 0;
			bool brk_out = false;
			for (int jb = i - 1; jb >= st && !brk_out; jb -= 64) {
				bool cand[2]; int sc[2], jj[2];
				#pragma unroll
				for (int h = 0; h < 2; ++h) {
					const int j = jb - 32 * h - lane;
					jj[h] = j; cand[h] = false; sc[h] = INT_MIN;
					if (j >= st) {
						wm128_dev aj; int fj, pj;
						if (j >= ring_lo) { const int s = j & MASK; aj.x = R->x[s]; aj.y = (uint64_t)(uint32_t)R->q[s]; fj = R->f[s]; pj = R->p[s]; }
						else { aj = a[j]; fj = f[j]; pj = p[j]; }
						int s0;
						if (wm_chain_score<CDNA>(aj, ri, qi, q_span, P, avg_d, scale_d, &s0)) {
							cand[h] = true; sc[h] = s0 + fj;
							if (pj >= 0) { if (pj >= ring_lo) R->t[pj & MASK] = i; else t[pj] = i; } // src/chain.c:87
						}
					}
				}
				__syncwarp();
				#pragma unroll
				for (int h = 0; h < 2; ++h) {
					if (h == 1 && jb - 32 < st) break; // the second half is empty
					const int j = jj[h];
					const bool marked = cand[h] && (j >= ring_lo ? R->t[j & MASK] : t[j]) == i;
					const unsigned G = __ballot_sync(FULL, cand[h] && sc[h] > max_f);
					unsigned Rm = G;
					if (G & (G - 1)) { // two or more lanes beat the running maximum: the records are the prefix maxima among them
						const int incl = wm_warp_incl_max(cand[h] ? sc[h] : INT_MIN, lane);
						int excl = __shfl_up_sync(FULL, incl, 1);
						if (lane == 0) excl = INT_MIN;
						excl = max(excl, max_f);
						Rm = __ballot_sync(FULL, cand[h] && sc[h] > excl);
					}
					const unsigned K = __ballot_sync(FULL, marked) & ~Rm;
					const int brk = wm_chain_replay(Rm, K, &n_skip, P.max_skip);
					const unsigned Rv = brk < 32 ? (Rm & ((1u << brk) - 1u)) : Rm;
					if (Rv) {
						const int top = 31 - __clz(Rv);
						max_f = __shfl_sync(FULL, sc[h], top);
						max_j = jb - 32 * h - top;
					}
					if (brk < 32) { brk_out = true; break; }
				}
			}
			// anchor i enters the ring (its slot held anchor i - RING, which is no longer addressed through the ring)
			int vj = INT_MIN;
			if (max_j >= 0) vj = max_j >= ring_lo ? R->v[max_j & MASK] : v[max_j];
			const int vi = (max_j >= 0 && vj > max_f) ? vj : max_f; // src/chain.c:89
			__syncwarp();
			if (lane == 0) {
				const int s = i & MASK;
				R->x[s] = ri; R->q[s] = qi; R->f[s] = max_f; R->p[s] = max_j; R->t[s] = 0; R->v[s] = vi;
			}
			__syncwarp();
		}
		// write the block's results back, coalesced (RING >= 64: the whole block is still in the ring)
		if (il < n) { const int s = il & MASK; f[il] = R->f[s]; p[il] = R->p[s]; v[il] = R->v[s]; }
		__syncwarp();
	}
}

// ---- fourth formulation: tiles of 32 consecutive anchors, one warp per anchor, dataflow between the warps -------------
// Giant tasks (a read inside a tandem array: 10^5..10^6 anchors) are serial in the formulations above: one warp walks
// the anchors one by one.  But anchor i depends on anchor j only if j is a CANDIDATE predecessor of i (it passes the
// three `continue`s of src/chain.c:61-73) -- a purely geometric property of a[] -- because a non-candidate touches
// neither max_f nor n_skip nor t[].  In a tandem lattice consecutive anchors mostly lie on different diagonals and
// are not candidates of each other.  So the CTA runs 32 warps; warp k owns anchors k, k + 32, k + 64, ... (anchor
// i0 + k of every 32-anchor tile).  There is no barrier in the loop: the warps drift apart as far as the dependencies allow.
// The scan of an anchor is split in two phases:
//  (A) list: before it waits for anything, the warp walks the window (32 predecessors per step; coordinates from the ring
//      for anchors three tiles back and older, which are complete, else from a[], which never changes) and appends the candidates, in scan order, with their scores without f[j] (the same wm_chain_score),
//      to its list in shared memory, until the list is full or the window is exhausted.  The steps over its own tile and
//      the tile before are tile aligned, so their ballots are also the sets of anchors there that anchor i depends on.
//  (B) resolve: the warp waits until exactly those have published f / p / v (done-masks in shared memory; anchors two
//      tiles back and older are complete by construction: a warp enters tile T only when tile T - 2 is complete), then
//      resolves the list 32 entries per step: f[j] and p[j] from the ring, the marks, the order-dependent part.  If the
//      list runs out before the reference's loop ends, the warp refills it from where phase A stopped and goes on.
// The list holds the first candidates in scan order and nothing else: a non-candidate touches neither max_f nor n_skip nor
// t[], and marks published for an entry can only reach indices below every entry before it (p[j] < j), so resolving the
// list in 32-entry steps gives what resolving the window in 32-predecessor steps gave.  The t[p[j]] = i marks of the
// reference are per-anchor state, so every warp keeps its own in a bitset over the ring window.  A scan that needs f / p or
// a mark below the ring (rare: it covers the last ~4000 anchors) is redone under a CTA-wide lock with the global arrays.
#define WM_CT_WARPS 32
#ifdef WM_HOST_EMUL
#define WM_LDCG(p) (*(p))
#else
#define WM_LDCG(p) __ldcg(p)
#endif
#ifndef WM_CT_RING
#define WM_CT_RING 4096 // (the single-warp emulation of the tests builds with a small ring to force the locked deep path; their CTA emulation keeps this one)
#endif
// List capacity per warp.  On tandem lattices with the map-ont options the reference's loop consumes 35 candidates per
// anchor in the median, 43 at the 99th percentile (tools/bench_chain.py --counts); a longer list would only make phase A
// test predecessors past the break.
#define WM_CT_LIST 48
struct wm_chain_tile_sm {
	uint64_t x[WM_CT_RING];
	int32_t q[WM_CT_RING], f[WM_CT_RING], p[WM_CT_RING], v[WM_CT_RING];
	uint32_t marks[WM_CT_WARPS][WM_CT_RING / 32];
	int2 list[WM_CT_WARPS][WM_CT_LIST]; // per warp: (j, score of j without f[j]) of the listed candidates, in scan order
	unsigned done[8];  // done[T & 7]: which anchors of tile T have published
	int lock;
};

// per-scan state of one anchor
struct wm_chain_scan {
	uint64_t ri; int32_t qi, q_span;
	int i, max_f, max_j, n_skip;
};

// the order-dependent part of a 32-entry step (running maximum with strict ">", n_skip replay): lane m holds the m-th
// entry in scan order (predecessor j), its score sc if it is a candidate, and whether it carries this anchor's mark.
// Returns true when the reference leaves its loop inside this step.
__device__ __forceinline__ bool wm_chain_resolve(wm_chain_scan &A, bool cand, int sc, bool marked, int j, int max_skip, int lane)
{
	const unsigned FULL = 0xffffffffu;
	const unsigned G = __ballot_sync(FULL, cand && sc > A.max_f);
	unsigned Rm = G;
	if (G & (G - 1)) { // two or more lanes beat the running maximum: the records are the prefix maxima among them
		const int incl = wm_warp_incl_max(cand ? sc : INT_MIN, lane);
		int excl = __shfl_up_sync(FULL, incl, 1);
		if (lane == 0) excl = INT_MIN;
		excl = max(excl, A.max_f);
		Rm = __ballot_sync(FULL, cand && sc > excl);
	}
	const unsigned K = __ballot_sync(FULL, marked) & ~Rm;
	const int brk = wm_chain_replay(Rm, K, &A.n_skip, max_skip);
	const unsigned Rv = brk < 32 ? (Rm & ((1u << brk) - 1u)) : Rm;
	if (Rv) {
		const int top = 31 - __clz(Rv);
		A.max_f = __shfl_sync(FULL, sc, top);
		A.max_j = __shfl_sync(FULL, j, top);
	}
	return brk < 32;
}

// Appends one step's candidates (lane: c, its predecessor j, its score s0, `before` = candidates of the step ahead of it in scan
// order) to the list L, which holds *cnt of at most cap entries.  Returns the predecessor of the first candidate that did not fit
// (INT_MIN if all did).
__device__ __forceinline__ int wm_chain_list_append(int2 *L, int *cnt, int cap, bool c, int j, int s0, unsigned m, int before)
{
	const int r = *cnt + before;
	if (c && r < cap) L[r] = make_int2(j, s0);
	const int room = cap - *cnt, nm = __popc(m);
	if (nm <= room) { *cnt += nm; return INT_MIN; }
	*cnt = cap;
	const unsigned o = __ballot_sync(0xffffffffu, c && r == cap);
	return __shfl_sync(0xffffffffu, j, __ffs(o) - 1);
}

// Coordinates of predecessor j for an anchor of the tile that starts at i0.  Anchors of tile T - 3 and older are complete before
// a warp enters tile T (it waited for tile T - 3 on entering T - 1), and the slots at or above ring_lo are not reused before tile
// T + 2, which needs tile T complete: those come from the ring.  Everything else comes from a[].
__device__ __forceinline__ wm128_dev wm_chain_coords(const wm128_dev *__restrict__ a, const wm_chain_tile_sm *S, int j, int i0, int ring_lo)
{
	if (j >= ring_lo && j < i0 - 64) {
		const int s = j & (WM_CT_RING - 1);
		wm128_dev aj; aj.x = S->x[s], aj.y = (uint64_t)(uint32_t)S->q[s];
		return aj;
	}
	return a[j];
}

// Phase A from predecessor jtop down: lane m looks at j = jtop - m, 32 per step, until the list is full or the window is
// exhausted.  Returns the next predecessor to look at (< st: the window is exhausted).
template <bool CDNA = false>
__device__ __forceinline__ int wm_chain_list_fill(const wm128_dev *__restrict__ a, const wm_chain_tile_sm *S, const wm_chain_scan &A, const wm_chain_params &P,
                                                  int2 *L, int *cnt, int cap, int jtop, int st, int i0, int ring_lo, double avg_d, double scale_d, int lane)
{
	while (jtop >= st && *cnt < cap) {
		const int j = jtop - lane;
		int s0 = 0;
		const bool c = j >= st && wm_chain_score<CDNA>(wm_chain_coords(a, S, j, i0, ring_lo), A.ri, A.qi, A.q_span, P, avg_d, scale_d, &s0);
		const unsigned m = __ballot_sync(0xffffffffu, c);
		const int jr = wm_chain_list_append(L, cnt, cap, c, j, s0, m, __popc(m & ((1u << lane) - 1u)));
		if (jr != INT_MIN) return jr;
		jtop -= 32;
	}
	return jtop;
}

// Phase A of anchor i = i0 + k, the part that waits for nothing.  cur / prev: lane l holds a[i0 + l] / a[i0 - 32 + l].  The first
// two steps cover the two register tiles, tile aligned (lane l looks at i0 + l, then at i0 - 32 + l; scan order is descending
// lane order): *Cc / *Cp receive the candidates among them, which are what anchor i has to wait for.  Returns the next predecessor
// to look at; *cnt receives the length of the list.
template <bool CDNA = false>
__device__ __forceinline__ int wm_chain_list_begin(const wm128_dev *__restrict__ a, const wm_chain_tile_sm *S, const wm_chain_scan &A, const wm_chain_params &P,
                                                   int2 *L, int cap, wm128_dev cur, wm128_dev prev, int i0, int k, int st, int ring_lo, double avg_d, double scale_d,
                                                   int lane, int *cnt, unsigned *Cc, unsigned *Cp)
{
	const unsigned FULL = 0xffffffffu;
	*cnt = 0;
	int jr = INT_MIN;
	{
		const int j = i0 + lane;
		int s0 = 0;
		const bool c = lane < k && j >= st && wm_chain_score<CDNA>(cur, A.ri, A.qi, A.q_span, P, avg_d, scale_d, &s0);
		const unsigned m = __ballot_sync(FULL, c);
		*Cc = m;
		jr = wm_chain_list_append(L, cnt, cap, c, j, s0, m, __popc(m >> lane >> 1));
	}
	{
		const int j = i0 - 32 + lane;
		int s0 = 0;
		const bool c = j >= st && wm_chain_score<CDNA>(prev, A.ri, A.qi, A.q_span, P, avg_d, scale_d, &s0);
		const unsigned m = __ballot_sync(FULL, c);
		*Cp = m;
		if (jr == INT_MIN) jr = wm_chain_list_append(L, cnt, cap, c, j, s0, m, __popc(m >> lane >> 1));
	}
	if (jr != INT_MIN) return jr;
	return wm_chain_list_fill<CDNA>(a, S, A, P, L, cnt, cap, i0 - 33, st, i0, ring_lo, avg_d, scale_d, lane);
}

// Phase B of the scan of anchor A.i: the list (cnt entries, next predecessor jr) was made by wm_chain_list_begin, and every
// listed entry at or above ring_lo has published.  f / p of entries j >= ring_lo come from the ring; older ones from global
// memory, and only when deep_ok (the caller holds the lock: the global t[] marks are then this anchor's alone).  Returns false
// if it would have had to go below the ring without deep_ok; on success A.max_f / A.max_j hold f[i] / p[i].
template <bool CDNA = false>
__device__ __forceinline__ bool wm_chain_list_resolve(const wm128_dev *__restrict__ a, const wm_chain_params &P, const int32_t *f, const int32_t *p, int32_t *t,
                                                      wm_chain_tile_sm *S, uint32_t *mk, int2 *L, int cap, wm_chain_scan &A, int cnt, int jr, int st, int i0,
                                                      int ring_lo, bool deep_ok, double avg_d, double scale_d, int lane)
{
	const unsigned FULL = 0xffffffffu;
	constexpr int MASK = WM_CT_RING - 1;
	A.max_f = A.q_span, A.max_j = -1, A.n_skip = 0;
	for (int w = lane; w < WM_CT_RING / 32; w += 32) mk[w] = 0;
	__syncwarp();
	for (;;) {
		for (int e = 0; e < cnt; e += 32) {
			const bool cand = e + lane < cnt;
			int j = -1, sc = INT_MIN;
			bool need_deep = false;
			if (cand) {
				const int2 E = L[e + lane];
				int fj = 0, pj = -1;
				j = E.x;
				if (j >= ring_lo) { const int s = j & MASK; fj = S->f[s]; pj = S->p[s]; }
				else if (deep_ok) { fj = WM_LDCG(f + j); pj = WM_LDCG(p + j); } // written by other warps of the CTA: read at L2
				else need_deep = true;
				sc = E.y + fj;
				if (pj >= 0) { // src/chain.c:87
					if (pj >= ring_lo) atomicOr(&mk[(pj & MASK) >> 5], 1u << (pj & 31));
					else if (deep_ok) t[pj] = A.i;
					else need_deep = true;
				}
			}
			if (__ballot_sync(FULL, need_deep)) return false;
			__syncwarp();
			bool marked = false;
			if (cand) marked = j >= ring_lo ? (mk[(j & MASK) >> 5] >> (j & 31) & 1) != 0 : t[j] == A.i;
			if (wm_chain_resolve(A, cand, sc, marked, j, P.max_skip, lane)) return true;
		}
		if (jr < st) return true;
		// the list ran out before the reference's loop ended: go on from where it stopped (everything that can be a candidate
		// of anchor i has published by now)
		__syncwarp();
		cnt = 0;
		jr = wm_chain_list_fill<CDNA>(a, S, A, P, L, &cnt, cap, jr, st, i0, ring_lo, avg_d, scale_d, lane);
		__syncwarp();
	}
}

struct wm_chain_no_wait { __device__ void operator()(unsigned, unsigned) const {} };

// The scan of anchor i = i0 + k by warp k: phase A into the warp's list S->list[k] (at most cap entries), then wait(Cc, Cp) with the
// candidates of the two register tiles (cur / prev: lane l holds a[i0 + l] / a[i0 - 32 + l]), then phase B.  Returns false if it
// would have had to go below the ring without deep_ok; on success *mf / *mj hold f[i] / p[i].
template <bool CDNA = false, class Wait = wm_chain_no_wait>
__device__ __forceinline__ bool wm_chain_tile_scan(const wm128_dev *__restrict__ a, const wm_chain_params &P, const int32_t *f, const int32_t *p, int32_t *t,
                                                   wm_chain_tile_sm *S, uint32_t *mk, wm128_dev cur, wm128_dev prev, int i0, int k, int st, int ring_lo, bool deep_ok,
                                                   double avg_d, double scale_d, int lane, int *mf, int *mj, Wait wait = Wait(), int cap = WM_CT_LIST)
{
	const unsigned FULL = 0xffffffffu;
	wm_chain_scan A;
	A.i = i0 + k, A.ri = __shfl_sync(FULL, cur.x, k);
	{ const uint64_t yi = __shfl_sync(FULL, cur.y, k); A.qi = (int32_t)yi, A.q_span = (int32_t)(yi >> 32 & 0xff); }
	int2 *L = S->list[k];
	int cnt; unsigned Cc, Cp;
	const int jr = wm_chain_list_begin<CDNA>(a, S, A, P, L, cap, cur, prev, i0, k, st, ring_lo, avg_d, scale_d, lane, &cnt, &Cc, &Cp);
	wait(Cc, Cp);
	if (!wm_chain_list_resolve<CDNA>(a, P, f, p, t, S, mk, L, cap, A, cnt, jr, st, i0, ring_lo, deep_ok, avg_d, scale_d, lane)) return false;
	*mf = A.max_f, *mj = A.max_j;
	return true;
}

// ---- backtracking (src/chain.c:92-165) by a group of threads: one warp (tasks of ordinary size) or one CTA (giant tasks) ----
template <bool CTA> __device__ __forceinline__ void wm_grp_sync()
{
#ifndef WM_HOST_EMUL
	if (CTA) __syncthreads(); else
#endif
	__syncwarp();
}

// descending bitonic sort of m (power of two) uint64 keys by the group
template <bool CTA>
__device__ void wm_grp_bitonic_desc(uint64_t *x, int m, int tid, int G)
{
	for (int k = 2; k <= m; k <<= 1)
		for (int j = k >> 1; j > 0; j >>= 1) {
			for (int i = tid; i < m; i += G) {
				const int l = i ^ j;
				if (l > i) {
					const uint64_t a = x[i], b = x[l];
					const bool up = (i & k) == 0; // first half of each k-block sorted descending
					if (up ? a < b : a > b) x[i] = b, x[l] = a;
				}
			}
			wm_grp_sync<CTA>();
		}
}

// exclusive prefix of (a, b) over the threads of the group; *ta / *tb receive the totals.  sm: 64 ints of shared memory (CTA only)
template <bool CTA>
__device__ __forceinline__ void wm_grp_scan2(int &a, int &b, int *ta, int *tb, int tid, int *sm)
{
	const unsigned FULL = 0xffffffffu;
	const int lane = tid & 31;
	int ia = a, ib = b;
	#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const int xa = __shfl_up_sync(FULL, ia, o), xb = __shfl_up_sync(FULL, ib, o);
		if (lane >= o) ia += xa, ib += xb;
	}
	int base_a = 0, base_b = 0, tot_a = __shfl_sync(FULL, ia, 31), tot_b = __shfl_sync(FULL, ib, 31);
#ifndef WM_HOST_EMUL
	if (CTA) {
		const int w = tid >> 5, nw = (int)(blockDim.x >> 5);
		if (lane == 31) sm[w] = ia, sm[32 + w] = ib;
		__syncthreads();
		tot_a = tot_b = 0;
		for (int k = 0; k < nw; ++k) { if (k == w) base_a = tot_a, base_b = tot_b; tot_a += sm[k]; tot_b += sm[32 + k]; }
		__syncthreads();
	}
#endif
	a = base_a + ia - a, b = base_b + ib - b;
	*ta = tot_a, *tb = tot_b;
}

// Backtracking of one task (src/chain.c:92-165).  On return a[] holds the chained anchors (*n_b_out of them), u2[] the
// (score << 32 | count) words (*n_u_out); both counts are 0 if there is no chain.  u has 2n entries, *n_u_out must be 0 on entry
// (it serves as the counter of the chain starts).
// The reference takes the chain starts in score order and lets each claim its path of predecessors up to the first anchor
// that is claimed already (:118-135).  That walk is order dependent only through "claimed by a better start": anchor x ends up
// with the best-ranked start among those whose path reaches it, so every start walks its path concurrently with an atomicMin
// of its rank and stops at the first anchor that already carries a better one.  The first anchor of a start is taken even
// when it is claimed (the do-while of :121-125).
template <bool CTA>
__device__ void wm_chain_backtrack_grp(wm128_dev *a, int n, const wm_chain_params &P, int32_t *f, int32_t *p, int32_t *t, int32_t *v,
                                       uint64_t *u, uint64_t *u2, wm128_dev *w, wm128_dev *b, wm_rs_warp_ws *W, int32_t *n_u_out, int64_t *n_b_out,
                                       int tid, int G, int *sm)
{
	// chain starts (:93-110): anchors that are nobody's predecessor and whose peak score passes; from each, back to the peak of f[]
	for (int i = tid; i < n; i += G) t[i] = 0;
	wm_grp_sync<CTA>();
	for (int i = tid; i < n; i += G) if (p[i] >= 0) t[p[i]] = 1;
	wm_grp_sync<CTA>();
	for (int i = tid; i < n; i += G)
		if (t[i] == 0 && v[i] >= P.min_sc) {
			int j = i;
			while (j >= 0 && f[j] < v[j]) j = p[j];
			if (j < 0) j = i;
			u[atomicAdd(n_u_out, 1)] = (uint64_t)(uint32_t)f[j] << 32 | (uint32_t)j;
		}
	wm_grp_sync<CTA>();
	const int n_e = *n_u_out;
	wm_grp_sync<CTA>();
	if (tid == 0) *n_u_out = 0, *n_b_out = 0;
	if (n_e == 0) { wm_grp_sync<CTA>(); return; } // :99-102
	{ // :112-116 best first.  Equal words are the same (score, anchor) pair, so any correct sort gives the reference's sequence.
		int m = 1; while (m < n_e) m <<= 1;
		for (int i = n_e + tid; i < m; i += G) u[i] = 0;
		wm_grp_sync<CTA>();
		wm_grp_bitonic_desc<CTA>(u, m, tid, G);
	}
	// owners: t[x] = rank of the best start that claims x
	for (int i = tid; i < n; i += G) t[i] = INT_MAX;
	wm_grp_sync<CTA>();
	for (int r = tid; r < n_e; r += G) {
		int j = (int32_t)u[r];
		while (j >= 0) {
			if (atomicMin(&t[j], r) < r) break;
			j = p[j];
		}
	}
	wm_grp_sync<CTA>();
	// length, score and fate of every start (:119-134); w[r] = { score << 32 | count (0: dropped), first anchor }
	for (int r = tid; r < n_e; r += G) {
		const int s0 = (int32_t)u[r];
		int cnt = 1, j = p[s0];
		if (t[s0] == r) while (j >= 0 && t[j] == r) ++cnt, j = p[j];
		const int32_t sc = j < 0 ? (int32_t)(u[r] >> 32) : (int32_t)(u[r] >> 32) - f[j];
		const bool keep = (j < 0 || sc >= P.min_sc) && cnt >= P.min_cnt;
		w[r].x = keep ? (uint64_t)(uint32_t)sc << 32 | (uint32_t)cnt : 0;
		w[r].y = (uint64_t)(uint32_t)s0;
	}
	wm_grp_sync<CTA>();
	// chain index and anchor offset of the kept starts, in rank order (:130-133, :141-147): a prefix over contiguous blocks of
	// ranks, kept per rank (t[r] = chain index, upper half of w[r].y = offset) so that the copies below can be dealt round-robin
	// (the best-ranked chains are the longest: a block of consecutive ranks per thread would leave all of them to thread 0)
	int n_u = 0, n_v = 0;
	{
		const int L = (n_e + G - 1) / G, r0 = tid * L < n_e ? tid * L : n_e, r1 = r0 + L < n_e ? r0 + L : n_e;
		int kc = 0, ac = 0;
		for (int r = r0; r < r1; ++r) if (w[r].x) ++kc, ac += (int32_t)w[r].x;
		wm_grp_scan2<CTA>(kc, ac, &n_u, &n_v, tid, sm);
		for (int r = r0; r < r1; ++r)
			if (w[r].x) { t[r] = kc; w[r].y |= (uint64_t)(uint32_t)ac << 32; ++kc; ac += (int32_t)w[r].x; }
	}
	wm_grp_sync<CTA>();
	if (n_u == 0) { wm_grp_sync<CTA>(); return; }
	// the chains into b[], each in ascending anchor order (:141-147); u[k] / v[k]: (score << 32 | count) and offset of chain k
	for (int r = tid; r < n_e; r += G)
		if (w[r].x) {
			const int cnt = (int32_t)w[r].x, off = (int32_t)(w[r].y >> 32), k = t[r];
			int j = (int32_t)w[r].y;
			for (int m = cnt - 1; m >= 0; --m) { b[off + m] = a[j]; j = p[j]; }
			u2[k] = w[r].x; v[k] = off;
		}
	wm_grp_sync<CTA>();
	// :150-155 chains ordered by the position of their first anchor (tie-exact sort of the reference)
	for (int k = tid; k < n_u; k += G) { w[k].x = b[v[k]].x; w[k].y = (uint64_t)(uint32_t)v[k] << 32 | (uint32_t)k; u[k] = u2[k]; }
	wm_grp_sync<CTA>();
	if (tid < 32) wm_radix_sort_warp(w, n_u, W, (wm_rs_range*)(u + n), tid);
	wm_grp_sync<CTA>();
	// :156-164 the chains in that order: offsets by a second prefix (t[i] = where chain i of the new order starts), then the copies
	{
		const int L2 = (n_u + G - 1) / G, k0 = tid * L2 < n_u ? tid * L2 : n_u, k1 = k0 + L2 < n_u ? k0 + L2 : n_u;
		int dummy = 0, off = 0, td, toff;
		for (int i = k0; i < k1; ++i) off += (int32_t)u[(int32_t)w[i].y];
		wm_grp_scan2<CTA>(dummy, off, &td, &toff, tid, sm);
		for (int i = k0; i < k1; ++i) { t[i] = off; off += (int32_t)u[(int32_t)w[i].y]; }
	}
	wm_grp_sync<CTA>();
	for (int i = tid; i < n_u; i += G) {
		const int j = (int32_t)w[i].y, nn = (int32_t)u[j], off = t[i];
		const wm128_dev *src = b + (w[i].y >> 32);
		u2[i] = u[j];
		for (int l = 0; l < nn; ++l) a[off + l] = src[l];
	}
	wm_grp_sync<CTA>();
	if (tid == 0) *n_u_out = n_u, *n_b_out = n_v;
	wm_grp_sync<CTA>();
}
