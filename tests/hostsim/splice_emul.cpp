// TEST INFRASTRUCTURE.  The chaining forward pass of csrc/chain_dev.cuh with the gap cost of is_cdna = 1 (the CDNA instantiations the
// kernels of csrc/chain.cu launch for spliced mapping) on the software warp of cuda_emul.h, and the scalar restatement of the reference's
// loop with that gap cost, the yardstick.  Links against libwm_hostsim.so (kernel_emul.cpp), which provides the fiber runtime; built by
// tests/splice_lib.py.
#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#define WM_CT_RING 128 // small ring: the tile formulation goes through its locked deep path all the time
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/wm_common.cuh"
#include "../../winnowmap_b200/csrc/chain_dev.cuh"

#define WMT_API extern "C" __attribute__((visibility("default")))

namespace {
// the shared-memory ring formulation: window starts first (closed form), then the sweep
template <int RING>
void run_ring(const wm128_dev *a, int n, const wm_chain_params *P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int lane)
{
	static thread_local wm_chain_ring<RING> *ring = 0;
	if (lane == 0) { if (!ring) ring = new wm_chain_ring<RING>(); memset(ring, 0xff, sizeof(*ring)); }
	for (int i = lane; i < n; i += 32) v[i] = wm_chain_window_start(a, i, *P);
	__syncwarp();
	wm_chain_fill_warp_ring<RING, true>(a, n, *P, f, p, t, v, ring, lane);
}

// the tile formulation: what one CTA of the giant-task kernel does, the 32 anchors of a tile taken in order by one software warp (the
// order satisfies every dependency), with lists of cap entries
void run_tile(const wm128_dev *a, int n, const wm_chain_params *P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int cap, int lane)
{
	static thread_local wm_chain_tile_sm *S = 0;
	constexpr int MASK = WM_CT_RING - 1;
	if (lane == 0) { if (!S) S = new wm_chain_tile_sm(); memset(S, 0xff, sizeof(*S)); }
	unsigned long long sum = 0;
	for (int i = 0; i < n; ++i) sum += a[i].y >> 32 & 0xff;
	for (int i = lane; i < n; i += 32) { v[i] = wm_chain_window_start(a, i, *P); t[i] = 0; }
	const float avg_qspan = (float)sum / (float)(long long)n;
	const double avg_d = (double)avg_qspan, scale_d = (double)P->gap_scale;
	__syncwarp();
	wm128_dev prev; prev.x = prev.y = 0;
	for (int i0 = 0; i0 < n; i0 += 32) {
		const int il = i0 + lane;
		wm128_dev al; al.x = al.y = 0; int stl = 0;
		if (il < n) { al = a[il]; stl = v[il]; }
		for (int k = 0; k < 32 && i0 + k < n; ++k) {
			const int i = i0 + k, st = __shfl_sync(0xffffffffu, stl, k), ring_lo = i0 + 64 - WM_CT_RING;
			int max_f = 0, max_j = -1;
			if (!wm_chain_tile_scan<true>(a, *P, f, p, t, S, S->marks[k], al, prev, i0, k, st, ring_lo, false, avg_d, scale_d, lane, &max_f, &max_j,
			                              wm_chain_no_wait(), cap))
				wm_chain_tile_scan<true>(a, *P, f, p, t, S, S->marks[k], al, prev, i0, k, st, ring_lo, true, avg_d, scale_d, lane, &max_f, &max_j,
				                         wm_chain_no_wait(), cap);
			int vj = INT_MIN;
			if (max_j >= 0) vj = max_j >= ring_lo ? S->v[max_j & MASK] : v[max_j];
			const int vi = (max_j >= 0 && vj > max_f) ? vj : max_f;
			const uint64_t xi = __shfl_sync(0xffffffffu, al.x, k), yi = __shfl_sync(0xffffffffu, al.y, k);
			__syncwarp();
			if (lane == 0) { const int s = i & MASK; S->x[s] = xi, S->q[s] = (int32_t)yi, S->f[s] = max_f, S->p[s] = max_j, S->v[s] = vi; f[i] = max_f; p[i] = max_j; v[i] = vi; }
			__syncwarp();
		}
		prev = al;
	}
}

struct Args { const wm128_dev *a; int n; const wm_chain_params *P; int32_t *f, *p, *t, *v, *D; int mode, cap; };

void run_fill(int l, void *q)
{
	Args &x = *(Args*)q;
	if (x.mode == 1) wm_chain_fill_warp_dense<true>(x.a, x.n, *x.P, x.f, x.p, x.t, x.v, x.D, l);
	else if (x.mode == 2) run_ring<64>(x.a, x.n, x.P, x.f, x.p, x.t, x.v, l);
	else if (x.mode == 3) run_ring<1024>(x.a, x.n, x.P, x.f, x.p, x.t, x.v, l);
	else if (x.mode == 4) run_tile(x.a, x.n, x.P, x.f, x.p, x.t, x.v, x.cap, l);
	else wm_chain_fill_warp<true>(x.a, x.n, *x.P, x.f, x.p, x.t, x.v, l);
}
} // namespace

// f / p / v of the forward pass with the cDNA gap cost on the software warp (a is n anchors, x then y).  mode: 0 the plain warp loop,
// 1 dense candidates, 2 / 3 the shared-memory ring of 64 / 1024 slots (64: the older-than-the-ring path), 4 the tile formulation with
// lists of cap entries (1 <= cap <= WM_CT_LIST) and a 128-slot ring (the locked deep path).  -1 on bad arguments.
WMT_API int wmt_emul_chain_fill_cdna(const uint64_t *a_xy, int n, int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                                     float gap_scale, int mode, int cap, int32_t *f, int32_t *p, int32_t *v)
{
	if (n <= 0) return 0;
	if (mode < 0 || mode > 4 || cap < 1 || cap > WM_CT_LIST) return -1;
	std::vector<wm128_dev> a((size_t)n + 1);
	for (int i = 0; i < n; ++i) a[i].x = a_xy[2 * i], a[i].y = a_xy[2 * i + 1];
	wm_chain_params P; memset(&P, 0, sizeof(P));
	P.max_dist_x = max_dist_x, P.min_dist_x = min_dist_x, P.max_dist_y = max_dist_y, P.bw = bw, P.max_skip = max_skip, P.max_iter = max_iter;
	P.gap_scale = gap_scale;
	std::vector<int32_t> t((size_t)n + 1, 0), D(WM_CHAIN_DENSE_CAP, 0);
	Args A = { a.data(), n, &P, f, p, t.data(), v, D.data(), mode, cap };
	wm_emul::run_warp(run_fill, &A);
	return 0;
}

// Scalar restatement of the forward pass of mm_chain_dp (src/chain.c:41-90, n_segs == 1) with is_cdna = 1: an anchor pair whose gap
// is longer on the reference than on the query (an intron) costs min(c_lin, c_log), any other c_lin + c_log / 2 (chain.c:69-77).
// is_cdna = 0 gives the plain gap cost, for comparison.
WMT_API int wmt_chain_fill_scalar_gap(const uint64_t *a_xy, int n, int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                                      float gap_scale, int is_cdna, int32_t *f, int32_t *p, int32_t *v)
{
	if (n <= 0) return 0;
	std::vector<int32_t> t((size_t)n, 0);
	uint64_t sum_qspan = 0;
	for (int i = 0; i < n; ++i) sum_qspan += a_xy[2 * i + 1] >> 32 & 0xff;
	const float avg_qspan = (float)sum_qspan / n;
	int st = 0;
	for (int i = 0; i < n; ++i) {
		const uint64_t ri = a_xy[2 * i];
		const int32_t qi = (int32_t)a_xy[2 * i + 1], q_span = (int32_t)(a_xy[2 * i + 1] >> 32 & 0xff);
		int32_t max_f = q_span, max_j = -1, n_skip = 0;
		while (st < i && ri > a_xy[2 * st] + (uint64_t)(int64_t)max_dist_x) ++st;
		if (i - st > max_iter)
			while (i - st > max_iter && ri > a_xy[2 * st] + (uint64_t)(int64_t)min_dist_x) ++st;
		for (int j = i - 1; j >= st; --j) {
			const int64_t dr = (int64_t)(ri - a_xy[2 * j]);
			const int32_t dq = qi - (int32_t)a_xy[2 * j + 1];
			if (dr == 0 || dq <= 0) continue;
			if (dq > max_dist_y || dq > max_dist_x) continue;
			const int32_t dd = (int32_t)(dr > dq ? dr - dq : dq - dr);
			if (dd > bw) continue;
			const int32_t min_d = dq < dr ? dq : (int32_t)dr;
			int32_t sc = min_d > q_span ? q_span : min_d;
			const int c_log = dd ? 31 - __builtin_clz((unsigned)dd) : 0, c_lin = (int)(dd * .01 * avg_qspan);
			const int gap_cost = is_cdna && dr > dq ? (c_lin < c_log ? c_lin : c_log) : c_lin + (c_log >> 1);
			sc -= (int)((double)gap_cost * gap_scale + .499);
			sc += f[j];
			if (sc > max_f) { max_f = sc, max_j = j; if (n_skip > 0) --n_skip; }
			else if (t[j] == i) { if (++n_skip > max_skip) break; }
			if (p[j] >= 0) t[p[j]] = i;
		}
		f[i] = max_f, p[i] = max_j;
		v[i] = max_j >= 0 && v[max_j] > max_f ? v[max_j] : max_f;
	}
	return 0;
}
