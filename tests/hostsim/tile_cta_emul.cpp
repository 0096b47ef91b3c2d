// TEST INFRASTRUCTURE.  The CTA body of the giant-task chaining kernel (csrc/chain_tile.cuh: wm_chain_fill_tile_cta, all of
// wm_chain_fill_tile_kernel) on an emulated CTA of WM_CT_WARPS software warps (cuda_emul.h: run_cta), at the kernel's own ring and list
// sizes, under a warp schedule chosen by the caller; and, at the same constants, which paths of that kernel each anchor's scan takes
// (from the scalar restatement of the reference's loop).  Build with build_tile_cta.sh: the product's headers come from the include
// path, so a modified copy of them can be built the same way.  Links against libwm_hostsim.so (kernel_emul.cpp), which provides the
// fiber runtime.
#include <stdio.h>
#include <stdlib.h>
#include <string>
#include <vector>
#include "cuda_emul.h"
#include "wm_common.cuh"
#include "chain_tile.cuh"

#define WMT_API extern "C" __attribute__((visibility("default")))

namespace {
struct Run {
	const wm128_dev *a; const int64_t *off; const int32_t *order; int n_tasks; const int32_t *n;
	wm_chain_params2 PP; const uint8_t *set_id;
	int32_t *f, *p, *t, *v; int counter;
	wm_chain_tile_sm *S; int s_task; unsigned long long s_sum[WM_CT_WARPS];
	// statistics from the atomic operations: the lock's compare-and-swaps, and the publishes on the done-masks.  Warp k's c-th
	// publish in a task is its anchor of tile c (it publishes every tile that has an anchor k), so the trace gives, per task and
	// tile, how many anchors have published, and the largest number of tiles that held published and unpublished anchors at once.
	long long lock_ok, lock_fail, publishes;
	int partial, max_partial;
	int task_of[WM_CT_WARPS], tile_of[WM_CT_WARPS];
	std::vector<std::vector<int>> pub; // per task (in CTA order) and tile: anchors published
};

int tiles_of_warp(int n, int k) { return n > k ? (n - k + 31) / 32 : 0; }

// what the warps of the kernel wait for: the done-masks and the lock (the other atomics set a warp's own marks)
bool on_atomic(void *user, int kind, int w, const void *addr, unsigned long long, bool ok)
{
	Run &R = *(Run*)user;
	if (addr == &R.S->lock) { if (kind == wm_emul::ATOM_CAS) ++(ok ? R.lock_ok : R.lock_fail); return true; }
	const unsigned *d = R.S->done;
	if (addr < (const void*)d || addr >= (const void*)(d + 8)) return false;
	if (kind != wm_emul::ATOM_OR) return true;
	++R.publishes;
	int &tk = R.task_of[w], &c = R.tile_of[w];
	while (tk < R.n_tasks && c == tiles_of_warp(R.n[R.order[tk]], w)) ++tk, c = 0;
	if (tk >= R.n_tasks) { R.max_partial = 1 << 20; return true; } // more publishes than anchors: reported as a bound violation
	const int n = R.n[R.order[tk]], full = n - 32 * c < 32 ? n - 32 * c : 32;
	const int before = R.pub[tk][c]++;
	R.partial += (before + 1 < full) - (before > 0 && before < full);
	if (R.partial > R.max_partial) R.max_partial = R.partial;
	++c;
	return true;
}

void body(int tid, void *arg)
{
	Run &R = *(Run*)arg;
	wm_chain_fill_tile_cta(R.a, R.off, R.order, 0, R.n_tasks, R.PP, R.set_id, R.f, R.p, R.t, R.v, &R.counter, R.S, &R.s_task, R.s_sum, tid);
}

wm_chain_params make_params(const int32_t *q, float gap_scale)
{
	wm_chain_params P; memset(&P, 0, sizeof(P));
	P.max_dist_x = q[0], P.min_dist_x = q[1], P.max_dist_y = q[2], P.bw = q[3], P.max_skip = q[4], P.max_iter = q[5];
	P.gap_scale = gap_scale;
	return P;
}
} // namespace

// Forward pass of n_tasks anchor arrays (task t: anchors off[t] .. off[t + 1] of a_xy, x then y) by one emulated CTA, which takes the
// tasks in the given order.  prm: two parameter sets of 6 ints (max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter), set_id[t]
// picks one per task.  sched / sched_warp / seed: cuda_emul.h SCHED_*.  Outputs f / p / v per anchor and stats[10]: deep scans
// (successful lock acquisitions), failed lock attempts, polls, most tiles partly published at once, anchors published, completed syncs,
// warp switches, retry rounds (every warp blocked), events, deadlock (0/1).  Returns 0, -1 after a deadlock (err: each warp's tile and
// anchor), -2 on bad arguments.
WMT_API int wmt_tile_cta(const uint64_t *a_xy, const int64_t *off, int n_tasks, const int32_t *order, const int32_t *prm, float gap_scale,
                         const uint8_t *set_id, int sched, int sched_warp, uint64_t seed, int32_t *f, int32_t *p, int32_t *v, int64_t *stats,
                         char *err, int err_len)
{
	if (n_tasks <= 0 || sched_warp < 0 || sched_warp >= WM_CT_WARPS) return -2;
	const int64_t n_all = off[n_tasks];
	std::vector<wm128_dev> a((size_t)n_all + 1);
	for (int64_t i = 0; i < n_all; ++i) a[i].x = a_xy[2 * i], a[i].y = a_xy[2 * i + 1];
	std::vector<int32_t> n(n_tasks), t((size_t)n_all + 1, 0);
	Run R; memset(R.s_sum, 0, sizeof(R.s_sum));
	R.PP.p[0] = make_params(prm, gap_scale), R.PP.p[1] = make_params(prm + 6, gap_scale);
	for (int k = 0; k < n_tasks; ++k) {
		n[k] = (int)(off[k + 1] - off[k]);
		if (n[k] < 0 || set_id[k] > 1) return -2;
		const wm_chain_params &P = R.PP.p[set_id[k]];
		for (int i = 0; i < n[k]; ++i) v[off[k] + i] = wm_chain_window_start(a.data() + off[k], i, P); // wm_chain_window_kernel
	}
	R.a = a.data(), R.off = off, R.order = order, R.n_tasks = n_tasks, R.n = n.data(), R.set_id = set_id;
	R.f = f, R.p = p, R.t = t.data(), R.v = v, R.counter = 0;
	R.S = new wm_chain_tile_sm();
	memset(R.S, 0xff, sizeof(*R.S)); // whatever the previous user of the shared memory left
	R.s_task = -1;
	R.lock_ok = R.lock_fail = R.publishes = 0, R.partial = R.max_partial = 0;
	for (int k = 0; k < WM_CT_WARPS; ++k) R.task_of[k] = 0, R.tile_of[k] = 0;
	R.pub.resize(n_tasks);
	for (int k = 0; k < n_tasks; ++k) R.pub[k].assign((n[order[k]] + 31) / 32, 0);
	wm_emul::Cta c; memset((void*)&c, 0, sizeof(c));
	c.n_warps = WM_CT_WARPS, c.sched = sched, c.sched_warp = sched_warp, c.rng = seed * 0x9e3779b97f4a7c15ull | 1;
	c.poll_bound = 1 << 22, c.on_atomic = on_atomic, c.user = &R;
	const int rc = wm_emul::run_cta(&c, body, &R);
	const int64_t st[10] = { R.lock_ok, R.lock_fail, c.polls, R.max_partial, R.publishes, c.syncs, c.switches, c.sweeps, c.events, c.deadlock };
	memcpy(stats, st, sizeof(st));
	if (rc != 0 && err && err_len > 0) {
		std::string s = "deadlock:";
		for (int k = 0; k < WM_CT_WARPS; ++k) {
			const int tk = R.task_of[k], T = R.tile_of[k];
			char b[96]; snprintf(b, sizeof(b), " w%d task %d tile %d anchor %d;", k, tk < n_tasks ? order[tk] : -1, T, 32 * T + k);
			s += b;
		}
		snprintf(err, (size_t)err_len, "%s", s.c_str());
	}
	delete R.S;
	return rc == 0 ? 0 : -1;
}

// Which paths of the tile kernel the scan of each anchor takes, at the kernel's WM_CT_RING and WM_CT_LIST, from the reference's loop
// (src/chain.c:58-88, restated like wmt_chain_fill_scalar).  The kernel resolves the list in steps of 32 entries (a list of WM_CT_LIST
// entries: steps [0, 32) and [32, WM_CT_LIST), then the refilled list likewise) and looks at every entry of a step before it knows where
// the loop breaks; so the candidates it examines are those up to the end of the step that holds the last one the loop consumes.  The
// scan needs the locked deep path when one of those lies below ring_lo = i0 + 64 - WM_CT_RING, or has its predecessor p[j] there.
// out: 5 ints per anchor: deep (bit 0: an examined candidate below ring_lo, bit 1: an examined candidate in the ring whose p[j] is
// below it), candidates in the window, candidates consumed up to and including the break (all when there is none), whether the loop
// ran to the window start (1) or broke (0), and ring_lo.
WMT_API int wmt_tile_scan_paths(const uint64_t *a_xy, int n, const int32_t *prm, float gap_scale, int32_t *out)
{
	if (n <= 0) return 0;
	const wm_chain_params P = make_params(prm, gap_scale);
	std::vector<int32_t> f((size_t)n), p((size_t)n), v((size_t)n), t((size_t)n, 0), cj;
	uint64_t sum_qspan = 0;
	for (int i = 0; i < n; ++i) sum_qspan += a_xy[2 * i + 1] >> 32 & 0xff;
	const float avg_qspan = (float)sum_qspan / n;
	int st = 0;
	for (int i = 0; i < n; ++i) {
		const uint64_t ri = a_xy[2 * i];
		const int32_t qi = (int32_t)a_xy[2 * i + 1], q_span = (int32_t)(a_xy[2 * i + 1] >> 32 & 0xff);
		int32_t max_f = q_span, max_j = -1, n_skip = 0;
		while (st < i && ri > a_xy[2 * st] + (uint64_t)(int64_t)P.max_dist_x) ++st;
		if (i - st > P.max_iter)
			while (i - st > P.max_iter && ri > a_xy[2 * st] + (uint64_t)(int64_t)P.min_dist_x) ++st;
		int n_used = 0, ended = 1;
		cj.clear();
		for (int j = i - 1; j >= st; --j) {
			const int64_t dr = (int64_t)(ri - a_xy[2 * j]);
			const int32_t dq = qi - (int32_t)a_xy[2 * j + 1];
			if (dr == 0 || dq <= 0) continue;
			if (dq > P.max_dist_y || dq > P.max_dist_x) continue;
			const int32_t dd = (int32_t)(dr > dq ? dr - dq : dq - dr);
			if (dd > P.bw) continue;
			cj.push_back(j);
			if (!ended) continue; // past the break: only the candidate total is still counted
			n_used = (int)cj.size();
			const int32_t min_d = dq < dr ? dq : (int32_t)dr;
			int32_t sc = min_d > q_span ? q_span : min_d;
			const int log_dd = dd ? 31 - __builtin_clz((unsigned)dd) : 0;
			const int gap_cost = (int)(dd * .01 * avg_qspan) + (log_dd >> 1);
			sc -= (int)((double)gap_cost * P.gap_scale + .499);
			sc += f[j];
			if (sc > max_f) { max_f = sc, max_j = j; if (n_skip > 0) --n_skip; }
			else if (t[j] == i) { if (++n_skip > P.max_skip) { ended = 0; continue; } }
			if (p[j] >= 0) t[p[j]] = i;
		}
		f[i] = max_f, p[i] = max_j;
		v[i] = max_j >= 0 && v[max_j] > max_f ? v[max_j] : max_f;
		const int ring_lo = (i & ~31) + 64 - WM_CT_RING;
		int deep = 0;
		if (n_used > 0) {
			const int c = n_used - 1, L = c / WM_CT_LIST, r = c % WM_CT_LIST;
			int end = L * WM_CT_LIST + (r < 32 ? 32 : WM_CT_LIST);
			if (end > (int)cj.size()) end = (int)cj.size();
			for (int e = 0; e < end; ++e) {
				const int j = cj[e];
				if (j < ring_lo) deep |= 1;
				else if (p[j] >= 0 && p[j] < ring_lo) deep |= 2;
			}
		}
		int32_t *o = out + 5 * (size_t)i;
		o[0] = deep, o[1] = (int)cj.size(), o[2] = n_used, o[3] = ended, o[4] = ring_lo;
	}
	return 0;
}

WMT_API int wmt_tile_constants(int32_t *out)
{
	out[0] = WM_CT_RING, out[1] = WM_CT_LIST, out[2] = WM_CT_WARPS;
	return 0;
}
