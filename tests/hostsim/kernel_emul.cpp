// TEST INFRASTRUCTURE.  The DP fill sweep (csrc/ksw_extd2_v2.cuh) and the traceback (csrc/ksw_extd2_common.cuh) of
// the product, compiled for the host on top of cuda_emul.h: one job at a time on a software warp of 32 threads.  The
// tests compare the result with the CPU oracle -- the kernels' arithmetic is checked without a GPU; the real kernels
// are checked on the device by the -m gpu tests.
#include <stdlib.h>
#include <vector>
#define WM_CT_RING 128 // small ring: the tile formulation goes through its locked deep path all the time
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/wm_common.cuh"
#include "../../winnowmap_b200/csrc/ksw_extd2_common.cuh"
#include "../../winnowmap_b200/csrc/ksw_extd2_v2.cuh"
#include "../../winnowmap_b200/csrc/ksw_extz2.cuh"
#include "../../winnowmap_b200/csrc/ksw_exts2.cuh"
#include "../../winnowmap_b200/csrc/chain_dev.cuh"
#include "../../winnowmap_b200/csrc/rsort.cuh"
#include "../../winnowmap_b200/csrc/pkseq.cuh"

namespace wm_emul {
thread_local Warp *warp = 0; thread_local int lane = 0;
static long long g_total_syncs = 0; // warp-wide synchronisation points executed so far (a proxy for dependent steps)
static void cta_warp_finished(Warp *w);
static void fiber_entry()
{
	Warp *w = warp;
	const int me = w->cur;
	lane = me;
	w->body(w->cta ? 32 * w->id + me : me, w->arg);
	w->done[me] = true;
	++w->n_done;
	// a finished lane never comes back: continue with another unfinished lane, or return to the caller
	for (int k = 1; k <= 32; ++k) {
		const int nxt = (me + k) & 31;
		if (!w->done[nxt]) { w->cur = nxt; setcontext(&w->ctx[nxt]); }
	}
	if (w->cta) cta_warp_finished(w); // (does not return)
	setcontext(&w->main_ctx);
}
void run_warp(void (*body)(int lane, void *arg), void *arg)
{
	Warp W;
	memset(W.done, 0, sizeof(W.done));
	W.cur = 0, W.arrived = 0, W.gen = 0, W.body = body, W.arg = arg, W.cta = 0, W.id = 0, W.n_done = 0;
	const size_t stack_bytes = (size_t)1 << 18;
	for (int l = 0; l < 32; ++l) {
		W.stack[l] = (char*)malloc(stack_bytes);
		getcontext(&W.ctx[l]);
		W.ctx[l].uc_stack.ss_sp = W.stack[l], W.ctx[l].uc_stack.ss_size = stack_bytes, W.ctx[l].uc_link = 0;
		makecontext(&W.ctx[l], (void (*)())fiber_entry, 0);
	}
	Warp *saved = warp;
	warp = &W;
	swapcontext(&W.main_ctx, &W.ctx[0]);
	warp = saved;
	g_total_syncs += W.gen;
	for (int l = 0; l < 32; ++l) free(W.stack[l]);
}

// ---- CTA runs (cuda_emul.h: run_cta) ----
static bool runnable(const Cta *c, const Warp *x) { return x->n_done < 32 && (x->blocked_at < 0 || x->blocked_at < c->events); }
// every unfinished lane of w waits at a sync or barrier, or has polled since w last resumed
static bool warp_blocked(const Warp *w)
{
	for (int l = 0; l < 32; ++l)
		if (!w->done[l] && (w->state[l] == LANE_RUN || (w->state[l] == LANE_POLL && w->polled_in[l] != w->run))) return false;
	return true;
}
static uint64_t next_rand(Cta *c) { c->rng ^= c->rng << 13; c->rng ^= c->rng >> 7; c->rng ^= c->rng << 17; return c->rng; }
// the warp to run after warp cur reached a switch point (-1: none is runnable)
static int pick(Cta *c, int cur)
{
	const int W = c->n_warps;
	auto next_after = [&](int skip) { // round robin from cur, skipping warp `skip`
		for (int d = 1; d <= W; ++d) { const int x = (cur + d) % W; if (x != skip && runnable(c, &c->w[x])) return x; }
		return -1;
	};
	if (c->sched == SCHED_RANDOM) {
		int cand[64], m = 0;
		for (int x = 0; x < W; ++x) if (runnable(c, &c->w[x])) cand[m++] = x;
		return m ? cand[next_rand(c) % m] : -1;
	}
	if (c->sched == SCHED_LAGGARD) { const int x = next_after(c->sched_warp); return x >= 0 ? x : runnable(c, &c->w[c->sched_warp]) ? c->sched_warp : -1; }
	if (c->sched == SCHED_LEADER && runnable(c, &c->w[c->sched_warp])) return c->sched_warp;
	return next_after(-1);
}
[[noreturn]] static void deadlock(Cta *c) { c->deadlock = 1; setcontext(&c->main_ctx); abort(); }
// when every warp is blocked, all are tried once more; if no sync or barrier completed since the last such round, none can go on
static int pick_or_retry(Cta *c, int cur)
{
	int x = pick(c, cur);
	if (x >= 0) return x;
	if (c->sweeps && c->syncs == c->syncs_at_sweep) deadlock(c);
	++c->sweeps, c->syncs_at_sweep = c->syncs;
	for (int k = 0; k < c->n_warps; ++k) c->w[k].blocked_at = -1;
	if ((x = pick(c, cur)) < 0) deadlock(c);
	return x;
}
static void enter(Warp *to) { ++to->run; to->blocked_at = -1; warp = to, lane = to->cur; }
// leave warp w (the current lane) for warp x; returns when w runs again
static void switch_to(Cta *c, Warp *w, int x)
{
	Warp *to = &c->w[x];
	const int me = lane;
	if (to == w) { ++w->run, w->blocked_at = -1; return; }
	++c->switches;
	enter(to);
	swapcontext(&w->ctx[me], &to->ctx[to->cur]);
	warp = w, lane = me;
}
static void release_barrier(Cta *c)
{
	c->bar_arrived = 0, ++c->bar_gen, ++c->syncs, ++c->events, c->polls_since_sync = 0;
	for (int k = 0; k < c->n_warps; ++k)
		for (int l = 0; l < 32; ++l) if (c->w[k].state[l] == LANE_BAR) c->w[k].state[l] = LANE_RUN;
}
void cta_sync_done(Warp *w)
{
	Cta *c = w->cta;
	++c->syncs, c->polls_since_sync = 0;
	for (int l = 0; l < 32; ++l) if (w->state[l] == LANE_SYNC) w->state[l] = LANE_RUN;
	switch_to(c, w, pick(c, w->id)); // (w itself is runnable)
}
void cta_poll()
{
	Warp *w = warp; Cta *c = w->cta;
	const int me = lane;
	++c->polls;
	if (++c->polls_since_sync > c->poll_bound) deadlock(c);
	w->state[me] = LANE_POLL, w->polled_in[me] = w->run;
	if (warp_blocked(w)) { w->blocked_at = c->events; switch_to(c, w, pick_or_retry(c, w->id)); }
	else yield_lane();
	w->state[me] = LANE_RUN;
}
void cta_barrier()
{
	Warp *w = warp; Cta *c = w->cta;
	const long long gen = c->bar_gen;
	if (++c->bar_arrived == c->live_threads) { release_barrier(c); switch_to(c, w, pick(c, w->id)); return; }
	w->state[lane] = LANE_BAR;
	while (c->bar_gen == gen) {
		if (warp_blocked(w)) { w->blocked_at = c->events; switch_to(c, w, pick_or_retry(c, w->id)); }
		else yield_lane();
	}
}
void cta_atomic(int kind, const void *addr, unsigned long long old, bool ok)
{
	Warp *w = warp; Cta *c = w->cta;
	// (a failed compare-and-swap changes nothing another warp could be waiting for)
	if (c->on_atomic ? c->on_atomic(c->user, kind, w->id, addr, old, ok) && ok : ok) ++c->events;
}
// the last lane of w has returned (on its own fiber, which is not resumed again)
static void cta_warp_finished(Warp *w)
{
	Cta *c = w->cta;
	++c->events, c->live_threads -= 32;
	if (c->bar_arrived > 0 && c->bar_arrived == c->live_threads) release_barrier(c);
	bool any = false;
	for (int k = 0; k < c->n_warps; ++k) any |= c->w[k].n_done < 32;
	if (!any) setcontext(&c->main_ctx);
	Warp *to = &c->w[pick_or_retry(c, w->id)];
	enter(to);
	setcontext(&to->ctx[to->cur]);
}
int run_cta(Cta *c, void (*body)(int tid, void *arg), void *arg)
{
	const int W = c->n_warps;
	if (W < 1 || W > 64) return -1;
	Warp *ws = new Warp[W];
	c->w = ws;
	c->events = c->syncs = c->polls = c->polls_since_sync = c->sweeps = c->syncs_at_sweep = c->switches = c->bar_gen = 0;
	c->bar_arrived = 0, c->live_threads = 32 * W, c->deadlock = 0;
	const size_t stack_bytes = (size_t)1 << 17;
	for (int k = 0; k < W; ++k) {
		Warp &X = ws[k];
		memset(X.done, 0, sizeof(X.done)); memset(X.state, 0, sizeof(X.state));
		X.cur = 0, X.arrived = 0, X.gen = 0, X.body = body, X.arg = arg, X.cta = c, X.id = k, X.n_done = 0, X.run = 0, X.blocked_at = -1;
		for (int l = 0; l < 32; ++l) {
			X.polled_in[l] = -1;
			X.stack[l] = (char*)malloc(stack_bytes);
			getcontext(&X.ctx[l]);
			X.ctx[l].uc_stack.ss_sp = X.stack[l], X.ctx[l].uc_stack.ss_size = stack_bytes, X.ctx[l].uc_link = 0;
			makecontext(&X.ctx[l], (void (*)())fiber_entry, 0);
		}
	}
	Warp *saved = warp; const int saved_lane = lane;
	Warp *first = &ws[pick(c, W - 1)];
	enter(first);
	swapcontext(&c->main_ctx, &first->ctx[0]);
	warp = saved, lane = saved_lane;
	for (int k = 0; k < W; ++k) { g_total_syncs += ws[k].gen; for (int l = 0; l < 32; ++l) free(ws[k].stack[l]); }
	delete[] ws;
	c->w = 0;
	return c->deadlock ? -1 : 0;
}
}
// defined by the CUDA library (ksw_extd2.cu); not used by the sweep itself
wm_prof_t g_wm_prof;
thread_local cudaStream_t wm_dbuf_stream = 0;
thread_local bool wm_dbuf_async = false;

// Same arithmetic as wm_dp_params_init / wm_extd2_bt_bytes of csrc/ksw_extd2.cu (host code of the CUDA library, not
// linkable here); src/ksw2_extd2_sse.c:61-97 and :84-86,114.
static void params_init(wm_dp_params *P, const int8_t *mat, int q, int e, int q2, int e2)
{
	P->qe_h = q + e;
	if (q2 + e2 < q + e) { int t = q; q = q2; q2 = t; t = e; e = e2; e2 = t; }
	P->q = q, P->e = e, P->q2 = q2, P->e2 = e2;
	P->sc_mch = mat[0], P->sc_mis = mat[1];
	P->sc_N = mat[24] == 0 ? -e2 : mat[24];
	int min_sc = mat[1];
	for (int t = 1; t < 25; ++t) min_sc = min_sc < mat[t] ? min_sc : mat[t];
	P->early_out = -min_sc > 2 * (q + e);
	int long_thres = e != e2 ? (q2 - q) / (e - e2) - 1 : 0;
	if (q2 + e2 + long_thres * e2 > q + e + long_thres * e) ++long_thres;
	P->long_thres = long_thres;
	P->long_diff = long_thres * (e - e2) - (q2 - q) - e2;
}

// one ksw_extd2 call through the product's sweep + traceback; global_state != 0 runs the instantiation that keeps
// the state rows in a global slice (the path of jobs that do not fit shared memory)
extern "C" int wmt_emul_extd2(const uint8_t *query, int qlen, const uint8_t *target, int tlen, const int8_t *mat, int q, int e, int q2, int e2,
                              int w, int zdrop, int end_bonus, int flag, int global_state, int32_t *ez_out, uint32_t *cigar, int cig_cap, int32_t *zd_out)
{
	wm_dp_params P; params_init(&P, mat, q, e, q2, e2);
	std::vector<uint8_t> seq((size_t)qlen + tlen + 64, 0);
	if (qlen > 0) memcpy(seq.data(), query, qlen);
	if (tlen > 0) memcpy(seq.data() + qlen, target, tlen);
	wm_dp_job J; memset(&J, 0, sizeof(J));
	J.q_off = 0, J.t_off = qlen, J.p_off = 0, J.cig_off = 0;
	J.qlen = qlen, J.tlen = tlen, J.w = w, J.zdrop = zdrop, J.end_bonus = end_bonus, J.flag = flag, J.cig_cap = cig_cap, J.pad = global_state ? 0 : -1;
	wm_extz_dev ez; memset(&ez, 0, sizeof(ez));
	const int tlen16 = (tlen + 15) / 16 * 16;
	if (!global_state && (tlen16 > WM_V2_T || qlen > WM_V2_Q)) return -1;
	if (qlen <= 0 || tlen <= 0 || P.early_out) { // what wm_extd2_fill_kernel's first-generation branch returns for these
		ez.max_q = ez.max_t = ez.mqe_t = ez.mte_q = -1;
		ez.max = 0, ez.score = ez.mqe = ez.mte = WM_NEG_INF;
	} else {
		int ww = w < 0 ? (tlen > qlen ? tlen : qlen) : w;
		const size_t bt_bytes = ((size_t)(qlen + tlen - 1) * (size_t)(wm_ncol16(qlen, tlen, ww) / 16) + 1) * 16;
		std::vector<uint8_t> bt(bt_bytes + 64, 0);
		const size_t slice = global_state ? wm_v2_slice_bytes(tlen16, qlen) : (size_t)WM_V2_SLICE + 64;
		std::vector<uint64_t> state(slice / 8 + 16, 0); // 8-byte aligned like the device slices
		struct Args { const wm_dp_job *J; const uint8_t *seq; uint8_t *bt; wm_extz_dev *ez; const wm_dp_params *P; uint8_t *state; int tlen16, qlen, global_state; }
			A = { &J, seq.data(), bt.data(), &ez, &P, (uint8_t*)state.data(), tlen16, qlen, global_state };
		wm_emul::run_warp([](int l, void *p) {
			Args &a = *(Args*)p;
			if (a.global_state) wm_extd2_fill_job_v2<false>(*a.J, a.seq, a.bt, a.ez, *a.P, a.state, a.tlen16, a.qlen, l, 0);
			else wm_extd2_fill_job_v2<true>(*a.J, a.seq, a.bt, a.ez, *a.P, a.state, 0, 0, l, 0);
		}, &A);
		wm_zd_params Z; memset(&Z, 0, sizeof(Z));
		Z.q = q, Z.e = e; memcpy(Z.mat, mat, 25);
		wm_extd2_backtrack_job(J, &ez, bt.data(), cigar, seq.data(), Z, zd_out);
	}
	memcpy(ez_out, &ez, sizeof(ez));
	return 0;
}

// one ksw_extz2 call (single gap pair) through the product's sweep (csrc/ksw_extz2.cuh) + the shared traceback
extern "C" int wmt_emul_extz2(const uint8_t *query, int qlen, const uint8_t *target, int tlen, const int8_t *mat, int q, int e,
                              int w, int zdrop, int end_bonus, int flag, int32_t *ez_out, uint32_t *cigar, int cig_cap, int32_t *zd_out)
{
	wm_dp_params P; params_init(&P, mat, q, e, q, e);
	P.single = 1;
	std::vector<uint8_t> seq((size_t)qlen + tlen + 64, 0);
	if (qlen > 0) memcpy(seq.data(), query, qlen);
	if (tlen > 0) memcpy(seq.data() + qlen, target, tlen);
	wm_dp_job J; memset(&J, 0, sizeof(J));
	J.q_off = 0, J.t_off = qlen, J.p_off = 0, J.cig_off = 0;
	J.qlen = qlen, J.tlen = tlen, J.w = w, J.zdrop = zdrop, J.end_bonus = end_bonus, J.flag = flag, J.cig_cap = cig_cap, J.pad = -1;
	wm_extz_dev ez; memset(&ez, 0, sizeof(ez));
	const int tlen16 = (tlen + 15) / 16 * 16;
	int ww = w < 0 ? (tlen > qlen ? tlen : qlen) : w;
	const size_t bt_bytes = (qlen > 0 && tlen > 0) ? ((size_t)(qlen + tlen - 1) * (size_t)(wm_ncol16(qlen, tlen, ww) / 16) + 1) * 16 : 16;
	std::vector<uint8_t> bt(bt_bytes + 64, 0);
	std::vector<uint64_t> state((size_t)tlen16 * 9 / 8 + 16, 0);
	struct Args { const wm_dp_job *J; const uint8_t *seq; uint8_t *bt; wm_extz_dev *ez; const wm_dp_params *P; int8_t *state; }
		A = { &J, seq.data(), bt.data(), &ez, &P, (int8_t*)state.data() };
	wm_emul::run_warp([](int l, void *p) { Args &a = *(Args*)p; wm_extz2_fill_job(*a.J, a.seq, a.bt, a.ez, *a.P, a.state, l, 0); }, &A);
	wm_zd_params Z; memset(&Z, 0, sizeof(Z));
	Z.q = q, Z.e = e; memcpy(Z.mat, mat, 25);
	wm_extd2_backtrack_job(J, &ez, bt.data(), cigar, seq.data(), Z, zd_out);
	memcpy(ez_out, &ez, sizeof(ez));
	return 0;
}

// one ksw_exts2 call (splice-aware extension) through the product's sweep (csrc/ksw_exts2.cuh) + the shared traceback
extern "C" int wmt_emul_exts2(const uint8_t *query, int qlen, const uint8_t *target, int tlen, const uint8_t *junc, const int8_t *mat, int q, int e, int q2,
                              int noncan, int junc_bonus, int zdrop, int flag, int32_t *ez_out, uint32_t *cigar, int cig_cap)
{
	wm_dp_params P; memset(&P, 0, sizeof(P)); // (wm_dp_params_init_splice of ksw_extd2.cu restated: src/ksw2_exts2_sse.c:61-84)
	P.splice = 1, P.noncan = noncan, P.junc_bonus = junc_bonus; memcpy(P.mat, mat, 25);
	P.q = q, P.e = e, P.q2 = q2, P.qe_h = q + e, P.sc_mch = mat[0], P.sc_mis = mat[1], P.sc_N = mat[24] == 0 ? -e : mat[24];
	int min_sc = mat[1];
	for (int t = 1; t < 25; ++t) min_sc = min_sc < mat[t] ? min_sc : mat[t];
	P.early_out = q2 <= q + e || -min_sc > 2 * (q + e) || e <= 0;
	if (!P.early_out) {
		P.long_thres = (q2 - q) / e - 1;
		if (q2 > q + e + P.long_thres * e) ++P.long_thres;
		P.long_diff = P.long_thres * e - (q2 - q);
	}
	std::vector<uint8_t> seq((size_t)qlen + tlen + 64, 0);
	if (qlen > 0) memcpy(seq.data(), query, qlen);
	if (tlen > 0) memcpy(seq.data() + qlen, target, tlen);
	wm_dp_job J; memset(&J, 0, sizeof(J));
	J.q_off = 0, J.t_off = qlen, J.p_off = 0, J.cig_off = 0;
	J.qlen = qlen, J.tlen = tlen, J.w = -1, J.zdrop = zdrop, J.end_bonus = -1, J.flag = flag, J.cig_cap = cig_cap, J.pad = -1;
	wm_extz_dev ez; memset(&ez, 0, sizeof(ez));
	const int tlen16 = (tlen + 15) / 16 * 16;
	const int ww = tlen > qlen ? tlen : qlen;
	const size_t bt_bytes = (qlen > 0 && tlen > 0) ? ((size_t)(qlen + tlen - 1) * (size_t)(wm_ncol16(qlen, tlen, ww) / 16) + 1) * 16 : 16;
	std::vector<uint8_t> bt(bt_bytes + 64, 0);
	std::vector<uint64_t> state((size_t)tlen16 * WM_EXTS2_CELL_BYTES / 8 + 16, 0);
	struct Args { const wm_dp_job *J; const uint8_t *seq, *junc; uint8_t *bt; wm_extz_dev *ez; const wm_dp_params *P; int8_t *state; }
		A = { &J, seq.data(), junc, bt.data(), &ez, &P, (int8_t*)state.data() };
	wm_emul::run_warp([](int l, void *p) { Args &a = *(Args*)p; wm_exts2_fill_job(*a.J, a.seq, a.junc, a.bt, a.ez, *a.P, a.state, l, 0); }, &A);
	wm_zd_params Z; memset(&Z, 0, sizeof(Z));
	wm_extd2_backtrack_job(J, &ez, bt.data(), cigar, seq.data(), Z, 0, 1, P.long_thres, P.early_out);
	memcpy(ez_out, &ez, sizeof(ez));
	return 0;
}

// the shared-memory-ring formulation (wm_chain_fill_warp_ring): window starts first (closed form), then the sweep.  The
// small ring (64 slots) forces the scans through the older-than-the-ring path that reads global memory.
template <int RING>
static void run_ring(const wm128_dev *a, int n, const wm_chain_params *P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int lane)
{
	static thread_local wm_chain_ring<RING> *ring = 0;
	if (lane == 0) { if (!ring) ring = new wm_chain_ring<RING>(); memset(ring, 0xff, sizeof(*ring)); }
	for (int i = lane; i < n; i += 32) v[i] = wm_chain_window_start(a, i, *P);
	__syncwarp();
	wm_chain_fill_warp_ring<RING>(a, n, *P, f, p, t, v, ring, lane);
}
// the tile formulation (wm_chain_tile_scan): what one CTA of csrc/chain.cu does, with the 32 anchors of a tile taken in
// order by one software warp (the order satisfies every dependency; the concurrency is exercised by tile_cta_emul.cpp and on the GPU)
static void run_tile(const wm128_dev *a, int n, const wm_chain_params *P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int lane)
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
			if (!wm_chain_tile_scan(a, *P, f, p, t, S, S->marks[k], al, prev, i0, k, st, ring_lo, false, avg_d, scale_d, lane, &max_f, &max_j))
				wm_chain_tile_scan(a, *P, f, p, t, S, S->marks[k], al, prev, i0, k, st, ring_lo, true, avg_d, scale_d, lane, &max_f, &max_j);
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
static void run_fill(int mode, const wm128_dev *a, int n, const wm_chain_params *P, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int32_t *D, int lane)
{
	if (mode == 1) wm_chain_fill_warp_dense(a, n, *P, f, p, t, v, D, lane);
	else if (mode == 2) run_ring<64>(a, n, P, f, p, t, v, lane);
	else if (mode == 3) run_ring<1024>(a, n, P, f, p, t, v, lane);
	else if (mode == 4) run_tile(a, n, P, f, p, t, v, lane);
	else wm_chain_fill_warp(a, n, *P, f, p, t, v, lane);
}

// The chaining forward pass (csrc/chain_dev.cuh) on the software warp: dense = 0 the production formulation (32
// predecessors per step), dense = 1 the dense-candidate formulation, 2 / 3 the shared-memory ring (64 / 1024 slots), 4 the tile formulation (ring of 128 slots here).  Outputs the f / p / v arrays the backtracking
// kernel consumes (a is `n` anchors, x then y).
extern "C" int wmt_emul_chain_fill(const uint64_t *a_xy, int n, int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                                   float gap_scale, int dense, int32_t *f, int32_t *p, int32_t *v)
{
	std::vector<wm128_dev> a((size_t)n + 1);
	for (int i = 0; i < n; ++i) a[i].x = a_xy[2 * i], a[i].y = a_xy[2 * i + 1];
	wm_chain_params P; memset(&P, 0, sizeof(P));
	P.max_dist_x = max_dist_x, P.min_dist_x = min_dist_x, P.max_dist_y = max_dist_y, P.bw = bw, P.max_skip = max_skip, P.max_iter = max_iter;
	P.gap_scale = gap_scale;
	std::vector<int32_t> t((size_t)n + 1, 0), D(WM_CHAIN_DENSE_CAP, 0);
	struct Args { const wm128_dev *a; int n; const wm_chain_params *P; int32_t *f, *p, *t, *v, *D; int dense; } A = { a.data(), n, &P, f, p, t.data(), v, D.data(), dense };
	if (n <= 0) return 0;
	wm_emul::run_warp([](int l, void *q) {
		Args &x = *(Args*)q;
		run_fill(x.dense, x.a, x.n, x.P, x.f, x.p, x.t, x.v, x.D, l);
	}, &A);
	return 0;
}

// Scalar restatement of the forward pass of mm_chain_dp (src/chain.c:41-90, n_segs == 1, is_cdna == 0): the yardstick
// for the two warp formulations above.
extern "C" int wmt_chain_fill_scalar(const uint64_t *a_xy, int n, int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                                     float gap_scale, int32_t *f, int32_t *p, int32_t *v)
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
			int log_dd = 0;
			if (dd) { log_dd = 31 - __builtin_clz((unsigned)dd); }
			const int gap_cost = (int)(dd * .01 * avg_qspan) + (log_dd >> 1);
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

extern "C" long long wmt_emul_sync_count(void) { return wm_emul::g_total_syncs; }

// The warp-cooperative tie-exact radix sort of the anchor arrays (csrc/rsort.cuh) on the software warp; a = n (x, y) pairs.
extern "C" int wmt_emul_sort128(uint64_t *a_xy, int n)
{
	std::vector<wm128_dev> a((size_t)n + 1);
	for (int i = 0; i < n; ++i) a[i].x = a_xy[2 * i], a[i].y = a_xy[2 * i + 1];
	wm_rs_warp_ws W; memset(&W, 0, sizeof(W));
	std::vector<wm_rs_range> wl((size_t)n / 64 + 4);
	struct Args { wm128_dev *a; int n; wm_rs_warp_ws *W; wm_rs_range *wl; } A = { a.data(), n, &W, wl.data() };
	wm_emul::run_warp([](int l, void *q) { Args &x = *(Args*)q; wm_radix_sort_warp(x.a, x.n, x.W, x.wl, l); }, &A);
	for (int i = 0; i < n; ++i) a_xy[2 * i] = a[i].x, a_xy[2 * i + 1] = a[i].y;
	return 0;
}

// mm_chain_dp end to end on the software warp: forward pass (either formulation) + backtracking (csrc/chain_dev.cuh).
// a_xy is overwritten with the chained anchors (n_b of them), u receives the (score << 32 | count) words (n_u).
extern "C" int wmt_emul_chain(uint64_t *a_xy, int n, int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                              int min_cnt, int min_sc, float gap_scale, int dense, uint64_t *u_out, int32_t *n_u_out, int64_t *n_b_out)
{
	*n_u_out = 0, *n_b_out = 0;
	if (n <= 0) return 0;
	std::vector<wm128_dev> a((size_t)n + 1), w((size_t)n + 1), b((size_t)n + 1);
	for (int i = 0; i < n; ++i) a[i].x = a_xy[2 * i], a[i].y = a_xy[2 * i + 1];
	wm_chain_params P; memset(&P, 0, sizeof(P));
	P.max_dist_x = max_dist_x, P.min_dist_x = min_dist_x, P.max_dist_y = max_dist_y, P.bw = bw, P.max_skip = max_skip, P.max_iter = max_iter;
	P.min_cnt = min_cnt, P.min_sc = min_sc, P.gap_scale = gap_scale;
	std::vector<int32_t> f((size_t)n + 1), p((size_t)n + 1), t((size_t)n + 1, 0), v((size_t)n + 1), D(WM_CHAIN_DENSE_CAP, 0);
	std::vector<uint64_t> u(2 * (size_t)n + 2), u2((size_t)n + 1);
	wm_rs_warp_ws stack; memset(&stack, 0, sizeof(stack));
	struct Args { wm128_dev *a, *w, *b; int n; const wm_chain_params *P; int32_t *f, *p, *t, *v, *D; uint64_t *u, *u2; wm_rs_warp_ws *stk; int dense; int32_t *n_u; int64_t *n_b; }
		A = { a.data(), w.data(), b.data(), n, &P, f.data(), p.data(), t.data(), v.data(), D.data(), u.data(), u2.data(), &stack, dense, n_u_out, n_b_out };
	wm_emul::run_warp([](int l, void *q) {
		Args &x = *(Args*)q;
		run_fill(x.dense, x.a, x.n, x.P, x.f, x.p, x.t, x.v, x.D, l);
		__syncwarp();
		wm_chain_backtrack_grp<false>(x.a, x.n, *x.P, x.f, x.p, x.t, x.v, x.u, x.u2, x.w, x.b, x.stk, x.n_u, x.n_b, l, 32, 0);
	}, &A);
	for (int i = 0; i < *n_u_out; ++i) u_out[i] = u2[i];
	for (int64_t i = 0; i < *n_b_out; ++i) a_xy[2 * i] = a[i].x, a_xy[2 * i + 1] = a[i].y;
	return 0;
}


// ---- the packed read pool (csrc/pkseq.cuh): packing, k-mer windows, masked copies and the DP gather against a plain
// byte-per-base restatement.  Returns 0, or the line of the first mismatch. ----
static uint64_t pk_rng(uint64_t *s) { *s = *s * 6364136223846793005ULL + 1442695040888963407ULL; return *s >> 33; }
extern "C" int wmt_pk_selftest(uint64_t seed, int64_t n, int k)
{
	uint8_t lut[256];
	for (int c = 0; c < 256; ++c) { // seq_nt4_table (src/sketch.c:19-36)
		uint8_t v = c < 4 ? (uint8_t)c : 4;
		if (c == 'A' || c == 'a') v = 0; else if (c == 'C' || c == 'c') v = 1; else if (c == 'G' || c == 'g') v = 2;
		else if (c == 'T' || c == 't' || c == 'U' || c == 'u') v = 3;
		lut[c] = v;
	}
	static const char alphabet[] = "ACGTacgtNnUuRY\x01\x03-";
	std::vector<unsigned char> ascii(n + 64, 'N');
	for (int64_t i = 0; i < n; ++i) {
		const uint64_t r = pk_rng(&seed);
		ascii[i] = (r & 63) < 60 ? "ACGT"[r >> 8 & 3] : (unsigned char)alphabet[(r >> 8) % (sizeof(alphabet) - 1)];
	}
	std::vector<uint8_t> code(n + 64, 4);
	for (int64_t i = 0; i < n; ++i) code[i] = lut[ascii[i]];
	const int64_t ng = (n + 31) / 32;
	std::vector<uint32_t> pk(2 * ng + WM_PK_SLACK + 4, 0), nm(ng + WM_PK_SLACK + 4, 0xffffffffu);
	for (int64_t g = 0; g < ng; ++g) {
		uint32_t raw[8];
		for (int j = 0; j < 8; ++j) { uint32_t v = 0; for (int b = 0; b < 4; ++b) v |= (uint32_t)ascii[g * 32 + 4 * j + b] << 8 * b; raw[j] = v; }
		uint64_t p; uint32_t m;
		wm_pk_pack32(raw, lut, &p, &m);
		pk[2 * g] = (uint32_t)p, pk[2 * g + 1] = (uint32_t)(p >> 32), nm[g] = m;
	}
	wm_pkseq S; S.pk = pk.data(), S.nm = nm.data();
	for (int64_t i = 0; i < n; ++i) if (wm_pk_get(S, i) != code[i]) return __LINE__;
	const uint32_t kmask = (1u << k) - 1u;
	for (int64_t b = 0; b + k <= n; ++b) { // every k-mer: src/sketch.c:162-163 base by base
		uint64_t f = 0, r = 0; bool amb = false;
		for (int j = 0; j < k; ++j) {
			const uint64_t c = code[b + j];
			amb |= c > 3;
			f = f << 2 | (c & 3);
			r = r >> 2 | (3ULL ^ (c & 3)) << (2 * (k - 1));
		}
		if (((wm_pk_nwindow(S.nm, b) & kmask) != 0) != amb) return __LINE__;
		uint64_t f2, r2;
		wm_pk_kmer(wm_pk_window(S.pk, b), k, &f2, &r2);
		if (!amb && (f2 != f || r2 != r)) return __LINE__;
	}
	// masked copies of random windows
	for (int it = 0; it < 200; ++it) {
		wm_mask_task T;
		T.len = 1 + (int)(pk_rng(&seed) % 3000); if (T.len > n) T.len = (int)n;
		T.src_off = (int64_t)(pk_rng(&seed) % (uint64_t)(n - T.len + 1)); T.dst_off = 0, T.mask_off = 3;
		std::vector<int32_t> pool(6, 0);
		int pos = (int)(pk_rng(&seed) % 40); T.n_mask = 0;
		while (pos < T.len + 50 && T.n_mask < 64) {
			const int e = pos + 1 + (int)(pk_rng(&seed) % 200);
			pool.push_back(pos), pool.push_back(e); ++T.n_mask;
			pos = e + (int)(pk_rng(&seed) % 300);
		}
		for (int p0 = 0; p0 < T.len; p0 += 32) {
			uint64_t v; uint32_t m;
			wm_pk_mask32(S, T, p0, pool.data(), &v, &m);
			for (int j = 0; j < 32; ++j) {
				const int p = p0 + j;
				int c = 4;
				if (p < T.len) {
					c = code[T.src_off + p];
					for (int a = 0; a < T.n_mask; ++a) if (p >= pool[6 + 2 * a] && p < pool[6 + 2 * a + 1]) c = 4;
				}
				const int got = (m >> j & 1) ? 4 : (int)(v >> 2 * j & 3);
				if (got != c) return __LINE__;
			}
		}
	}
	// DP gather: slices of "reads" (both strands, both directions) and of a 4-bit packed reference
	std::vector<uint32_t> S4((n + 7) / 8 + 4, 0);
	for (int64_t i = 0; i < n; ++i) S4[i >> 3] |= (uint32_t)code[i] << ((i & 7) << 2);
	for (int it = 0; it < 4000; ++it) {
		const int64_t L = 1 + (int64_t)(pk_rng(&seed) % (uint64_t)(n < 5000 ? n : 5000)), r0 = (int64_t)(pk_rng(&seed) % (uint64_t)(n - L + 1));
		wm_gather_job J;
		J.len = 1 + (int)(pk_rng(&seed) % (uint64_t)L); if (it % 7 == 0 && J.len > 17) J.len = 1 + (int)(pk_rng(&seed) % 17);
		const int64_t o = (int64_t)(pk_rng(&seed) % (uint64_t)(L - J.len + 1)); // offset of the slice on its strand
		J.kind = (int)(pk_rng(&seed) % 3), J.reversed = (int)(pk_rng(&seed) & 1), J.pad = 0, J.dst_off = 0;
		J.src_off = J.kind == 2 ? r0 + (L - 1 - o) : r0 + o;
		for (int p0 = 0; p0 < J.len + 16; p0 += 16) {
			uint32_t out[4];
			wm_pk_gather16(J, p0, S, S4.data(), out);
			for (int j = 0; j < 16; ++j) {
				const int p = p0 + j;
				int want = 0;
				if (p < J.len) {
					const int64_t q = o + (J.reversed ? J.len - 1 - p : p); // position on the slice's strand
					if (J.kind == 2) { const int c = code[r0 + (L - 1 - q)]; want = c < 4 ? 3 - c : 4; } // src/align.c:874-876
					else want = code[r0 + q];
				}
				if ((int)(out[j >> 2] >> 8 * (j & 3) & 255) != want) return __LINE__;
			}
		}
	}
	return 0;
}
