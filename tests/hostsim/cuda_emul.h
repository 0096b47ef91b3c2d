// TEST INFRASTRUCTURE.  Host emulation of the CUDA device features the DP sweeps use, so that the kernels' arithmetic
// (csrc/ksw_extd2_v2.cuh, csrc/ksw_extd2_common.cuh) can be compiled with g++ and checked against the oracle without a
// GPU: a warp is 32 lockstep fibers of one host thread, shuffles and __syncwarp are barriers around a shared exchange buffer,
// the 16x2 SIMD intrinsics and prmt/funnel-shift are restated from the PTX ISA.
#pragma once
#include <ucontext.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <cuda_runtime.h> // types only (uint2, cudaStream_t); __device__ / __forceinline__ expand to host-neutral forms

#define WM_HOST_EMUL 1

namespace wm_emul {
struct Cta;
// The 32 lanes are fibers (ucontext) of one host thread, scheduled round-robin; a barrier is "yield until everybody
// has arrived", so a warp-level operation costs a few context switches instead of an OS barrier.
struct Warp {
	ucontext_t main_ctx, ctx[32];
	char *stack[32];
	bool done[32];
	int cur, arrived, gen;
	uint64_t xchg[32];
	void (*body)(int lane, void *arg); void *arg; // (in a CTA, body receives the thread index 32 * id + lane)
	// the rest is used by CTA runs only (run_cta): the CTA (0 for a lone warp of run_warp), the warp's index there, what each lane
	// waits for (LANE_*), the warp's run count and, per polling lane, the run in which it polled, and the CTA event count at which
	// the warp was found blocked (-1: runnable)
	Cta *cta; int id, n_done;
	int8_t state[32]; long long run, polled_in[32], blocked_at;
};
enum { LANE_RUN = 0, LANE_SYNC = 1, LANE_POLL = 2, LANE_BAR = 3 };
extern thread_local Warp *warp;
extern thread_local int lane;
inline void yield_lane()
{ // hand over to the next unfinished lane; returns when this lane is scheduled again
	Warp *w = warp;
	const int me = w->cur;
	int nxt = me;
	do { nxt = (nxt + 1) & 31; } while (w->done[nxt] && nxt != me);
	if (nxt == me) return;
	w->cur = nxt;
	swapcontext(&w->ctx[me], &w->ctx[nxt]);
	warp = w, lane = me; // (thread_local shared by all fibers; in a CTA another warp may have run meanwhile)
}
void cta_sync_done(Warp *w); // kernel_emul.cpp: a warp-wide sync of w completed: the CTA's scheduler may run another warp
inline void sync()
{
	Warp *w = warp;
	const int gen = w->gen;
	if (++w->arrived == 32) {
		w->arrived = 0; ++w->gen;
		if (w->cta) cta_sync_done(w);
		return;
	}
	if (w->cta) w->state[lane] = LANE_SYNC;
	while (w->gen == gen) yield_lane();
}
template <typename T> inline T exchange(T v, int src_lane)
{
	uint64_t u = 0; memcpy(&u, &v, sizeof(T));
	warp->xchg[lane] = u;
	sync();
	const uint64_t r = warp->xchg[src_lane & 31];
	sync();
	T out; memcpy(&out, &r, sizeof(T));
	return out;
}
void run_warp(void (*body)(int lane, void *arg), void *arg); // kernel_emul.cpp: runs body on 32 lockstep lanes

// ---- a CTA of several software warps (kernel_emul.cpp: run_cta) ----
// Lanes of a warp stay lockstep fibers.  Warps are switched only where a warp can stall on the hardware: when one of its warp-wide
// syncs completes (ballot, shuffle, __syncwarp), at __syncthreads and at __nanosleep.  A warp is blocked when every unfinished lane
// polls (__nanosleep) or waits at a sync or barrier; it becomes runnable again after an atomic operation, a barrier release or the
// end of a warp (what lets a polling warp of the kernels go on), or when every warp is blocked: then all are tried once more, and
// if no sync or barrier completes before they block again, the run stops with a deadlock.
enum { SCHED_ROUND_ROBIN = 0, SCHED_RANDOM = 1, SCHED_LAGGARD = 2, SCHED_LEADER = 3 };
enum { ATOM_ADD = 0, ATOM_OR = 1, ATOM_CAS = 2, ATOM_EXCH = 3 };
struct Cta {
	int n_warps; Warp *w;
	// SCHED_ROUND_ROBIN: the next runnable warp after every completed sync; SCHED_RANDOM: a runnable warp drawn with rng;
	// SCHED_LAGGARD: warp sched_warp runs only when every other warp is blocked; SCHED_LEADER: warp sched_warp runs whenever it can
	int sched, sched_warp; uint64_t rng;
	long long poll_bound;  // polls without a completed sync or barrier after which the run counts as deadlocked
	// observer of the atomic operations (kind ATOM_*, the warp, the address, the old value, whether a CAS succeeded), may be 0; it
	// returns whether a polling warp could be waiting for that operation (without an observer, every one that changes memory counts)
	bool (*on_atomic)(void *user, int kind, int warp, const void *addr, unsigned long long old, bool ok); void *user;
	// statistics and state
	long long events, syncs, polls, polls_since_sync, sweeps, syncs_at_sweep, switches, bar_gen;
	int bar_arrived, live_threads, deadlock;
	ucontext_t main_ctx;
};
void cta_poll();    // __nanosleep of a lane in a CTA
void cta_barrier(); // __syncthreads
void cta_atomic(int kind, const void *addr, unsigned long long old, bool ok);
// Runs body(tid, arg) on c->n_warps warps of 32 lanes; the caller sets the schedule fields, poll_bound and on_atomic of c.  Returns 0,
// or -1 after a deadlock (c->deadlock = 1; the lanes are abandoned where they stood).
int run_cta(Cta *c, void (*body)(int tid, void *arg), void *arg);
inline void note_atomic(int kind, const void *addr, unsigned long long old, bool ok) { if (warp && warp->cta) cta_atomic(kind, addr, old, ok); }
} // namespace wm_emul

inline void __syncwarp(unsigned = 0xffffffffu) { wm_emul::sync(); }
template <typename T> inline T __shfl_sync(unsigned, T v, int src, int = 32) { return wm_emul::exchange(v, src); }
template <typename T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32)
{ const int src = wm_emul::lane - (int)d; const T r = wm_emul::exchange(v, src < 0 ? wm_emul::lane : src); return src < 0 ? v : r; }
template <typename T> inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return wm_emul::exchange(v, wm_emul::lane ^ m); }
inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v)
{ const unsigned long long o = __atomic_fetch_add(p, v, __ATOMIC_RELAXED); wm_emul::note_atomic(wm_emul::ATOM_ADD, p, o, true); return o; }
inline int atomicAdd(int *p, int v) { const int o = __atomic_fetch_add(p, v, __ATOMIC_RELAXED); wm_emul::note_atomic(wm_emul::ATOM_ADD, p, (unsigned)o, true); return o; }
inline int atomicMin(int *p, int v) { int o = *p; if (v < o) *p = v; return o; }
inline unsigned atomicOr(unsigned *p, unsigned v) { const unsigned o = __atomic_fetch_or(p, v, __ATOMIC_RELAXED); wm_emul::note_atomic(wm_emul::ATOM_OR, p, o, true); return o; }
inline int atomicCAS(int *p, int cmp, int v) { const int o = *p; if (o == cmp) *p = v; wm_emul::note_atomic(wm_emul::ATOM_CAS, p, (unsigned)o, o == cmp); return o; }
inline int atomicExch(int *p, int v) { const int o = *p; *p = v; wm_emul::note_atomic(wm_emul::ATOM_EXCH, p, (unsigned)o, true); return o; }
// a lone warp (run_warp) has nobody to wait for: its polls only let the other lanes go on
inline void __nanosleep(unsigned) { if (wm_emul::warp->cta) wm_emul::cta_poll(); else wm_emul::yield_lane(); }
inline void __syncthreads() { if (wm_emul::warp->cta) wm_emul::cta_barrier(); else wm_emul::sync(); }
// the emulation is sequentially consistent: fences and cache hints have nothing to do
inline void __threadfence_block() {}
template <typename T> inline T __ldcg(const T *p) { return *p; }

// ---- integer SIMD-in-a-word intrinsics (CUDA math API semantics) ----
inline uint32_t wm_emul_pack(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }
inline int wm_emul_lo(uint32_t a) { return (int16_t)(a & 0xffffu); }
inline int wm_emul_hi(uint32_t a) { return (int16_t)(a >> 16); }
inline unsigned __vadd2(unsigned a, unsigned b) { return wm_emul_pack(wm_emul_lo(a) + wm_emul_lo(b), wm_emul_hi(a) + wm_emul_hi(b)); }
inline unsigned __vsub2(unsigned a, unsigned b) { return wm_emul_pack(wm_emul_lo(a) - wm_emul_lo(b), wm_emul_hi(a) - wm_emul_hi(b)); }
inline unsigned __vmins2(unsigned a, unsigned b)
{ return wm_emul_pack(wm_emul_lo(a) < wm_emul_lo(b) ? wm_emul_lo(a) : wm_emul_lo(b), wm_emul_hi(a) < wm_emul_hi(b) ? wm_emul_hi(a) : wm_emul_hi(b)); }
inline unsigned __vmaxs2(unsigned a, unsigned b)
{ return wm_emul_pack(wm_emul_lo(a) > wm_emul_lo(b) ? wm_emul_lo(a) : wm_emul_lo(b), wm_emul_hi(a) > wm_emul_hi(b) ? wm_emul_hi(a) : wm_emul_hi(b)); }
// max(a + b, c) per signed 16-bit half; the sum wraps to 16 bits first
inline unsigned __viaddmax_s16x2(unsigned a, unsigned b, unsigned c) { return __vmaxs2(__vadd2(a, b), c); }
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift)
{ const uint64_t v = (uint64_t)hi << 32 | lo; return (uint32_t)(v >> (shift & 31)); }
inline unsigned long long __brevll(unsigned long long x)
{ unsigned long long r = 0; for (int i = 0; i < 64; ++i) r |= (x >> i & 1ULL) << (63 - i); return r; }
// prmt.b32, default mode: byte i of the result is byte (sel nibble i & 7) of {b,a}; nibble bit 3 replicates that byte's sign
inline uint32_t wm_emul_prmt(uint32_t a, uint32_t b, uint32_t sel)
{
	const uint64_t v = (uint64_t)b << 32 | a;
	uint32_t r = 0;
	for (int i = 0; i < 4; ++i) {
		const unsigned n = sel >> (4 * i) & 0xf;
		uint32_t byte = (uint32_t)(v >> (8 * (n & 7))) & 0xffu;
		if (n & 8) byte = (byte & 0x80u) ? 0xffu : 0u;
		r |= byte << (8 * i);
	}
	return r;
}
inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel) { return wm_emul_prmt(a, b, sel & 0x7777u); }

// ---- warp votes, bit utilities and the rounding-mode intrinsics of the chaining kernels ----
inline unsigned __ballot_sync(unsigned, bool pred)
{ // two rounds: everybody publishes, everybody collects
	wm_emul::warp->xchg[wm_emul::lane] = pred ? 1 : 0;
	wm_emul::sync();
	unsigned m = 0;
	for (int l = 0; l < 32; ++l) m |= (unsigned)(wm_emul::warp->xchg[l] & 1) << l;
	wm_emul::sync();
	return m;
}
inline bool __any_sync(unsigned mask, bool pred) { return __ballot_sync(mask, pred) != 0; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __clz(int x) { return x == 0 ? 32 : __builtin_clz((unsigned)x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
// compiled with -ffp-contract=off: plain C operations round to nearest even, once, like the _rn intrinsics
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __ull2float_rn(unsigned long long x) { return (float)x; }
inline float __ll2float_rn(long long x) { return (float)x; }
using std::max;
using std::min;
