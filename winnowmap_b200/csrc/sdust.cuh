// SDUST low-complexity regions (the mapper's -T, reference src/sdust.c:134-164 with W = 64, run by src/map.c:43-67 on every
// sequence collect_minimizers sketches) and the test that squeezes minimizers out of them.  The device code here is also
// compiled for the host by the emulation tests (tests/hostsim/sdust_emul.cpp), so it uses no CUDA runtime call.
//
// One thread runs one sequence.  SDUST is a scan with a state that never resets: a base outside ACGT flushes the pending
// intervals, but the triplet window, its counts and its scores carry on into the next piece, so neither pieces nor windows
// can be scanned independently and give the same regions.  What a thread holds:
//   win, cw, cv  the last W - 2 triplets (a ring), their counts in the window and in its valid suffix (local memory)
//   P            the perfect intervals still inside the window, sorted by descending start, then ascending finish.  In the
//                first W bases of a piece after a non-ACGT base the window start stays put while the window is full of the
//                last piece's triplets, so every base may add up to W - 2 intervals with the same finish, none leaving: P
//                reaches (W - 2)^2 + (W - 2) = 3906 entries at W = 64 (2067 are reached by T = 1 on a CA repeat cut by an N).
//                Such lists are rare (a mapping at T = 20 rarely holds more than a few dozen), so a first pass gives each
//                thread WM_SDUST_PCAP_FAST entries and hands a sequence whose list would outgrow them to a second pass of
//                few threads with WM_SDUST_PCAP entries each (global slices of 8-byte entries)
//   res          the regions, merged when one touches or overlaps the last: sorted and disjoint, each at least 3 bases long
//                and starting after the last one's end, so a sequence of n bases has at most (n + W) / 4 + 1 of them
#pragma once
#include <stdint.h>

#define WM_SDUST_WMAX 64                                   // largest window (the mapper's)
#define WM_SDUST_PCAP (WM_SDUST_WMAX * WM_SDUST_WMAX)      // perfect intervals per thread (>= (WMAX - 2)^2 + WMAX - 2)
#define WM_SDUST_PCAP_FAST 256                             // the same in the first pass
#define WM_SDUST_MAX_T (1 << 20)                           // largest threshold: keeps T * 2 and T * 62 inside an int

// a perfect interval [start, start + l + 3): l + 1 triplets, score r (r <= C(W - 2, 2), l < W)
struct wm_sdust_perf { int32_t start; int16_t r, l; };

// regions bound of a sequence of n bases (see above)
static inline int64_t wm_sdust_reg_cap(int64_t n, int W) { return (n + W) / 4 + 1; }

// The regions of the sequence base(0) .. base(len - 1) (codes 0..3, 4 = outside ACGT) as start << 32 | end in res[0, return
// value), or -1 when P would outgrow pcap entries (the regions are then incomplete).  *err is set when res would overflow
// res_cap (never at the bound above).
template <class Base>
__device__ __forceinline__ int64_t wm_sdust_seq(const Base &base, int len, int T, int W, wm_sdust_perf *P, int pcap, uint64_t *res,
                                                int64_t res_cap, int *err)
{
	int win[WM_SDUST_WMAX], cw[64], cv[64];
	for (int j = 0; j < 64; ++j) cw[j] = cv[j] = 0;
	const int cap = W - 2;
	int head = 0, n = 0, L = 0, rw = 0, rv = 0, nP = 0;
	int64_t n_res = 0;
	// the leftmost interval of P goes out once it starts before the window, then every interval that does is dropped
	auto flush = [&](int wstart) {
		if (nP == 0 || P[nP - 1].start >= wstart) return;
		const int ps = P[nP - 1].start, pf = ps + P[nP - 1].l + 3;
		if (n_res > 0 && ps <= (int)(uint32_t)res[n_res - 1]) {
			const int f = (int)(uint32_t)res[n_res - 1];
			res[n_res - 1] = (res[n_res - 1] >> 32) << 32 | (uint32_t)(f > pf ? f : pf);
		} else if (n_res < res_cap) res[n_res++] = (uint64_t)(uint32_t)ps << 32 | (uint32_t)pf;
		else *err = 1;
		while (nP > 0 && P[nP - 1].start < wstart) --nP;
	};
	for (int i = 0, l = 0, t = 0; i <= len; ++i) {
		const int b = i < len ? base(i) : 4;
		if (b < 4) {
			++l, t = (t << 2 | b) & 63;
			if (l < 3) continue;
			const int wstart = (l > W ? l - W : 0) + (i + 1 - l);
			flush(wstart);
			// shift_window: the oldest triplet leaves (and the valid suffix, if that reaches so far), t enters
			if (n >= cap) {
				const int o = win[head];
				head = head + 1 == cap ? 0 : head + 1, --n;
				rw -= --cw[o];
				if (L > n) --L, rv -= --cv[o];
			}
			{ int p = head + n; if (p >= cap) p -= cap; win[p] = t; }
			++n, ++L;
			rw += cw[t]++;
			rv += cv[t]++;
			if (cv[t] * 10 > 2 * T) { // t too frequent in the valid suffix: cut it just past t's oldest occurrence there
				int o;
				do {
					int p = head + n - L; if (p >= cap) p -= cap;
					o = win[p];
					rv -= --cv[o];
					--L;
				} while (o != t);
			}
			if (rw * 10 > L * T) { // find_perfect: the suffixes longer than the valid one, shortest first
				int c[64];
				for (int j = 0; j < 64; ++j) c[j] = cv[j];
				int r = rv, best_r = 0, best_l = 0;
				for (int x = n - L - 1; x >= 0; --x) {
					int p = head + x; if (p >= cap) p -= cap;
					const int u = win[p];
					r += c[u]++;
					const int nl = n - x - 1;
					if (r * 10 <= T * nl) continue;
					int j = 0;
					for (; j < nP && P[j].start >= x + wstart; ++j) // the intervals this one contains: the best ratio among them
						if (best_r == 0 || P[j].r * best_l > best_r * P[j].l) best_r = P[j].r, best_l = P[j].l;
					if (best_r != 0 && r * best_l < best_r * nl) continue;
					best_r = r, best_l = nl;
					if (nP == pcap) return -1;
					for (int m = nP; m > j; --m) P[m] = P[m - 1];
					++nP;
					wm_sdust_perf q; q.start = x + wstart, q.r = (int16_t)r, q.l = (int16_t)nl;
					P[j] = q;
				}
			}
		} else { // end of a piece: what is pending goes out, the window start advancing one base per interval
			int wstart = (l - W + 1 > 0 ? l - W + 1 : 0) + (i + 1 - l);
			while (nP) flush(wstart++);
			l = t = 0;
		}
	}
	return n_res;
}

// mm_dust_minier's test (src/map.c:52-62) for a minimizer ending at base pos with span `span`, against the sorted regions reg[0, n):
// kept unless more than half of [pos - span + 1, pos] is in them.  The reference walks the regions with a cursor that only moves
// forward; the spans' starts rise with the minimizers' positions, plain or homopolymer-compressed, so a binary search for the
// first region that ends after the start finds the same one.
__device__ __forceinline__ bool wm_dust_keep(const uint64_t *reg, int n, int32_t pos, int32_t span)
{
	const int32_t s = pos - (span - 1), e = s + span;
	int lo = 0, hi = n;
	while (lo < hi) { const int m = (lo + hi) >> 1; if ((int32_t)(uint32_t)reg[m] <= s) lo = m + 1; else hi = m; }
	int32_t l = 0;
	for (int v = lo; v < n && (int32_t)(reg[v] >> 32) < e; ++v) {
		const int32_t rs = (int32_t)(reg[v] >> 32), re = (int32_t)(uint32_t)reg[v];
		l += (e < re ? e : re) - (s > rs ? s : rs);
	}
	return l <= span >> 1;
}

// the regions of the tasks of one sketch call, on the device: task i owns reg[reg_off[i], reg_off[i] + reg_n[i])
struct wm_dust_view { const uint64_t *reg; const int64_t *reg_off; const int32_t *reg_n; };
