// Junction annotation of a DP target (mm_idx_bed_junc, reference src/index.c:780-803): for the window [off, off + len) of
// sequence rid, byte p gets bit 1 / 2 where a + strand interval starts / ends (its first and last base), bit 8 / 4 for a
// - strand interval, for every interval with strand != 0 that lies inside the window.  mm_align1 reverses the left extension's
// bytes (mm_seq_rev, src/align.c:693-694) without swapping the bits; a reversed window is written that way.
//
// One warp per window.  The intervals of a sequence are sorted by start; the warp finds the first one starting at or after
// off and its lanes stride over the following ones until one starts at or after the window's end (every interval has
// st < en, so none further can lie inside).  Isoforms share donors and acceptors, so lanes OR their bits into the 32-bit word
// that holds the byte.  The device code is also compiled for the host by the emulation tests (tests/hostsim/junc_emul.cpp).
#pragma once
#include <stdint.h>

// the intervals of an index on the device: those of sequence rid at [off[rid], off[rid + 1]), sorted by st, strand-0 ones dropped
// (they never mark); n_seq == 0: no intervals
struct wm_junc_dev {
	const int32_t *st, *en;
	const int8_t *strand; // 1: +, -1: -
	const int64_t *off;   // n_seq + 1
	int32_t n_seq;
};

// one target window; its bytes go to out + dst_off, which is 4-byte aligned
struct wm_junc_win { int64_t dst_off; int32_t rid, off, len, reversed; };

// The annotation of window W into `out` (the window's first byte; 4-byte aligned, with (len + 3) / 4 whole words that belong to
// this window alone), by the 32 lanes of one warp.
__device__ __forceinline__ void wm_bed_junc_window(const wm_junc_dev &I, const wm_junc_win &W, uint8_t *out, int lane)
{
	uint32_t *w = (uint32_t*)out;
	const int n_words = (W.len + 3) >> 2;
	for (int i = lane; i < n_words; i += 32) w[i] = 0;
	__syncwarp();
	if (W.rid < 0 || W.rid >= I.n_seq || W.len <= 0) return;
	int64_t lo = I.off[W.rid], hi = I.off[W.rid + 1];
	while (hi > lo) { // the first interval with st >= off (every lane searches; the loads are the same for all)
		const int64_t mid = lo + ((hi - lo) >> 1);
		if (I.st[mid] >= W.off) hi = mid;
		else lo = mid + 1;
	}
	const int64_t end = I.off[W.rid + 1], w_en = (int64_t)W.off + W.len;
	for (int64_t i = lo + lane; i < end; i += 32) {
		const int32_t st = I.st[i];
		if (st >= w_en) break; // sorted: this lane's later intervals start further right
		const int32_t en = I.en[i];
		if (en > w_en) continue;
		const bool plus = I.strand[i] > 0;
		int p0 = st - W.off, p1 = en - 1 - W.off;
		if (W.reversed) p0 = W.len - 1 - p0, p1 = W.len - 1 - p1;
		const uint32_t b0 = plus ? 1u : 8u, b1 = plus ? 2u : 4u;
		atomicOr((unsigned*)&w[p0 >> 2], b0 << ((p0 & 3) * 8));
		atomicOr((unsigned*)&w[p1 >> 2], b1 << ((p1 & 3) * 8));
	}
}

#ifndef WM_HOST_EMUL
#include <cuda_runtime.h>
struct wm_host_idx;
wm_junc_dev wm_junc_upload(const wm_host_idx &H); // bed_junc.cu
void wm_junc_free(wm_junc_dev *I);
void wm_bed_junc_run(const wm_junc_dev &I, const wm_junc_win *d_wins, int n, uint8_t *d_out, cudaStream_t st);
#endif
