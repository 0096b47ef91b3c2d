#pragma once
#include "chain_dev.cuh"

// The CTA body of wm_chain_fill_tile_kernel (chain.cu): tasks order[first .. last) pulled from a counter, one CTA per task, thread tid of
// WM_CT_WARPS * 32.  S: the dynamic shared memory, s_task / s_sum: the kernel's static shared variables.  A function of its own so that
// the tests can run it, unchanged, on an emulated CTA (tests/hostsim/tile_cta_emul.cpp).  It lives apart from chain_dev.cuh, whose
// warp-level functions also compile for the host with nothing but the warp intrinsics: this one needs the CTA ones (__syncthreads,
// __nanosleep, atomicCAS, atomicExch, __threadfence_block, __ldcg).  CDNA: the gap cost of is_cdna (wm_chain_score).
template <bool CDNA = false>
__device__ __forceinline__ void wm_chain_fill_tile_cta(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int first,
                                                       int last, const wm_chain_sets &PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ f_all,
                                                       int32_t *__restrict__ p_all, int32_t *__restrict__ t_all, int32_t *__restrict__ v_all, int *counter,
                                                       wm_chain_tile_sm *S, int *s_task, unsigned long long *s_sum, int tid)
{
	const unsigned FULL = 0xffffffffu;
	constexpr int MASK = WM_CT_RING - 1;
	const int lane = tid & 31, k = tid >> 5;
	for (;;) {
		if (tid == 0) *s_task = first + atomicAdd(counter, 1);
		__syncthreads();
		const int ti = *s_task;
		__syncthreads();
		if (ti >= last) break;
		const int task = order[ti];
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (n <= 0) continue;
		const wm128_dev *a = a_all + base;
		int32_t *f = f_all + base, *p = p_all + base, *t = t_all + base, *v = v_all + base;
		const wm_chain_params P = PP.p[set_id ? set_id[task] : 0];
		// avg_qspan (src/chain.c:41-42); t[] is only used by the locked deep path
		unsigned long long sum = 0;
		for (int i = tid; i < n; i += WM_CT_WARPS * 32) { sum += a[i].y >> 32 & 0xff; t[i] = 0; }
		for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
		if (lane == 0) s_sum[k] = sum;
		if (tid < 8) S->done[tid] = 0;
		if (tid == 0) S->lock = 0;
		__syncthreads();
		sum = 0;
		for (int w = 0; w < WM_CT_WARPS; ++w) sum += s_sum[w];
		const float avg_qspan = __fdiv_rn(__ull2float_rn(sum), __ll2float_rn((long long)n));
		const double avg_d = (double)avg_qspan, scale_d = (double)P.gap_scale;
		uint32_t *mk = S->marks[k];
		volatile unsigned *done = S->done;
		wm128_dev prev; prev.x = prev.y = 0;
		for (int T = 0, i0 = 0; i0 < n; ++T, i0 += 32) {
			const int il = i0 + lane;
			wm128_dev cur; cur.x = cur.y = 0; int stl = 0;
			if (il < n) { cur = a[il]; stl = v[il]; }
			const int i = i0 + k;
			if (i < n) {
				const int st = __shfl_sync(FULL, stl, k);
				const int ring_lo = i0 + 64 - WM_CT_RING; // older slots are being overwritten by the anchors of the two active tiles
				const uint64_t ri = __shfl_sync(FULL, cur.x, k); const int32_t qi = (int32_t)__shfl_sync(FULL, cur.y, k);
				// between its two phases the scan waits here: Cc / Cp are the anchors of this tile and of the one before that this one
				// depends on, its candidate predecessors there (phase A, before the wait, lists the window's candidates)
				auto wait = [&](unsigned Cc, unsigned Cp) {
					// tile T - 2 and everything before it must be complete; its done-slot + 6 (tile T - 4's) is free for tile T + 4
					// (the polls sleep a little: 32 warps spinning on shared memory slow the loads of the warps that are scanning)
					if (T >= 2) { while (done[(T - 2) & 7] != FULL) __nanosleep(64); }
					if (lane == 0) done[(T + 4) & 7] = 0;
					if (Cp) { while ((done[(T - 1) & 7] & Cp) != Cp) __nanosleep(32); }
					if (Cc) { while ((done[T & 7] & Cc) != Cc) __nanosleep(32); }
					__threadfence_block();
				};
				int max_f, max_j;
				if (!wm_chain_tile_scan<CDNA>(a, P, f, p, t, S, mk, cur, prev, i0, k, st, ring_lo, false, avg_d, scale_d, lane, &max_f, &max_j, wait)) {
					if (lane == 0) { while (atomicCAS(&S->lock, 0, 1) != 0) __nanosleep(64); }
					__syncwarp();
					__threadfence_block();
					wm_chain_tile_scan<CDNA>(a, P, f, p, t, S, mk, cur, prev, i0, k, st, ring_lo, true, avg_d, scale_d, lane, &max_f, &max_j);
					__syncwarp();
					__threadfence_block();
					if (lane == 0) atomicExch(&S->lock, 0);
				}
				int vj = INT_MIN;
				if (max_j >= 0) vj = max_j >= ring_lo ? S->v[max_j & MASK] : __ldcg(v + max_j);
				const int vi = (max_j >= 0 && vj > max_f) ? vj : max_f; // src/chain.c:89
				if (lane == 0) {
					const int s = i & MASK;
					S->x[s] = ri; S->q[s] = qi; S->f[s] = max_f; S->p[s] = max_j; S->v[s] = vi;
					f[i] = max_f; p[i] = max_j; v[i] = vi;
					__threadfence_block();
					atomicOr(&S->done[T & 7], 1u << k);
				}
				__syncwarp();
			}
			prev = cur;
		}
		__syncthreads();
	}
}
