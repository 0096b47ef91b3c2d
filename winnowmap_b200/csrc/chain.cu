// Anchor chaining on sm_90a: mm_chain_dp (reference src/chain.c:22-167) for n_segs == 1 and
// is_cdna == 0, one warp per task.
//
// Forward pass (:45-90): anchors are taken in order; for anchor i the 32 lanes score 32 predecessors
// j = i-1, i-2, ... at a time.  The reference's inner loop is order dependent (running maximum with
// strict ">", the n_skip counter fed by t[j]==i marks, "break" above max_skip, and the t[p[j]] = i side
// effects); a chunk is resolved exactly by (1) letting every candidate lane publish t[p[j]] = i, which
// can only touch indices below every j still to be examined, (2) a prefix maximum over the lanes to
// find the record-setting lanes, and (3) replaying the n_skip arithmetic over the ballot masks.
// Backtracking (:92-165) is a second warp-per-task kernel: the data-parallel sweeps use all lanes, the
// greedy claim walk (:118-135) is inherently serial and runs on lane 0.
#include <vector>
#include <algorithm>
#include <limits.h>
#include <stdlib.h>
#include "wm_common.cuh"
#include "sketch.cuh"
#include "rsort.cuh"
#include "chain.cuh"

#define WM_CHAIN_WARPS 4
#define WM_CHAIN_DENSE_MIN 1024 // tasks with more anchors use the dense-candidate scan when WM_CHAIN_DENSE=1

#include "chain_dev.cuh"

// Tasks come largest first (order[]), one warp per task.
__global__ void __launch_bounds__(WM_CHAIN_WARPS * 32)
wm_chain_fill_kernel(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int n_tasks,
                     wm_chain_params2 PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all, int32_t *__restrict__ v_all,
                     int *counter)
{
	const unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	for (;;) {
		int ti = 0;
		if (lane == 0) ti = atomicAdd(counter, 1);
		ti = __shfl_sync(FULL, ti, 0);
		if (ti >= n_tasks) break;
		const int task = order ? order[ti] : ti;
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (n <= 0) continue;
		wm_chain_fill_warp(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base, lane);
	}
}

// The same forward pass with the dense-candidate scan of chain_dev.cuh (selected with WM_CHAIN_DENSE=1).
__global__ void __launch_bounds__(WM_CHAIN_WARPS * 32)
wm_chain_fill_dense_kernel(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int n_tasks,
                           wm_chain_params2 PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all,
                           int32_t *__restrict__ v_all, int *counter)
{
	const unsigned FULL = 0xffffffffu;
	__shared__ int32_t D[WM_CHAIN_WARPS][WM_CHAIN_DENSE_CAP];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (;;) {
		int ti = 0;
		if (lane == 0) ti = atomicAdd(counter, 1);
		ti = __shfl_sync(FULL, ti, 0);
		if (ti >= n_tasks) break;
		const int task = order ? order[ti] : ti;
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (n <= 0) continue;
		// the dense scan pays off where windows are long (big tasks: repeats); ordinary tasks keep the plain chunk loop
		if (n > WM_CHAIN_DENSE_MIN) wm_chain_fill_warp_dense(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base, D[wid], lane);
		else wm_chain_fill_warp(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base, lane);
	}
}

// Window start of every anchor (src/chain.c:49-55 in closed form, chain_dev.cuh), one thread per anchor, into v[].
__global__ void wm_chain_window_kernel(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, int n_tasks, int64_t n_a,
                                       wm_chain_params2 PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ v_all)
{
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n_a) return;
	int lo = 0, hi = n_tasks; // the task that holds anchor g: last t with off[t] <= g
	while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (off[m] <= g) lo = m; else hi = m; }
	const int64_t base = off[lo];
	v_all[g] = wm_chain_window_start(a_all + base, (int)(g - base), PP.p[set_id ? set_id[lo] : 0]);
}

// The forward pass with the sliding window of each warp's task in a shared-memory ring (chain_dev.cuh).  Tasks
// order[first .. last), one warp per task, pulled from a counter.
template <int RING, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
wm_chain_fill_ring_kernel(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int first, int last,
                          wm_chain_params2 PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all,
                          int32_t *__restrict__ v_all, int *counter)
{
	const unsigned FULL = 0xffffffffu;
	extern __shared__ __align__(16) unsigned char wm_chain_smem[];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	wm_chain_ring<RING> *R = (wm_chain_ring<RING>*)wm_chain_smem + wid;
	for (;;) {
		int ti = 0;
		if (lane == 0) ti = first + atomicAdd(counter, 1);
		ti = __shfl_sync(FULL, ti, 0);
		if (ti >= last) break;
		const int task = order[ti];
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (n <= 0) continue;
		wm_chain_fill_warp_ring<RING>(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base, R, lane);
		__syncwarp();
	}
}

// Giant tasks: one CTA per task, warp k owns anchor k of every 32-anchor tile, dataflow between the warps (chain_dev.cuh).
__global__ void __launch_bounds__(WM_CT_WARPS * 32, 1)
wm_chain_fill_tile_kernel(const wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int first, int last,
                          wm_chain_params2 PP, const uint8_t *__restrict__ set_id, int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all,
                          int32_t *__restrict__ v_all, int *counter)
{
	const unsigned FULL = 0xffffffffu;
	constexpr int MASK = WM_CT_RING - 1;
	extern __shared__ __align__(16) unsigned char wm_chain_smem[];
	wm_chain_tile_sm *S = (wm_chain_tile_sm*)wm_chain_smem;
	__shared__ int s_task;
	__shared__ unsigned long long s_sum[WM_CT_WARPS];
	const int tid = threadIdx.x, lane = tid & 31, k = tid >> 5;
	for (;;) {
		if (tid == 0) s_task = first + atomicAdd(counter, 1);
		__syncthreads();
		const int ti = s_task;
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
				// tile T - 2 and everything before it must be complete; its done-slot + 6 (tile T - 4's) is free for tile T + 4
				// (the polls sleep a little: 32 warps spinning on shared memory slow the loads of the warps that are scanning)
				if (T >= 2) { while (done[(T - 2) & 7] != FULL) __nanosleep(64); }
				if (lane == 0) done[(T + 4) & 7] = 0;
				const int st = __shfl_sync(FULL, stl, k);
				const int ring_lo = i0 + 64 - WM_CT_RING; // older slots are being overwritten by the anchors of the two active tiles
				const uint64_t ri = __shfl_sync(FULL, cur.x, k); const int32_t qi = (int32_t)__shfl_sync(FULL, cur.y, k);
				// the anchors of this tile and of the one before that this one depends on: its candidate predecessors (a geometric property)
				const unsigned Cc = __ballot_sync(FULL, lane < k && il >= st && wm_chain_is_cand(cur, ri, qi, P));
				const unsigned Cp = T > 0 ? __ballot_sync(FULL, il - 32 >= st && wm_chain_is_cand(prev, ri, qi, P)) : 0u;
				if (Cp) { while ((done[(T - 1) & 7] & Cp) != Cp) __nanosleep(32); }
				if (Cc) { while ((done[T & 7] & Cc) != Cc) __nanosleep(32); }
				__threadfence_block();
				int max_f, max_j;
				if (!wm_chain_tile_scan(a, P, f, p, t, S, mk, cur, prev, i0, k, st, ring_lo, false, avg_d, scale_d, lane, &max_f, &max_j)) {
					if (lane == 0) { while (atomicCAS(&S->lock, 0, 1) != 0) __nanosleep(64); }
					__syncwarp();
					__threadfence_block();
					wm_chain_tile_scan(a, P, f, p, t, S, mk, cur, prev, i0, k, st, ring_lo, true, avg_d, scale_d, lane, &max_f, &max_j);
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

#define WM_CHAIN_SMALL_N 128    // tasks up to this many anchors: ring of the same size, eight warps per CTA
template <int RING, int WARPS>
static void wm_chain_launch_ring(int grid, cudaStream_t st, const wm128_dev *a, const int64_t *off, const int32_t *order, int first, int last,
                                 const wm_chain_params2 &PP, const uint8_t *set_id, int32_t *f, int32_t *p, int32_t *t, int32_t *v, int *counter)
{
	const size_t smem = sizeof(wm_chain_ring<RING>) * WARPS;
	static bool attr_set = false;
	if (!attr_set) { WM_CUDA_CHECK(cudaFuncSetAttribute(wm_chain_fill_ring_kernel<RING, WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr_set = true; }
	wm_count_launch();
	wm_chain_fill_ring_kernel<RING, WARPS><<<grid, WARPS * 32, smem, st>>>(a, off, order, first, last, PP, set_id, f, p, t, v, counter);
	WM_CUDA_CHECK(cudaGetLastError());
}

// Backtracking (chain_dev.cuh): tasks order[first .. last), one warp per task ...
__global__ void __launch_bounds__(WM_CHAIN_WARPS * 32)
wm_chain_backtrack_kernel(wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int first, int last,
                          wm_chain_params2 PP, const uint8_t *__restrict__ set_id,
                          int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all, int32_t *__restrict__ v_all,
                          uint64_t *__restrict__ u_all, uint64_t *__restrict__ u2_all, wm128_dev *__restrict__ w_all, wm128_dev *__restrict__ b_all,
                          int32_t *__restrict__ n_u_out, int64_t *__restrict__ n_b_out, int *counter)
{
	const unsigned FULL = 0xffffffffu;
	__shared__ wm_rs_warp_ws W[WM_CHAIN_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (;;) {
		int ti = 0;
		if (lane == 0) ti = first + atomicAdd(counter, 1);
		ti = __shfl_sync(FULL, ti, 0);
		if (ti >= last) break;
		const int task = order[ti];
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (lane == 0) n_u_out[task] = 0, n_b_out[task] = 0;
		if (n <= 0) continue;
		__syncwarp();
		wm_chain_backtrack_grp<false>(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base,
		                              u_all + 2 * base, u2_all + base, w_all + base, b_all + base, &W[wid], n_u_out + task, n_b_out + task, lane, 32, 0);
	}
}

// ... and one CTA per giant task
__global__ void __launch_bounds__(1024)
wm_chain_backtrack_cta_kernel(wm128_dev *__restrict__ a_all, const int64_t *__restrict__ off, const int32_t *__restrict__ order, int n_giant,
                              wm_chain_params2 PP, const uint8_t *__restrict__ set_id,
                              int32_t *__restrict__ f_all, int32_t *__restrict__ p_all, int32_t *__restrict__ t_all, int32_t *__restrict__ v_all,
                              uint64_t *__restrict__ u_all, uint64_t *__restrict__ u2_all, wm128_dev *__restrict__ w_all, wm128_dev *__restrict__ b_all,
                              int32_t *__restrict__ n_u_out, int64_t *__restrict__ n_b_out)
{
	__shared__ wm_rs_warp_ws W;
	__shared__ int sm[64];
	for (int ti = blockIdx.x; ti < n_giant; ti += gridDim.x) {
		const int task = order[ti];
		const int64_t base = off[task];
		const int n = (int)(off[task + 1] - base);
		if (threadIdx.x == 0) n_u_out[task] = 0, n_b_out[task] = 0;
		__syncthreads();
		if (n <= 0) continue;
		wm_chain_backtrack_grp<true>(a_all + base, n, PP.p[set_id ? set_id[task] : 0], f_all + base, p_all + base, t_all + base, v_all + base,
		                             u_all + 2 * base, u2_all + base, w_all + base, b_all + base, &W, n_u_out + task, n_b_out + task, (int)threadIdx.x, (int)blockDim.x, sm);
		__syncthreads();
	}
}

// Chains for n_tasks anchor arrays a[off[t]..off[t+1]) (device, sorted).  Results are left in place:
// d_a holds the chained anchors of task t at off[t].. (n_b[t] of them), ws->u2 the (score<<32|cnt) words
// at off[t].. (n_u[t] of them).
void wm_chain_run(wm_chain_ws *ws, wm128_dev *d_a, const int64_t *d_off, const int64_t *h_off, int n_tasks, const wm_chain_params2 &PP, const uint8_t *d_set_id, cudaStream_t st)
{
	if (n_tasks <= 0) return;
	const int64_t n_a = h_off[n_tasks];
	int32_t *f = (int32_t*)ws->f.need(sizeof(int32_t) * (n_a + 1)), *p = (int32_t*)ws->p.need(sizeof(int32_t) * (n_a + 1));
	int32_t *t = (int32_t*)ws->t.need(sizeof(int32_t) * (n_a + 1)), *v = (int32_t*)ws->v.need(sizeof(int32_t) * (n_a + 1));
	uint64_t *u = (uint64_t*)ws->u.need(sizeof(uint64_t) * (2 * n_a + 2)), *u2 = (uint64_t*)ws->u2.need(sizeof(uint64_t) * (n_a + 1));
	wm128_dev *w = (wm128_dev*)ws->w.need(sizeof(wm128_dev) * (n_a + 1)), *b = (wm128_dev*)ws->b.need(sizeof(wm128_dev) * (n_a + 1));
	int32_t *n_u = (int32_t*)ws->n_u.need(sizeof(int32_t) * (n_tasks + 1));
	int64_t *n_b = (int64_t*)ws->n_b.need(sizeof(int64_t) * (n_tasks + 1));
	if (n_a == 0) { // no task has an anchor (a wave of reads without a seed hit in this index): no chain, and no launch of size 0
		WM_CUDA_CHECK(cudaMemsetAsync(n_u, 0, sizeof(int32_t) * n_tasks, st));
		WM_CUDA_CHECK(cudaMemsetAsync(n_b, 0, sizeof(int64_t) * n_tasks, st));
		return;
	}
	int *counter = (int*)ws->counter.need(8 * sizeof(int));
	WM_CUDA_CHECK(cudaMemsetAsync(counter, 0, 8 * sizeof(int), st));
	// largest tasks first
	std::vector<int32_t> order(n_tasks);
	for (int i = 0; i < n_tasks; ++i) order[i] = i;
	std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return h_off[x + 1] - h_off[x] > h_off[y + 1] - h_off[y]; });
	int32_t *d_order = (int32_t*)ws->order.need(sizeof(int32_t) * n_tasks);
	WM_CUDA_CHECK(wm_memcpy_async(d_order, order.data(), sizeof(int32_t) * n_tasks, cudaMemcpyHostToDevice, st));
	const int n_sm = wm_sm_count();
	int grid = n_sm * (32 / WM_CHAIN_WARPS);
	const int need = (n_tasks + WM_CHAIN_WARPS - 1) / WM_CHAIN_WARPS;
	if (grid > need) grid = need;
	// formulation of the forward pass: 0 = plain warp loop, 1 = dense candidates, 2 = shared-memory ring (default)
	static int mode = -1, ring_big = 1024, tile_min = 2048, bt_cta_min = 4096;
	if (mode < 0) {
		const char *e = getenv("WM_CHAIN_DENSE"), *m = getenv("WM_CHAIN_MODE"), *r = getenv("WM_CHAIN_RING"), *tm = getenv("WM_CHAIN_TILE_MIN");
		if (tm && atoi(tm) > 0) tile_min = atoi(tm);
		if (getenv("WM_CHAIN_BT_CTA_MIN") && atoi(getenv("WM_CHAIN_BT_CTA_MIN")) > 0) bt_cta_min = atoi(getenv("WM_CHAIN_BT_CTA_MIN"));
		mode = m ? atoi(m) : (e && *e == '1') ? 1 : 2;
		if (r) ring_big = atoi(r);
		if (ring_big != 512 && ring_big != 1024 && ring_big != 2048) ring_big = 1024;
	}
	const int pslot = wm_prof_launch_begin(WM_PK_CHAIN, st, st, 0);
	wm_prof_add(WM_PK_CHAIN, 32.0 * (double)n_a, (double)n_a, 0); // SURVEY.md 8d: 16 A in (anchors) + 16 A out (f, p, t, v)
	if (mode == 2) {
		if (!ws->side_st[0]) {
			int lo = 0, hi = 0;
			WM_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
			for (int i = 0; i < 2; ++i) {
				WM_CUDA_CHECK(cudaStreamCreateWithPriority(&ws->side_st[i], cudaStreamNonBlocking, hi));
				WM_CUDA_CHECK(cudaEventCreateWithFlags(&ws->ev_join[i], cudaEventDisableTiming));
			}
			WM_CUDA_CHECK(cudaEventCreateWithFlags(&ws->ev_fork, cudaEventDisableTiming));
		}
		// counters: [0] giant tasks, [1] backtrack, [2] medium tasks, [3] small tasks
		wm_count_launch();
		wm_chain_window_kernel<<<(unsigned)((n_a + 255) / 256), 256, 0, st>>>(d_a, d_off, n_tasks, n_a, PP, d_set_id, v);
		WM_CUDA_CHECK(cudaGetLastError());
		// order[] is by size, descending: giant tasks (tile kernel, one CTA each), medium (one warp each, ring), small
		int n_giant = 0, n_big = 0;
		while (n_giant < n_tasks && h_off[order[n_giant] + 1] - h_off[order[n_giant]] > tile_min) ++n_giant;
		n_big = n_giant;
		while (n_big < n_tasks && h_off[order[n_big] + 1] - h_off[order[n_big]] > WM_CHAIN_SMALL_N) ++n_big;
		const int n_medium = n_big - n_giant, n_small = n_tasks - n_big;
		const int n_classes = (n_giant > 0) + (n_medium > 0) + (n_small > 0);
		if (n_classes > 1) WM_CUDA_CHECK(cudaEventRecord(ws->ev_fork, st));
		int side = 0; bool main_used = false;
		cudaStream_t joined[2]; int n_joined = 0;
		auto pick = [&]() -> cudaStream_t { // the first class present runs on the caller's stream, the others beside it
			if (!main_used) { main_used = true; return st; }
			cudaStream_t s2 = ws->side_st[side++];
			WM_CUDA_CHECK(cudaStreamWaitEvent(s2, ws->ev_fork, 0));
			joined[n_joined++] = s2;
			return s2;
		};
		if (n_giant > 0) {
			cudaStream_t s2 = pick();
			static bool attr_set = false;
			const size_t smem = sizeof(wm_chain_tile_sm);
			if (!attr_set) { WM_CUDA_CHECK(cudaFuncSetAttribute(wm_chain_fill_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr_set = true; }
			wm_count_launch();
			static int tile_ctas = -1; // WM_CHAIN_TILE_CTAS: SMs the tile kernel may hold at once (a CTA takes a whole SM's registers)
			if (tile_ctas < 0) { const char *e = getenv("WM_CHAIN_TILE_CTAS"); tile_ctas = e && atoi(e) > 0 ? atoi(e) : n_sm; }
			const int g_t = n_giant < tile_ctas ? n_giant : tile_ctas;
			wm_chain_fill_tile_kernel<<<g_t, WM_CT_WARPS * 32, smem, s2>>>(d_a, d_off, d_order, 0, n_giant, PP, d_set_id, f, p, t, v, counter);
			WM_CUDA_CHECK(cudaGetLastError());
		}
		if (n_medium > 0) {
			cudaStream_t s2 = pick();
			const int per_sm = ring_big == 512 ? 3 : ring_big == 1024 ? 2 : 1; // CTAs of 4 warps
			int g = n_sm * per_sm; const int need_b = (n_medium + 3) / 4;
			if (g > need_b) g = need_b;
			if (ring_big == 512) wm_chain_launch_ring<512, 4>(g, s2, d_a, d_off, d_order, n_giant, n_big, PP, d_set_id, f, p, t, v, counter + 2);
			else if (ring_big == 1024) wm_chain_launch_ring<1024, 4>(g, s2, d_a, d_off, d_order, n_giant, n_big, PP, d_set_id, f, p, t, v, counter + 2);
			else wm_chain_launch_ring<2048, 4>(g, s2, d_a, d_off, d_order, n_giant, n_big, PP, d_set_id, f, p, t, v, counter + 2);
		}
		if (n_small > 0) {
			cudaStream_t s2 = pick();
			int g = n_sm * 6; const int need_s = (n_small + 7) / 8;
			if (g > need_s) g = need_s;
			wm_chain_launch_ring<WM_CHAIN_SMALL_N, 8>(g, s2, d_a, d_off, d_order, n_big, n_tasks, PP, d_set_id, f, p, t, v, counter + 3);
		}
		for (int i = 0; i < n_joined; ++i) {
			WM_CUDA_CHECK(cudaEventRecord(ws->ev_join[i], joined[i]));
			WM_CUDA_CHECK(cudaStreamWaitEvent(st, ws->ev_join[i], 0));
		}
	} else {
		wm_count_launch();
		if (mode == 1) wm_chain_fill_dense_kernel<<<grid, WM_CHAIN_WARPS * 32, 0, st>>>(d_a, d_off, d_order, n_tasks, PP, d_set_id, f, p, t, v, counter);
		else wm_chain_fill_kernel<<<grid, WM_CHAIN_WARPS * 32, 0, st>>>(d_a, d_off, d_order, n_tasks, PP, d_set_id, f, p, t, v, counter);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	wm_prof_launch_end(pslot, st);
	{ // backtracking: giant tasks by a CTA each, the others by a warp each (order[] is by size, descending)
		int n_giant = 0;
		while (n_giant < n_tasks && h_off[order[n_giant] + 1] - h_off[order[n_giant]] > bt_cta_min) ++n_giant;
		if (n_giant > 0) {
			wm_count_launch();
			wm_chain_backtrack_cta_kernel<<<n_giant < 2 * n_sm ? n_giant : 2 * n_sm, 1024, 0, st>>>(d_a, d_off, d_order, n_giant, PP, d_set_id, f, p, t, v, u, u2, w, b, n_u, n_b);
			WM_CUDA_CHECK(cudaGetLastError());
		}
		if (n_tasks > n_giant) {
			wm_count_launch();
			wm_chain_backtrack_kernel<<<grid, WM_CHAIN_WARPS * 32, 0, st>>>(d_a, d_off, d_order, n_giant, n_tasks, PP, d_set_id, f, p, t, v, u, u2, w, b, n_u, n_b, counter + 1);
			WM_CUDA_CHECK(cudaGetLastError());
		}
	}
}

// ---- C ABI ----
extern "C" int wm_chain_dp_batch(int n_tasks, const wm128_dev *a, const int64_t *off,
                                 int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter,
                                 int min_cnt, int min_sc, float gap_scale,
                                 int32_t *n_u, uint64_t *u, wm128_dev *b, int64_t *n_b)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] wm_chain_dp_batch: no CUDA device visible; winnowmap-b200 has no CPU fallback\n");
		exit(1);
	}
	if (n_tasks <= 0) return 0;
	const int64_t n = off[n_tasks];
	wm128_dev *d_a = wm_dev_alloc<wm128_dev>(n + 1);
	int64_t *d_off = wm_dev_alloc<int64_t>(n_tasks + 1);
	WM_CUDA_CHECK(cudaMemcpy(d_a, a, sizeof(wm128_dev) * n, cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_off, off, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice));
	wm_chain_params2 PP;
	wm_chain_params &P = PP.p[0];
	P.max_dist_x = max_dist_x, P.min_dist_x = min_dist_x, P.max_dist_y = max_dist_y, P.bw = bw, P.max_skip = max_skip, P.max_iter = max_iter;
	P.min_cnt = min_cnt, P.min_sc = min_sc, P.gap_scale = gap_scale;
	PP.p[1] = P;
	wm_chain_ws ws;
	wm_chain_run(&ws, d_a, d_off, off, n_tasks, PP, 0, 0);
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	WM_CUDA_CHECK(cudaMemcpy(n_u, ws.n_u.p, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(n_b, ws.n_b.p, sizeof(int64_t) * n_tasks, cudaMemcpyDeviceToHost));
	if (n > 0) {
		WM_CUDA_CHECK(cudaMemcpy(u, ws.u2.p, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost));
		WM_CUDA_CHECK(cudaMemcpy(b, d_a, sizeof(wm128_dev) * n, cudaMemcpyDeviceToHost));
	}
	ws.release();
	cudaFree(d_a); cudaFree(d_off);
	return 0;
}
