// SDUST on the device (sdust.cuh): the low-complexity regions of every sequence one sketch call covers, one thread per
// sequence, and the C-ABI batch entry the parity tests drive.
#include <string.h>
#include <algorithm>
#include <vector>
#include "wm_common.cuh"
#include "sketch.cuh"
#include "sdust.cuh"

struct wm_sdust_pk_base { // base i of a task of the packed pool
	wm_pkseq s; int64_t off;
	__device__ __forceinline__ int operator()(int i) const { return wm_pk_get(s, off + i); }
};

// Pass 1: threads take the tasks longest first (order[]), grid-stride, each with WM_SDUST_PCAP_FAST perfect intervals at
// P[g * WM_SDUST_PCAP_FAST, ..); a task that needs more goes to the list `back`.  Pass 2 (back != 0 in pass 1 only) runs the
// listed tasks again with WM_SDUST_PCAP entries per thread.
template <bool FIRST>
__global__ void __launch_bounds__(128)
wm_sdust_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int32_t *__restrict__ order, const int32_t *__restrict__ n_order,
                int T, int W, wm_sdust_perf *__restrict__ P_all, uint64_t *__restrict__ reg, const int64_t *__restrict__ reg_off,
                int32_t *__restrict__ reg_n, int32_t *__restrict__ back, int32_t *__restrict__ n_back, int *__restrict__ err)
{
	const int pcap = FIRST ? WM_SDUST_PCAP_FAST : WM_SDUST_PCAP;
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
	wm_sdust_perf *P = P_all + g * pcap;
	const int n = *n_order;
	for (int64_t j = g; j < n; j += stride) {
		const int t = order[j];
		const wm_sk_task T_ = tasks[t];
		wm_sdust_pk_base b; b.s = seq, b.off = T_.seq_off;
		const int64_t cap = reg_off[t + 1] - reg_off[t];
		const int64_t r = wm_sdust_seq(b, T_.len, T, W, P, pcap, reg + reg_off[t], cap, err);
		if (r >= 0) reg_n[t] = (int32_t)r;
		else if (FIRST) back[atomicAdd(n_back, 1)] = t;
		else *err = 1; // cannot happen at WM_SDUST_PCAP
	}
}

void wm_sdust_run(wm_sdust_ws *ws, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks, int T, int W, wm_dust_view *view, cudaStream_t st)
{
	std::vector<int64_t> off(n_tasks + 1, 0);
	std::vector<int32_t> order(n_tasks + 1);
	for (int i = 0; i < n_tasks; ++i) off[i + 1] = off[i] + wm_sdust_reg_cap(h_tasks[i].len > 0 ? h_tasks[i].len : 0, W), order[i] = i;
	std::stable_sort(order.begin(), order.begin() + n_tasks, [&](int a, int b) { return h_tasks[a].len > h_tasks[b].len; });
	order[n_tasks] = n_tasks; // the number of tasks, read by pass 1 from the device
	int dev = 0, n_sm = 0;
	WM_CUDA_CHECK(cudaGetDevice(&dev));
	WM_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	// pass 1: 4 warps per SM with 2 KB of P each (35 MB on 132 SMs); pass 2: one warp per SM with 32 KB each (138 MB); one buffer
	const int n_blk1 = (int)((std::min<int64_t>(std::max(n_tasks, 1), (int64_t)n_sm * 128) + 127) / 128), n_blk2 = (n_sm + 3) / 4;
	const size_t n_p1 = (size_t)WM_SDUST_PCAP_FAST * n_blk1 * 128, n_p2 = (size_t)WM_SDUST_PCAP * n_blk2 * 128;
	wm_sk_task *d_tasks = (wm_sk_task*)ws->tasks.need(sizeof(wm_sk_task) * (n_tasks + 1));
	int32_t *d_order = (int32_t*)ws->order.need(sizeof(int32_t) * (n_tasks + 1));
	int32_t *d_back = (int32_t*)ws->back.need(sizeof(int32_t) * (n_tasks + 1)); // [0, n): tasks of pass 2, [n]: their number
	int64_t *d_off = (int64_t*)ws->reg_off.need(sizeof(int64_t) * (n_tasks + 1));
	int32_t *d_n = (int32_t*)ws->reg_n.need(sizeof(int32_t) * (n_tasks + 1));
	uint64_t *d_reg = (uint64_t*)ws->reg.need(sizeof(uint64_t) * (off[n_tasks] + 1));
	wm_sdust_perf *d_P = (wm_sdust_perf*)ws->P.need(sizeof(wm_sdust_perf) * std::max(n_p1, n_p2));
	int *d_err = (int*)ws->err.need(sizeof(int));
	if (!ws->h_err) WM_CUDA_CHECK(cudaMallocHost((void**)&ws->h_err, sizeof(int)));
	WM_CUDA_CHECK(wm_memcpy_async(d_tasks, h_tasks, sizeof(wm_sk_task) * n_tasks, cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_order, order.data(), sizeof(int32_t) * (n_tasks + 1), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_off, off.data(), sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_back + n_tasks, 0, sizeof(int32_t), st));
	if (n_tasks > 0) {
		wm_count_launch(); wm_sdust_kernel<true><<<n_blk1, 128, 0, st>>>(seq, d_tasks, d_order, d_order + n_tasks, T, W, d_P, d_reg, d_off, d_n,
		                                                                 d_back, d_back + n_tasks, d_err);
		WM_CUDA_CHECK(cudaGetLastError());
		wm_count_launch(); wm_sdust_kernel<false><<<n_blk2, 128, 0, st>>>(seq, d_tasks, d_back, d_back + n_tasks, T, W, d_P, d_reg, d_off, d_n,
		                                                                  0, 0, d_err);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	// read at the caller's next synchronisation of st (wm_sdust_check): no round trip of its own
	WM_CUDA_CHECK(cudaMemcpyAsync(ws->h_err, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
	view->reg = d_reg, view->reg_off = d_off, view->reg_n = d_n;
}

void wm_sdust_check(const wm_sdust_ws *ws)
{
	if (ws->h_err && *ws->h_err) { // cannot happen at the bounds of sdust.cuh; a wrong region list must not pass silently
		fprintf(stderr, "[ERROR] winnowmap-b200: SDUST overflowed its interval or region list\n");
		exit(1);
	}
}

// ---- C ABI: batched sdust_core ----
extern "C" int wm_sdust_batch(int n, const char *seq, const int64_t *off, int T, int W, uint64_t **reg, int64_t **reg_off)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] wm_sdust_batch: no CUDA device visible; winnowmap-b200 has no CPU fallback\n");
		exit(1);
	}
	if (!(T >= 1 && T <= WM_SDUST_MAX_T && W >= 3 && W <= WM_SDUST_WMAX) || n < 0) {
		fprintf(stderr, "[ERROR] wm_sdust_batch: T must be in 1..%d and W in 3..%d\n", WM_SDUST_MAX_T, WM_SDUST_WMAX);
		return -1;
	}
	*reg_off = (int64_t*)calloc(n + 1, sizeof(int64_t));
	*reg = (uint64_t*)malloc(sizeof(uint64_t));
	if (n == 0) return 0;
	const int64_t tot = off[n];
	char *d_ascii = wm_dev_alloc<char>(tot + 16);
	uint32_t *d_pk = wm_dev_alloc<uint32_t>(wm_pk_words(tot)), *d_nm = wm_dev_alloc<uint32_t>(wm_nm_words(tot));
	if (tot > 0) WM_CUDA_CHECK(cudaMemcpy(d_ascii, seq, tot, cudaMemcpyHostToDevice));
	wm_pack_ascii(d_ascii, tot, d_pk, d_nm, 0);
	wm_pkseq pks; pks.pk = d_pk, pks.nm = d_nm;
	std::vector<wm_sk_task> tasks(n);
	for (int i = 0; i < n; ++i) tasks[i].seq_off = off[i], tasks[i].len = (int32_t)(off[i + 1] - off[i]), tasks[i].rid = 0;
	wm_sdust_ws ws;
	wm_dust_view v;
	wm_sdust_run(&ws, pks, tasks.data(), n, T, W, &v, 0);
	WM_CUDA_CHECK(cudaStreamSynchronize(0));
	wm_sdust_check(&ws);
	std::vector<int64_t> cap_off(n + 1);
	std::vector<int32_t> cnt(n);
	WM_CUDA_CHECK(cudaMemcpy(cap_off.data(), v.reg_off, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(cnt.data(), v.reg_n, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
	std::vector<uint64_t> all(cap_off[n] + 1);
	WM_CUDA_CHECK(cudaMemcpy(all.data(), v.reg, sizeof(uint64_t) * cap_off[n], cudaMemcpyDeviceToHost));
	for (int i = 0; i < n; ++i) (*reg_off)[i + 1] = (*reg_off)[i] + cnt[i];
	free(*reg);
	*reg = (uint64_t*)malloc(sizeof(uint64_t) * ((*reg_off)[n] + 1));
	for (int i = 0; i < n; ++i) memcpy(*reg + (*reg_off)[i], all.data() + cap_off[i], sizeof(uint64_t) * cnt[i]);
	ws.release();
	cudaFree(d_ascii); cudaFree(d_pk); cudaFree(d_nm);
	return 0;
}

// bench: the SDUST kernel alone over a batch (as wm_sdust_batch lays it out); *ms = CUDA-event time of one wm_sdust_run, the mean
// over `reps` runs after one untimed run (workspaces sized).  The host's part of a run (task order, offsets) is inside the window,
// and so are both passes.
extern "C" int wm_bench_sdust(int n, const char *seq, const int64_t *off, int T, int reps, double *ms)
{
	if (n <= 0 || reps <= 0 || T < 1 || T > WM_SDUST_MAX_T) return -1;
	const int64_t tot = off[n];
	char *d_ascii = wm_dev_alloc<char>(tot + 16);
	uint32_t *d_pk = wm_dev_alloc<uint32_t>(wm_pk_words(tot)), *d_nm = wm_dev_alloc<uint32_t>(wm_nm_words(tot));
	WM_CUDA_CHECK(cudaMemcpy(d_ascii, seq, tot, cudaMemcpyHostToDevice));
	wm_pack_ascii(d_ascii, tot, d_pk, d_nm, 0);
	wm_pkseq pks; pks.pk = d_pk, pks.nm = d_nm;
	std::vector<wm_sk_task> tasks(n);
	for (int i = 0; i < n; ++i) tasks[i].seq_off = off[i], tasks[i].len = (int32_t)(off[i + 1] - off[i]), tasks[i].rid = 0;
	wm_sdust_ws ws;
	wm_dust_view v;
	cudaEvent_t e0, e1;
	WM_CUDA_CHECK(cudaEventCreate(&e0)); WM_CUDA_CHECK(cudaEventCreate(&e1));
	for (int r = -1; r < reps; ++r) {
		if (r == 0) WM_CUDA_CHECK(cudaEventRecord(e0, 0));
		wm_sdust_run(&ws, pks, tasks.data(), n, T, 64, &v, 0);
	}
	WM_CUDA_CHECK(cudaEventRecord(e1, 0));
	WM_CUDA_CHECK(cudaEventSynchronize(e1));
	wm_sdust_check(&ws);
	float f = 0.f;
	WM_CUDA_CHECK(cudaEventElapsedTime(&f, e0, e1));
	*ms = f / reps;
	cudaEventDestroy(e0); cudaEventDestroy(e1);
	ws.release();
	cudaFree(d_ascii); cudaFree(d_pk); cudaFree(d_nm);
	return 0;
}
