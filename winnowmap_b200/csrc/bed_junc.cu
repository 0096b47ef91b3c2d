// Junction annotation on the device (bed_junc.cuh): the intervals of an index uploaded once, one kernel over the target windows
// of a DP launch, the batch entry point wm_bed_junc_batch and the counters of wm_junc_stats.
#include <string.h>
#include <mutex>
#include <utility>
#include <vector>
#include "wm_common.cuh"
#include "bed_junc.cuh"
#include "host_types.h"

__global__ void wm_bed_junc_kernel(const wm_junc_dev I, const wm_junc_win *__restrict__ wins, int n_win, uint8_t *__restrict__ out)
{
	const int64_t wi = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (wi >= n_win) return;
	const wm_junc_win W = wins[wi];
	wm_bed_junc_window(I, W, out + W.dst_off, threadIdx.x & 31);
}

// the intervals of H with strand != 0, on the device; n_seq == 0 when H has none of them
wm_junc_dev wm_junc_upload(const wm_host_idx &H)
{
	wm_junc_dev I; memset(&I, 0, sizeof(I));
	if (!H.has_junc()) return I;
	const size_t n_seq = H.junc_off.size() - 1;
	std::vector<int32_t> st, en; std::vector<int8_t> sd; std::vector<int64_t> off(1, 0);
	for (size_t r = 0; r < n_seq; ++r) {
		for (int64_t i = H.junc_off[r]; i < H.junc_off[r + 1]; ++i) {
			const wm_idx_intv1_t &a = H.junc_iv[i];
			if (a.strand == 0) continue;
			st.push_back(a.st), en.push_back(a.en), sd.push_back((int8_t)(a.strand > 0 ? 1 : -1));
		}
		off.push_back((int64_t)st.size());
	}
	if (st.empty()) return I;
	int32_t *d_st = wm_dev_alloc<int32_t>(st.size()), *d_en = wm_dev_alloc<int32_t>(en.size());
	int8_t *d_sd = wm_dev_alloc<int8_t>(sd.size());
	int64_t *d_off = wm_dev_alloc<int64_t>(off.size());
	WM_CUDA_CHECK(cudaMemcpy(d_st, st.data(), sizeof(int32_t) * st.size(), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_en, en.data(), sizeof(int32_t) * en.size(), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_sd, sd.data(), sd.size(), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_off, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice));
	I.st = d_st, I.en = d_en, I.strand = d_sd, I.off = d_off, I.n_seq = (int32_t)n_seq;
	return I;
}

void wm_junc_free(wm_junc_dev *I)
{
	cudaFree((void*)I->st); cudaFree((void*)I->en); cudaFree((void*)I->strand); cudaFree((void*)I->off);
	memset(I, 0, sizeof(*I));
}

// ---- counters (wm_junc_stats) ----
static std::mutex g_junc_mu;
static long long g_junc_launches = 0, g_junc_windows = 0;
static double g_junc_ms = 0;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_junc_ev; // launches timed while wm_prof_enable is on, not yet read

// the annotation of n windows into `out` (each window's bytes at out + dst_off), on stream st
void wm_bed_junc_run(const wm_junc_dev &I, const wm_junc_win *d_wins, int n, uint8_t *d_out, cudaStream_t st)
{
	if (n <= 0) return;
	cudaEvent_t e0 = 0, e1 = 0;
	if (g_wm_prof.enabled) {
		WM_CUDA_CHECK(cudaEventCreate(&e0)); WM_CUDA_CHECK(cudaEventCreate(&e1));
		WM_CUDA_CHECK(cudaEventRecord(e0, st));
	}
	wm_count_launch(); wm_bed_junc_kernel<<<(unsigned)(((int64_t)n * 32 + 255) / 256), 256, 0, st>>>(I, d_wins, n, d_out);
	WM_CUDA_CHECK(cudaGetLastError());
	std::lock_guard<std::mutex> lk(g_junc_mu);
	if (e0) { WM_CUDA_CHECK(cudaEventRecord(e1, st)); g_junc_ev.push_back(std::make_pair(e0, e1)); }
	++g_junc_launches, g_junc_windows += n;
}

extern "C" void wm_junc_stats(double *o, int reset)
{
	std::lock_guard<std::mutex> lk(g_junc_mu);
	for (auto &e : g_junc_ev) {
		float f = 0.f;
		WM_CUDA_CHECK(cudaEventSynchronize(e.second));
		WM_CUDA_CHECK(cudaEventElapsedTime(&f, e.first, e.second));
		g_junc_ms += f;
		cudaEventDestroy(e.first); cudaEventDestroy(e.second);
	}
	g_junc_ev.clear();
	o[0] = (double)g_junc_launches, o[1] = (double)g_junc_windows, o[2] = g_junc_ms;
	if (reset) g_junc_launches = g_junc_windows = 0, g_junc_ms = 0;
}

extern "C" int wm_bed_junc_batch(const wm_idx_intv_t *I, int n_seq, int n_win, const int32_t *win, uint8_t *out, const int64_t *out_off)
{
	if (n_seq < 0 || n_win < 0 || (n_seq > 0 && !I)) return -1;
	if (n_win == 0) return 0;
	wm_host_idx H;
	H.junc_off.assign(1, 0);
	for (int r = 0; r < n_seq; ++r) {
		for (int32_t i = 0; i < I[r].n; ++i) H.junc_iv.push_back(I[r].a[i]);
		H.junc_off.push_back((int64_t)H.junc_iv.size());
	}
	std::vector<wm_junc_win> w(n_win);
	int64_t pool = 0;
	for (int i = 0; i < n_win; ++i) {
		if (win[4 * i + 2] < 0) return -1;
		w[i].dst_off = pool, w[i].rid = win[4 * i], w[i].off = win[4 * i + 1], w[i].len = win[4 * i + 2], w[i].reversed = win[4 * i + 3] != 0;
		pool += (w[i].len + 15) & ~15; // as run_dp lays out its target slices
	}
	wm_junc_dev D = wm_junc_upload(H);
	wm_junc_win *d_w = wm_dev_alloc<wm_junc_win>(n_win);
	uint8_t *d_out = wm_dev_alloc<uint8_t>(pool + 16);
	WM_CUDA_CHECK(cudaMemcpy(d_w, w.data(), sizeof(wm_junc_win) * n_win, cudaMemcpyHostToDevice));
	wm_bed_junc_run(D, d_w, n_win, d_out, 0);
	std::vector<uint8_t> h((size_t)pool + 1);
	WM_CUDA_CHECK(cudaMemcpy(h.data(), d_out, pool, cudaMemcpyDeviceToHost));
	for (int i = 0; i < n_win; ++i) memcpy(out + out_off[i], h.data() + w[i].dst_off, w[i].len);
	cudaFree(d_w); cudaFree(d_out);
	wm_junc_free(&D);
	return 0;
}
