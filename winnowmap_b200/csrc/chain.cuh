#pragma once
#include "wm_common.cuh"
#include "sketch.cuh"

// arguments of mm_chain_dp (reference src/chain.c:22)
struct wm_chain_params {
	int32_t max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float gap_scale;
};

struct wm_chain_sets { wm_chain_params p[2]; }; // stage-1/fallback and stage-2 parameter sets: what the kernels read
// is_cdna: the cDNA gap cost of mm_chain_dp (src/chain.c:69-77), the same for both sets (map.c passes is_splice at every call);
// wm_chain_run launches the instantiation of the forward pass it selects
struct wm_chain_params2 : wm_chain_sets { int32_t is_cdna = 0; };

struct wm_chain_ws {
	wm_dbuf f, p, t, v, u, u2, w, b, n_u, n_b, counter, order, stacks;
	// the forward passes of the three task classes (giant / medium / small) run side by side
	cudaStream_t side_st[2] = {0, 0}; cudaEvent_t ev_fork = 0, ev_join[2] = {0, 0};
	void drop_streams() {
		if (!side_st[0]) return;
		for (int i = 0; i < 2; ++i) { cudaStreamDestroy(side_st[i]); cudaEventDestroy(ev_join[i]); side_st[i] = 0; }
		cudaEventDestroy(ev_fork);
	}
	~wm_chain_ws() { drop_streams(); }
	void release() {
		drop_streams();
 f.release(); p.release(); t.release(); v.release(); u.release(); u2.release(); w.release(); b.release();
	                 n_u.release(); n_b.release(); counter.release(); order.release(); stacks.release();
	}
};

void wm_chain_run(wm_chain_ws *ws, wm128_dev *d_a, const int64_t *d_off, const int64_t *h_off, int n_tasks, const wm_chain_params2 &PP, const uint8_t *d_set_id, cudaStream_t st);
