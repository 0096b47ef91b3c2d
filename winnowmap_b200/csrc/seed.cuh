#pragma once
#include "wm_common.cuh"
#include "sketch.cuh"

// Flattened minimizer index resident in HBM (one replica per GPU).
struct wm_idx_dev {
	int32_t k, w;
	uint32_t n_seq;
	int64_t n_keys;
	const uint64_t *keys;      // sorted unique minimizer hashes (mm128_t.x >> 8)
	const uint64_t *pos_off;   // n_keys + 1
	const uint64_t *pos;       // rid<<32 | pos<<1 | strand, ascending within each list
	const uint64_t *ht_key;    // open addressing: key -> index into keys[]
	const uint32_t *ht_val;
	uint64_t ht_mask;
	const uint32_t *S;         // 4-bit packed reference (mm_idx_t.S)
	const uint64_t *seq_offset;
	const uint32_t *seq_len;
};

struct wm_seed_ws {
	wm_dbuf n_occ, cnt, list_off, tandem, mz_task, a_off, scan_tmp, a, task_a_off, rep_len, n_mini_pos, mini_pos, big_ids, small_ids, rs_stacks, sort_tmp, sort_idx, sort_tok;
	int64_t n_a;
	wm_seed_ws() : n_a(0) {}
	void release() {
		n_occ.release(); cnt.release(); list_off.release(); tandem.release(); mz_task.release(); a_off.release(); scan_tmp.release();
		a.release(); task_a_off.release(); rep_len.release(); n_mini_pos.release(); mini_pos.release(); big_ids.release(); small_ids.release(); rs_stacks.release(); sort_tmp.release(); sort_idx.release(); sort_tok.release();
	}
};

void wm_idx_dev_build_ht(wm_idx_dev *ix, cudaStream_t st);
void wm_anchor_sort_run(wm_seed_ws *ws, wm128_dev *d_a, const int64_t *d_off, const int64_t *h_off, int n_arr, cudaStream_t st, const int32_t *only = 0, int n_only = 0);
void wm_seed_run(wm_seed_ws *ws, const wm_idx_dev &ix, const wm128_dev *d_mz, const int64_t *d_mz_off, int64_t n_mz, int n_tasks,
                 const int32_t *d_qlen, int max_occ, int64_t *h_task_a_off, cudaStream_t st);
