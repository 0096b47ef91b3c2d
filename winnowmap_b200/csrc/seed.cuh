#pragma once
#include "wm_common.cuh"
#include "sketch.cuh"

// the seed filter's per-task bits, same values as SKIP_* of host_backend.h
#define WM_SKIP_NO_DIAG  1
#define WM_SKIP_NO_DUAL  2
#define WM_SKIP_FOR_ONLY 4
#define WM_SKIP_REV_ONLY 8
#define WM_SKIP_NAME_EQ  16

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
	const uint32_t *name_rank; // number of sequence names strictly less than each name under strcmp (wm_host_idx::name_rank)
};

struct wm_seed_ws {
	wm_dbuf n_occ, cnt, list_off, tandem, mz_task, a_off, scan_tmp, a, task_a_off, rep_len, n_mini_pos, mini_pos, big_ids, small_ids, rs_stacks, sort_tmp, sort_idx, sort_tok;
	wm_dbuf keep_off; // the seed filter: exclusive scan of the keep flags
	wm_dbuf heap_flag, heap_ids, heap_g, heap_l; // heap sort: tasks with ties, and the heaps that outgrow shared memory
	int64_t n_a;
	wm_seed_ws() : n_a(0) {}
	void release() {
		n_occ.release(); cnt.release(); list_off.release(); tandem.release(); mz_task.release(); a_off.release(); scan_tmp.release();
		a.release(); task_a_off.release(); rep_len.release(); n_mini_pos.release(); mini_pos.release(); big_ids.release(); small_ids.release(); rs_stacks.release(); sort_tmp.release(); sort_idx.release(); sort_tok.release();
		keep_off.release(); heap_flag.release(); heap_ids.release(); heap_g.release(); heap_l.release();
	}
};

void wm_idx_dev_build_ht(wm_idx_dev *ix, cudaStream_t st);
void wm_anchor_sort_run(wm_seed_ws *ws, wm128_dev *d_a, const int64_t *d_off, const int64_t *h_off, int n_arr, cudaStream_t st, const int32_t *only = 0, int n_only = 0);
void wm_seed_run(wm_seed_ws *ws, const wm_idx_dev &ix, const wm128_dev *d_mz, const int64_t *d_mz_off, int64_t n_mz, int n_tasks,
                 const int32_t *d_qlen, int max_occ, int64_t *h_task_a_off, cudaStream_t st, const uint2 *d_skip = 0, bool heap = false);
// --heap-sort=yes: exits when a replay disagreed with its task's sorted anchors (read after the stream's work is done)
void wm_seed_heap_check(void);
