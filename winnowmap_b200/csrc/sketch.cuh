#pragma once
#include "wm_common.cuh"
#include "pkseq.cuh"
#include "sdust.cuh"

struct wm128_dev { uint64_t x, y; };

// device view of the down-weight filter (ext/bloom/bloom_filter.hpp table + salts)
struct wm_bloom_dev {
	const uint8_t *table;
	uint64_t bits;
	uint32_t salt[2];
	int n_salt;
};

// one sequence to sketch: a slice of the packed pool (pkseq.cuh), seq_off in bases
struct wm_sk_task {
	int64_t seq_off;
	int32_t len;
	uint32_t rid;
};

struct wm_sketch_ws {
	wm_dbuf tasks, offs, ord, elig, flag, cnt, rank, scan_tmp, mz, mz_off;
	wm_dbuf hpc_tasks, hpc_goff, hpc_coff, hpc_ends, hpc_pos, hpc_pk, hpc_nm; // the compressed pool of wm_sketch_run_hpc (untouched otherwise)
	void release()
	{
		tasks.release(); offs.release(); ord.release(); elig.release(); flag.release(); cnt.release(); rank.release(); scan_tmp.release(); mz.release(); mz_off.release();
		hpc_tasks.release(); hpc_goff.release(); hpc_coff.release(); hpc_ends.release(); hpc_pos.release(); hpc_pk.release(); hpc_nm.release();
	}
};

struct wm_bloom_s;
// sizes (in 32-bit words) of the two arrays of a packed pool of n bases, look-ahead included
static inline size_t wm_pk_words(int64_t n) { return (size_t)((n + 31) / 32) * 2 + WM_PK_SLACK + 4; }
static inline size_t wm_nm_words(int64_t n) { return (size_t)((n + 31) / 32) + WM_PK_SLACK + 4; }
// ASCII (16-byte aligned device buffer) -> packed pool; the second form gathers reads scattered over a device ASCII pool
void wm_pack_ascii(const char *d_in, int64_t n, uint32_t *d_pk, uint32_t *d_nm, cudaStream_t st);
void wm_pack_gather(const char *d_pool, const int64_t *d_src_off, const int64_t *d_dst_off, int n_reads, int64_t n, uint32_t *d_pk, uint32_t *d_nm, cudaStream_t st);
// dust (may be null): the SDUST regions of the tasks (wm_sdust_run); a minimizer mm_dust_minier would remove is not emitted
void wm_sketch_run(wm_sketch_ws *ws, const wm_bloom_dev &bf, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks,
                   int w, int k, int64_t *n_mz, cudaStream_t st, const wm_dust_view *dust = 0);
// the same on homopolymer-compressed sequences (mm_sketch with is_hpc = 1): the tasks are compacted on the device first;
// positions and spans of the minimizers refer to the uncompressed bases (and the SDUST regions to the uncompressed tasks)
void wm_sketch_run_hpc(wm_sketch_ws *ws, const wm_bloom_dev &bf, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks,
                       int w, int k, int64_t *n_mz, cudaStream_t st, const wm_dust_view *dust = 0);
// SDUST (sdust.cu) of every task with threshold T and window W (3..WM_SDUST_WMAX); *view points into ws on return
// (asynchronous on st: wm_sdust_check after the caller's next synchronisation of st exits if the regions overflowed)
struct wm_sdust_ws {
	wm_dbuf tasks, order, back, reg_off, reg_n, reg, P, err;
	int *h_err = 0; // pinned
	void release()
	{
		tasks.release(); order.release(); back.release(); reg_off.release(); reg_n.release(); reg.release(); P.release(); err.release();
		if (h_err) cudaFreeHost(h_err), h_err = 0;
	}
	~wm_sdust_ws() { if (h_err) cudaFreeHost(h_err); }
};
void wm_sdust_run(wm_sdust_ws *ws, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks, int T, int W, wm_dust_view *view, cudaStream_t st);
void wm_sdust_check(const wm_sdust_ws *ws);
// span (x & 0xff) of each of n minimizers
void wm_mz_spans(const wm128_dev *d_mz, int64_t n, uint8_t *d_span, cudaStream_t st);
void wm_bloom_dev_from_table(wm_bloom_dev *d, const uint8_t *d_table, uint64_t bits);
void wm_bloom_params(const wm_bloom_s *b, uint64_t *bits, uint32_t *salt, int *n_salt);
