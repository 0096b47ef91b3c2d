// The device boundary of the mapping path.  The orchestrator (host_map.cpp) drives a batch through three
// coarse operations; everything data-parallel lives behind them on the GPU (gpu_backend.cu):
//   seed_chain : sketch -> seed lookup -> anchor sort (-> merge with pre-computed anchors) -> chaining
//   run_dp     : batched ksw_extd2 with traceback
//   run_ll     : batched ksw_ll
// The product links exactly one implementation, the CUDA one.
#pragma once
#include <stdint.h>
#include <vector>
#include "host_types.h"
#include "host_align.h"

namespace wmh {

struct MapWin { int32_t read, wb, wl; }; // a query window: bases [wb, wb+wl) of read `read`

enum { SEED_MASKED = 1, SEED_NO_SKETCH = 2 };

// The per-occurrence filter of skip_seed (src/map.c:132-154) as integer tests.  SKIP_NO_DIAG / SKIP_NO_DUAL are set only
// when the read has a name; with the index names in strcmp order (wm_host_idx::name_rank), for the occurrence's rid:
//   strcmp(qname, name[rid]) > 0   <=>  name_rank[rid] < name_lt
//   strcmp(qname, name[rid]) == 0  <=>  SKIP_NAME_EQ && name_rank[rid] == name_lt
enum { SKIP_NO_DIAG = 1, SKIP_NO_DUAL = 2, SKIP_FOR_ONLY = 4, SKIP_REV_ONLY = 8, SKIP_NAME_EQ = 16 };

struct SeedTask {
	MapWin win;
	int32_t flags;      // SEED_MASKED: sketch a copy whose covered bases are 'N' (src/map.c:793-803); SEED_NO_SKETCH: chain `pre` only
	int32_t chain_set;  // which of the two chaining parameter sets applies (stage-1/fallback vs stage-2)
	int32_t n_mask; int64_t mask_off; // covered intervals [s,e) as int32 pairs in the mask pool
	int32_t n_pre; int64_t pre_off;   // anchors from stage 1 (sorted) in the pre pool (src/map.c:742-774)
	// the filter of the fresh look-ups (the `pre` anchors went through it in stage 1): SKIP_* bits (0: every occurrence is
	// kept, no filter runs) and the number of index names strictly less than the read's name
	uint32_t skip = 0, name_lt = 0;
};

// name_rank / name_sorted of the index (one sort of the names per index)
void set_name_order(wm_host_idx *mi);
// SKIP_* bits and name_lt of one read under the mapping flags `flag` (mi's name order must be set when -D / --dual=no is on)
uint32_t skip_bits(const wm_host_idx *mi, int64_t flag, const wm_read *rd, uint32_t *name_lt);

struct ChainParams { // arguments of mm_chain_dp (src/chain.c:22)
	int32_t max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float gap_scale;
};

struct SeedOut { // views into backend-owned host buffers, valid until the next seed_chain call
	int32_t rep_len;
	int32_t n_mz; const uint32_t *mz_pos; // per query minimizer: position | kept << 31 (kept == passed the occurrence filter)
	const uint8_t *mz_span;               // per query minimizer: its span, with an HPC index only (else null: every span is k)
	int32_t n_u; const uint64_t *u;       // score << 32 | count per chain
	int64_t n_b; const wm_pair_t *b;      // chained anchors, chains concatenated
};

struct DpScoring { int8_t mat[25]; int32_t q, e, q2, e2; };

class Backend {
public:
	virtual ~Backend() {}
	virtual void begin_batch(const std::vector<const wm_read*> &reads) = 0;
	virtual void set_resident_pool(const char *device_ascii) { (void)device_ascii; } // reads with dev_off >= 0 are taken from here instead of the host
	virtual void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool,
	                        const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) = 0;
	// `wins[job.task]` locates the query window of each job
	virtual void run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res) = 0;
	virtual void run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res) = 0;
	virtual void end_batch() = 0;
};

struct MapStats { // work counters for the roofline accounting (SURVEY.md 8d)
	int64_t n_reads, n_bases, n_minimaps, n_sketched_bases, n_minimizers, n_anchors, n_chained, n_dp_jobs, n_dp_cells, n_bt_bytes, n_ll_jobs, n_rounds;
	double t_seed, t_dp, t_host;
};

// mm_map_frag for every read of a batch (src/map.c:279-974 with n_segs == 1): fills regs[i] (malloc-owned, as the
// reference returns them), rep_len[i] and frag_gap[i] exactly as worker_for does (src/map.c:1025-1034).
void map_batch(Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
               std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, MapStats *stats);

} // namespace wmh
