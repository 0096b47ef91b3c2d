// TEST INFRASTRUCTURE ONLY: --heap-sort=yes through the product's host orchestration on the oracle backend.  parts_backend.cpp
// (with cpu_backend.cpp) is compiled unchanged into this file, with wmo_collect_seed_hits redirected by the preprocessor to
// wmt_collect_heap: while a mapping runs with heap sort, the oracle's restatement of collect_seed_hits_heap
// (oracle/wm_oracle_heap.c) instead of the sorted collection.  Every seed collection the backend makes (stage-1 windows, masked
// copies, whole reads) goes through it, as every call site of the reference does.  Batches are mapped through a wrapper whose
// set_heap_sort sets the switch, so the product's map_batch sees a backend that applies it.
#include <atomic>
#include <vector>
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" {
long wmt_collect_heap(const void *ix, int max_occ, const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a, int *rep_len,
                      uint64_t *mini_pos, int *n_mini_pos);
long wmo_collect_seed_hits(const void *ix, int max_occ, const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a, int *rep_len,
                           uint64_t *mini_pos, int *n_mini_pos);
long wmo_collect_seed_hits_heap(const void *ix, int64_t flag, int max_occ, const char *qname, const char *const *names, const uint32_t *seq_len,
                                const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a, int *rep_len, uint64_t *mini_pos,
                                int *n_mini_pos);
}

#define wmo_collect_seed_hits wmt_collect_heap
#include "parts_backend.cpp"
#undef wmo_collect_seed_hits

static std::atomic<int> g_heap(0); // set only while a batch maps with heap sort

// (this backend serves no seed filter: no flag, no read name)
extern "C" long wmt_collect_heap(const void *ix, int max_occ, const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a, int *rep_len,
                                 uint64_t *mini_pos, int *n_mini_pos)
{
	if (!g_heap.load()) return wmo_collect_seed_hits(ix, max_occ, mv_xy, n_mv, qlen, a_xy, max_a, rep_len, mini_pos, n_mini_pos);
	return wmo_collect_seed_hits_heap(ix, 0, max_occ, 0, 0, 0, mv_xy, n_mv, qlen, a_xy, max_a, rep_len, mini_pos, n_mini_pos);
}

namespace {
struct HeapBackend : wmh::Backend {
	wmh::Backend *in;
	bool set_heap_sort(bool on) override { g_heap = on ? 1 : 0; return true; }
	void begin_batch(const std::vector<const wm_read*> &r) override { in->begin_batch(r); }
	void set_resident_pool(const char *p) override { in->set_resident_pool(p); }
	void seed_chain(const std::vector<wmh::SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const wmh::ChainParams cp[2], int max_occ,
	                std::vector<wmh::SeedOut> &out) override { in->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out); }
	void run_dp(const std::vector<wmh::DpJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::DpRes> &r) override { in->run_dp(j, w, s, r); }
	void run_ll(const std::vector<wmh::LlJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::LlRes> &r) override { in->run_ll(j, w, s, r); }
	void end_batch() override { in->end_batch(); }
};

void map_batch_heap(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                    std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, wmh::MapStats *stats)
{
	HeapBackend h;
	h.in = be;
	wmh::map_batch(&h, mi, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
	g_heap = 0;
}
const bool g_heap_mapping = (g_map_batch = map_batch_heap, true);
} // namespace

// winnowmap -x preset [-c | -a | neither] --heap-sort=yes [-I part_bases [--split-prefix]] ref.fa reads.fa: out 0 = PAF without
// CIGAR, 1 = -c, 2 = -a.  The number of index parts, or what the run returned when it failed.
extern "C" int wmt_map_file_heap(const char *ref_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads, int out,
                                 uint64_t part_bases, int split)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	set_opt(0, &io, &mo);
	if (set_opt(preset, &io, &mo) < 0) return -1;
	if (out == 1) mo.flag |= WM_F_OUT_CG | WM_F_CIGAR;
	else if (out == 2) mo.flag |= WM_F_OUT_SAM | WM_F_CIGAR;
	mo.flag |= WM_F_HEAP_SORT;
	if (split) mo.split_prefix = "split"; // any prefix: the merge runs in memory
	if (check_opt(&io, &mo) < 0) return -2;
	int rc;
	OracleIndex F;
	if ((rc = load_kmer_filter(0, io.k, F)) < 0) return rc;
	std::vector<std::unique_ptr<OracleIndex>> X;
	for (int n = 1; (int)X.size() < n;) {
		X.emplace_back(new OracleIndex());
		n = load_oracle_seqs(ref_fn, io.k, io.w, F.bloom, *X.back(), part_bases ? part_bases : UINT64_MAX, io.mini_batch_size, (int)X.size() - 1);
		if (n < 0) return n;
	}
	std::vector<CpuBackend> be(X.size());
	OracleParts ix;
	for (size_t p = 0; p < X.size(); ++p) {
		be[p].hidx = &X[p]->H, be[p].bloom = F.bloom, be[p].idx = wmo_idx_build(X[p]->mz.data(), (long)X[p]->mz.size() / 2);
		ix.add(&be[p], &X[p]->H);
	}
	rc = ix.run(mo, reads_fn, out_fn, n_threads);
	for (size_t p = 0; p < X.size(); ++p) wmo_idx_free(be[p].idx);
	return rc < 0 ? rc : (int)X.size();
}
