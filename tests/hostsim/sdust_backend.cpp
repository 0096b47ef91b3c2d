// TEST INFRASTRUCTURE ONLY: -T through the product's host orchestration on the oracle backend.  parts_backend.cpp (with
// cpu_backend.cpp) is compiled unchanged into this file, with wmo_sketch redirected by the preprocessor to wmt_sketch_dust: the
// oracle's sketch followed, while a mapping runs with T > 0, by the oracle's squeeze of the minimizers that lie in the SDUST
// regions of the sequence sketched (oracle/wm_oracle_sdust.c).  The oracle backend sketches exactly what the reference sketches
// (stage-1 windows, masked copies, whole reads), so the regions are taken on that.  Batches are mapped through a wrapper whose
// set_sdust sets that T, so the product's map_batch sees a backend that applies it.
#include <atomic>
#include <vector>
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" {
long wmt_sketch_dust(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
long wmo_sketch(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
long wmo_sdust(const char *seq, int len, int T, int W, uint64_t *out, long max_out, int *max_nP);
long wmo_dust_minier(uint64_t *xy, long n, const uint64_t *reg, long n_reg);
}

#define wmo_sketch wmt_sketch_dust
#include "parts_backend.cpp"
#undef wmo_sketch

static std::atomic<int> g_sdust_T(0); // set only while a batch maps: the index is sketched without it

extern "C" long wmt_sketch_dust(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out)
{
	const long n = wmo_sketch(str, len, w, k, rid, bf, out_xy, max_out);
	const int T = g_sdust_T.load();
	if (T <= 0 || n <= 0 || n > max_out) return n;
	std::vector<uint64_t> reg((size_t)len + 80);
	const long n_reg = wmo_sdust(str, len, T, 64, reg.data(), (long)reg.size(), 0);
	return wmo_dust_minier(out_xy, n, reg.data(), n_reg);
}

namespace {
struct DustBackend : wmh::Backend {
	wmh::Backend *in;
	bool set_sdust(int T) override { g_sdust_T = T; return true; }
	void begin_batch(const std::vector<const wm_read*> &r) override { in->begin_batch(r); }
	void set_resident_pool(const char *p) override { in->set_resident_pool(p); }
	void seed_chain(const std::vector<wmh::SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const wmh::ChainParams cp[2], int max_occ,
	                std::vector<wmh::SeedOut> &out) override { in->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out); }
	void run_dp(const std::vector<wmh::DpJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::DpRes> &r) override { in->run_dp(j, w, s, r); }
	void run_ll(const std::vector<wmh::LlJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::LlRes> &r) override { in->run_ll(j, w, s, r); }
	void end_batch() override { in->end_batch(); }
};

void map_batch_dust(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                    std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, wmh::MapStats *stats)
{
	DustBackend d;
	d.in = be;
	wmh::map_batch(&d, mi, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
	g_sdust_T = 0;
}
const bool g_dust_mapping = (g_map_batch = map_batch_dust, true);
} // namespace

// winnowmap [-W kmers] -x preset [-c | -a | neither] [flags] -T T [-I part_bases [--split-prefix]] ref.fa reads.fa: out 0 = PAF
// without CIGAR, 1 = -c, 2 = -a; set_flags are the MM_F_* bits of the other options (-X).  The number of index parts, or what
// the run returned when it failed.
extern "C" int wmt_map_file_sdust(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads,
                                  int out, int64_t set_flags, int T, uint64_t part_bases, int split)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	set_opt(0, &io, &mo);
	if (set_opt(preset, &io, &mo) < 0) return -1;
	if (out == 1) mo.flag |= WM_F_OUT_CG | WM_F_CIGAR;
	else if (out == 2) mo.flag |= WM_F_OUT_SAM | WM_F_CIGAR;
	mo.flag |= set_flags;
	mo.sdust_thres = T;
	if (split) mo.split_prefix = "split"; // any prefix: the merge runs in memory
	if (check_opt(&io, &mo) < 0) return -2;
	int rc;
	OracleIndex F;
	if ((rc = load_kmer_filter(kmer_fn, io.k, F)) < 0) return rc;
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
