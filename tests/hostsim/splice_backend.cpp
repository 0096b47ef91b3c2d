// TEST INFRASTRUCTURE ONLY: spliced mapping without base alignment (-x splice / splice:hq / cdna, --splice, -G) through the product's
// host orchestration on the oracle backend.  One of the existing harnesses is compiled unchanged into this file (tests/splice_lib.py
// picks it): parts_backend.cpp (the plain and the -I / --split-prefix runs), with WMT_SPLICE_HPC hpc_backend.cpp (-H), with
// WMT_SPLICE_TEE tee_backend.cpp (the CUDA backend and the oracle side by side).  Two things change:
//   the oracle's chaining, wmo_chain_dp, is redirected by the preprocessor to wmt_chain_dp_splice, which runs the cDNA restatement
//              (oracle/wm_oracle_cdna.c) when the batch's chaining parameters ask for it;
//   every batch is mapped through a backend wrapper that reads is_cdna from the ChainParams the product's orchestration passes to
//              seed_chain, so the oracle side chains as the product asked, not as the options say.
// The runs map without -c / -a: the options are made here, from the preset, --splice and -G.
#include <stdint.h>
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" {
int wmo_chain_dp(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc, float gap_scale, long n,
                 uint64_t *a_xy, uint64_t *u_out, uint64_t *b_xy, long *n_b);
int wmo_chain_dp_cdna(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc, float gap_scale,
                      long n, uint64_t *a_xy, uint64_t *u_out, uint64_t *b_xy, long *n_b);
}

static int g_cdna = 0;            // is_cdna of the seed_chain call in progress
static int g_cdna_mismatch = 0;   // calls whose two parameter sets disagreed on is_cdna

extern "C" int wmt_chain_dp_splice(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc,
                                   float gap_scale, long n, uint64_t *a_xy, uint64_t *u_out, uint64_t *b_xy, long *n_b)
{
	return (g_cdna ? wmo_chain_dp_cdna : wmo_chain_dp)(max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc, gap_scale, n,
	                                                   a_xy, u_out, b_xy, n_b);
}

#define wmo_chain_dp wmt_chain_dp_splice
#if defined(WMT_SPLICE_TEE)
#include "tee_backend.cpp"
#elif defined(WMT_SPLICE_HPC)
#include "hpc_backend.cpp"
#else
#include "parts_backend.cpp"
#endif
#undef wmo_chain_dp

namespace {
struct CdnaFromParams : wmh::Backend {
	wmh::Backend *in;
	void begin_batch(const std::vector<const wm_read*> &r) override { in->begin_batch(r); }
	void set_resident_pool(const char *p) override { in->set_resident_pool(p); }
	void seed_chain(const std::vector<wmh::SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const wmh::ChainParams cp[2], int max_occ,
	                std::vector<wmh::SeedOut> &out) override
	{
		g_cdna = cp[0].is_cdna;
		g_cdna_mismatch += cp[0].is_cdna != cp[1].is_cdna;
		in->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out);
	}
	void run_dp(const std::vector<wmh::DpJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::DpRes> &r) override { in->run_dp(j, w, s, r); }
	void run_ll(const std::vector<wmh::LlJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::LlRes> &r) override { in->run_ll(j, w, s, r); }
	void end_batch() override { in->end_batch(); }
};

void map_batch_splice(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                      std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, wmh::MapStats *stats)
{
	CdnaFromParams w;
	w.in = be;
#if defined(WMT_SPLICE_HPC)
	// what wmt_map_batch_hpc of hpc_backend.cpp does, with the wrapper between the span backend and the oracle backend
	wm_host_idx H = *mi;
	H.flag = WM_I_HPC;
	SpanBackend sb;
	sb.in = &w, sb.mi = &H, sb.bloom = static_cast<CpuBackend*>(be)->bloom;
	wmh::map_batch(&sb, &H, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
#else
	wmh::map_batch(&w, mi, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
#endif
}
const bool g_splice_mapping = (g_map_batch = map_batch_splice, true);

// winnowmap -x preset [--splice] [-G max_intron_len] without -c / -a (src/main.c:172,216)
int splice_opts(const char *preset, int splice, int max_intron_len, wm_idxopt_t &io, wm_mapopt_t &mo)
{
	wmh::set_opt(0, &io, &mo);
	if (wmh::set_opt(preset, &io, &mo) < 0) return -1;
	if (splice) mo.flag |= WM_F_SPLICE;
	wmh::mapopt_max_intron_len(&mo, max_intron_len);
	return wmh::check_opt(&io, &mo) < 0 ? -2 : 0;
}
} // namespace

extern "C" int wmt_splice_cdna_mismatch(void) { return g_cdna_mismatch; }

#if defined(WMT_SPLICE_TEE)
// the spliced run through the tee: writes the PAF of the served backend and the report (wmt_tee_map_file of tee_backend.cpp)
extern "C" int wmt_tee_map_file_splice(const char *ref_fn, const char *kmer_fn, const char *preset, int splice, int max_intron_len, const char *reads_fn,
                                       const char *out_fn, int n_threads, int64_t budget, int dev_kind, const char *report_fn)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	int rc = splice_opts(preset, splice, max_intron_len, io, mo);
	if (rc < 0) return rc;
	TeeRun R;
	if ((rc = R.init(ref_fn, kmer_fn, io.k, io.w, 0, dev_kind, 0, budget)) < 0) return rc;
	rc = map_file_on(&R.tee, R.X.H, mo, reads_fn, out_fn, n_threads);
	if (R.finish(report_fn) < 0) return -6;
	return rc;
}
#else
// winnowmap [-W kmers] -x preset [--splice] [-G N] [-H] [-I part_bases [--split-prefix]] ref.fa reads.fa: the number of index parts,
// or what the run returned when it failed.  part_bases 0: one index (the HPC build takes no parts).
extern "C" int wmt_map_file_splice(const char *ref_fn, const char *kmer_fn, const char *preset, int splice, int max_intron_len, const char *reads_fn,
                                   const char *out_fn, int n_threads, uint64_t part_bases, int split)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	int rc = splice_opts(preset, splice, max_intron_len, io, mo);
	if (rc < 0) return rc;
	if (!part_bases) {
		OracleIndex X;
		if ((rc = load_oracle_index(ref_fn, kmer_fn, io.k, io.w, X)) < 0) return rc;
		CpuBackend be;
		be.hidx = &X.H; be.bloom = X.bloom; be.idx = wmo_idx_build(X.mz.data(), (long)X.mz.size() / 2);
		rc = map_file_on(&be, X.H, mo, reads_fn, out_fn, n_threads);
		wmo_idx_free(be.idx);
		return rc < 0 ? rc : 1;
	}
#if defined(WMT_SPLICE_HPC)
	return -3;
#else
	if (split) mo.split_prefix = "split"; // any prefix: the merge runs in memory
	OracleIndex F; // the -W filter of every part
	if ((rc = load_kmer_filter(kmer_fn, io.k, F)) < 0) return rc;
	std::vector<std::unique_ptr<OracleIndex>> X;
	for (int n = 1; (int)X.size() < n;) {
		X.emplace_back(new OracleIndex());
		n = load_oracle_seqs(ref_fn, io.k, io.w, F.bloom, *X.back(), part_bases, io.mini_batch_size, (int)X.size() - 1);
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
#endif
}
#endif
