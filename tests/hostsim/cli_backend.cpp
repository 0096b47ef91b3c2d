// TEST INFRASTRUCTURE ONLY: the product's command line (csrc/host_cli.cpp) over oracle-backed index parts, as
// parts_backend.cpp (compiled unchanged into this file) runs the file driver: the reference cut into parts as mm_idx_gen
// cuts it, one oracle index per part sketched with one -W filter, -f resolved per part by the restatement of
// mm_idx_cal_max_occ.  tests/cli_lib.py compiles it with the product's host sources into a temporary directory.
#include "parts_backend.cpp"
#include "../../winnowmap_b200/csrc/host_cli.h"

namespace {

struct CliOracleParts : OracleParts {
	OracleIndex F;
	std::vector<std::unique_ptr<OracleIndex>> X;
	std::vector<std::unique_ptr<CpuBackend>> owned;
	~CliOracleParts() override { for (auto &b : owned) if (b->idx) wmo_idx_free(b->idx); }
};

std::unique_ptr<IndexParts> build_oracle_parts(const CliArgs &a)
{
	std::unique_ptr<CliOracleParts> ix(new CliOracleParts());
	if (load_kmer_filter(a.has_kmer ? a.kmer_fn.c_str() : 0, a.ipt.k, ix->F) < 0) return nullptr;
	for (int n = 1; (int)ix->X.size() < n;) {
		ix->X.emplace_back(new OracleIndex());
		n = load_oracle_seqs(a.files[0].c_str(), a.ipt.k, a.ipt.w, ix->F.bloom, *ix->X.back(), a.ipt.batch_size, a.ipt.mini_batch_size, (int)ix->X.size() - 1);
		if (n < 0) return nullptr;
	}
	for (auto &x : ix->X) {
		x->H.flag = a.ipt.flag & WM_I_HPC;
		if (x->H.flag) { fprintf(stderr, "[ERROR] the oracle command-line harness has no -H index\n"); return nullptr; }
		ix->owned.emplace_back(new CpuBackend());
		CpuBackend &b = *ix->owned.back();
		b.hidx = &x->H, b.bloom = ix->F.bloom, b.idx = wmo_idx_build(x->mz.data(), (long)x->mz.size() / 2);
		ix->add(&b, &x->H);
		const std::vector<uint32_t> c = occ_counts(*x);
		ix->f_mid_occ.push_back(wm_oracle_cal_max_occ(c.data(), (int64_t)c.size(), a.opt.mid_occ_frac));
	}
	return std::unique_ptr<IndexParts>(ix.release());
}

} // namespace

// `winnowmap argv[1..]` on oracle backends: the exit status
extern "C" int wmt_cli_main(int argc, char **argv)
{
	const int rc = cli_main(argc, argv, build_oracle_parts);
	fflush(stdout);
	return rc;
}

#include "../../oracle/cli_dump.h"

// The options `winnowmap argv[1..]` maps with, with n_cpu processors, written to dump_fn in the format of
// oracle/cli_dump.h when the command line gets as far as mapping; otherwise nothing is written.  The status cli_main
// would return at that point, 0 when mapping would start.
extern "C" int wmt_cli_parse(int argc, char **argv, int n_cpu, const char *dump_fn)
{
	CliArgs a;
	const int rc = cli_parse(argc, argv, a, n_cpu);
	if (rc >= 0) return rc;
	cli_update_opt(&a.opt);
	std::vector<const char*> files;
	for (auto &f : a.files) files.push_back(f.c_str());
	FILE *fp = fopen(dump_fn, "w");
	wm_cli_dump(fp, &a.ipt, sizeof(a.ipt), &a.opt, sizeof(a.opt), offsetof(wm_mapopt_t, kmer_freq_filename), offsetof(wm_mapopt_t, split_prefix),
	            a.n_threads, (a.opt.flag & WM_F_OUT_SAM) && a.has_rg ? a.rg.c_str() : 0, (int)files.size(), files.data());
	fclose(fp);
	return 0;
}
