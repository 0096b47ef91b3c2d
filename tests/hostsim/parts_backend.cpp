// TEST INFRASTRUCTURE ONLY: multi-part indexes (-I), --split-prefix and -f on the oracle backend of cpu_backend.cpp (compiled
// unchanged into this file): the reference cut into parts as mm_idx_gen cuts it, one oracle index per part sketched with one
// -W filter, -f resolved per part by the restatement of mm_idx_cal_max_occ (oracle/wm_oracle_occ.c), and the product's
// file driver run part-major or merged.  tests/hostsim/build.sh builds it into libwm_hostsim.so.
#include <memory>
#include "cpu_backend.cpp"

extern "C" int32_t wm_oracle_cal_max_occ(const uint32_t *counts, int64_t n, float f);

// the occurrence count of every key of an index (a singleton counts 1)
static std::vector<uint32_t> occ_counts(const OracleIndex &X)
{
	std::vector<uint64_t> keys(X.mz.size() / 2);
	for (size_t i = 0; i < keys.size(); ++i) keys[i] = X.mz[2 * i] >> 8;
	std::sort(keys.begin(), keys.end());
	std::vector<uint32_t> c;
	for (size_t i = 0; i < keys.size(); ++i) {
		if (i == 0 || keys[i] != keys[i - 1]) c.push_back(0);
		++c.back();
	}
	return c;
}

// winnowmap [-W kmers] -x preset [-c | -a] [-f mid_occ_frac] [-I part_bases] [--split-prefix] ref.fa reads.fa: the number of
// index parts, or what the run returned when it failed.  part_bases 0: one part; mid_occ_frac < 0: no -f.  mid_occ[p]
// (p < cap) is the mid_occ part p mapped with, -1 where it did not map.
extern "C" int wmt_map_file_parts(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads,
                                  int sam, uint64_t part_bases, int split, float mid_occ_frac, int32_t *mid_occ, int cap)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	int rc = run_opts(preset, sam, 0, io, mo);
	if (rc < 0) return rc;
	if (mid_occ_frac >= 0) mo.mid_occ_frac = mid_occ_frac;
	if (split) mo.split_prefix = "split"; // any prefix: the merge runs in memory
	OracleIndex F; // the -W filter of every part
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
		const std::vector<uint32_t> c = occ_counts(*X[p]);
		ix.f_mid_occ.push_back(wm_oracle_cal_max_occ(c.data(), (int64_t)c.size(), mo.mid_occ_frac));
	}
	rc = ix.run(mo, reads_fn, out_fn, n_threads);
	for (size_t p = 0; p < X.size(); ++p) wmo_idx_free(be[p].idx);
	for (int p = 0; p < (int)X.size() && p < cap; ++p) mid_occ[p] = ix.mid_occ[p];
	return rc < 0 ? rc : (int)X.size();
}
