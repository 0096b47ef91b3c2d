// TEST INFRASTRUCTURE ONLY: the host orchestration on the oracle backend of cpu_backend.cpp (compiled unchanged into this
// file) with the seed filter of overlap_oracle.h: whole mapping runs under -D / --dual=no / -X / --for-only / --rev-only.
#include "cpu_backend.cpp"
#include "overlap_oracle.h"

// winnowmap [-W kmers] -x preset [-c | -a] <flags> ref.fa reads.fa on the oracle backend with the filter.  out_mode: 0 PAF
// without CIGAR, 1 -c, 2 -a.  `flags` is or-ed into the mapping flags (MM_F_NO_DIAG, MM_F_NO_DUAL, MM_F_ALL_CHAINS, ...).
extern "C" int wmt_map_file_overlap(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads,
                                    int out_mode, int64_t flags)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	set_opt(0, &io, &mo);
	if (preset && set_opt(preset, &io, &mo) < 0) return -1;
	if (out_mode == 2) mo.flag |= WM_F_OUT_SAM | WM_F_CIGAR;
	else if (out_mode == 1) mo.flag |= WM_F_OUT_CG | WM_F_CIGAR;
	mo.flag |= flags;
	if (check_opt(&io, &mo) < 0) return -2;
	OracleIndex X;
	int rc = load_oracle_index(ref_fn, kmer_fn, io.k, io.w, X);
	if (rc < 0) return rc;
	set_name_order(&X.H);
	OverlapCpuBackend be;
	be.flag = mo.flag;
	be.hidx = &X.H; be.bloom = X.bloom; be.idx = wmo_idx_build(X.mz.data(), (long)X.mz.size() / 2);
	rc = map_reads_to(&be, X.H, mo, reads_fn, out_fn, n_threads, out_mode == 2);
	wmo_idx_free(be.idx);
	return rc;
}

// The rank reduction of the device filter against strcmp: for n index names and m query names (query j with has[j] == 0 has
// no name), out[j * n + i] = the (cmp > 0, cmp == 0) pair the SKIP_* bits and ranks imply, as bit 0 and bit 1, or 4 when
// the filter would not test names.
extern "C" void wmt_name_filter(int n, const char *const *names, int m, const char *const *qnames, const int *has, uint8_t *out)
{
	wm_host_idx H;
	for (int i = 0; i < n; ++i) H.name.push_back(names[i]);
	set_name_order(&H);
	for (int j = 0; j < m; ++j) {
		wm_read r; r.name = has[j] ? qnames[j] : ""; r.has_name = has[j] != 0;
		uint32_t lt;
		const uint32_t b = skip_bits(&H, WM_F_NO_DIAG | WM_F_NO_DUAL, &r, &lt);
		for (int i = 0; i < n; ++i) {
			if (!(b & SKIP_NO_DUAL)) { out[(size_t)j * n + i] = 4; continue; }
			const uint32_t rk = H.name_rank[i];
			out[(size_t)j * n + i] = (uint8_t)((rk < lt ? 1 : 0) | ((b & SKIP_NAME_EQ) && rk == lt ? 2 : 0));
		}
	}
}
