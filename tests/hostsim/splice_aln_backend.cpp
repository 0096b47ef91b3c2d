// TEST INFRASTRUCTURE ONLY: spliced base-level alignment (-x splice / splice:hq / cdna or --splice, with -c / -a) through the
// product's host orchestration on the oracle backend.  splice_backend.cpp is compiled unchanged into this file, with the harness it
// picks (parts_backend.cpp, or hpc_backend.cpp under WMT_SPLICE_HPC), so the chaining is the cDNA restatement as there.  What this
// file adds: the oracle's run_dp serves a batch whose DpScoring asks for splice with the oracle's ksw_exts2 (wmo_ksw_exts2, no
// junction annotation), from the scoring the orchestration passes, not from the options; and an entry point that makes the options
// of a -c / -a run, which check_opt answers with -8 (spliced alignment is a library path).
#include "splice_backend.cpp"

extern "C" int wmo_ksw_exts2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, const int8_t *mat, int q, int e, int q2, int noncan,
                             int zdrop, int junc_bonus, int flag, const uint8_t *junc, wmo_ez_t *ez, uint32_t *cigar_out, int max_cigar);

namespace {
int64_t g_n_exts2 = 0; // DP jobs served by wmo_ksw_exts2

struct SpliceDp : wmh::Backend { // in front of the oracle backend itself
	CpuBackend *cpu;
	std::vector<std::vector<uint32_t>> cigs;
	void begin_batch(const std::vector<const wm_read*> &r) override { cpu->begin_batch(r); }
	void set_resident_pool(const char *p) override { cpu->set_resident_pool(p); }
	void seed_chain(const std::vector<wmh::SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const wmh::ChainParams cp[2], int max_occ,
	                std::vector<wmh::SeedOut> &out) override { cpu->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out); }
	void run_dp(const std::vector<wmh::DpJob> &jobs, const std::vector<wmh::MapWin> &wins, const wmh::DpScoring &sc, std::vector<wmh::DpRes> &res) override
	{
		if (!sc.splice) { cpu->run_dp(jobs, wins, sc, res); return; }
		const int n = (int)jobs.size();
		res.assign(n, wmh::DpRes()); cigs.assign(n, {});
		g_n_exts2 += n;
		#pragma omp parallel for schedule(dynamic, 8)
		for (int i = 0; i < n; ++i) {
			const wmh::DpJob &J = jobs[i];
			std::vector<uint8_t> q, t;
			cpu->fetch(J.q, wins[J.task], q); cpu->fetch(J.t, wins[J.task], t);
			wmo_ez_t ez;
			cigs[i].resize(J.q.len + J.t.len + 2);
			wmo_ksw_exts2(J.q.len, q.data(), J.t.len, t.data(), sc.mat, sc.q, sc.e, sc.q2, sc.noncan, J.zdrop, sc.junc_bonus, J.flag & 0xffff, 0, &ez,
			              cigs[i].data(), (int)cigs[i].size());
			wmh::DpRes &r = res[i];
			r.max = ez.max, r.zdropped = ez.zdropped, r.max_q = ez.max_q, r.max_t = ez.max_t, r.mqe = ez.mqe, r.mqe_t = ez.mqe_t, r.mte = ez.mte, r.mte_q = ez.mte_q;
			r.score = ez.score, r.reach_end = ez.reach_end, r.n_cigar = ez.n_cigar, r.cigar = cigs[i].data();
		}
	}
	void run_ll(const std::vector<wmh::LlJob> &j, const std::vector<wmh::MapWin> &w, const wmh::DpScoring &s, std::vector<wmh::LlRes> &r) override { cpu->run_ll(j, w, s, r); }
	void end_batch() override { cpu->end_batch(); }
};

void map_batch_aln(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                   std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, wmh::MapStats *stats)
{
	SpliceDp d;
	d.cpu = static_cast<CpuBackend*>(be);
#if defined(WMT_SPLICE_HPC)
	CdnaFromParams w; // map_batch_splice's -H route, with SpliceDp under the cDNA wrapper
	w.in = &d;
	wm_host_idx H = *mi;
	H.flag = WM_I_HPC;
	SpanBackend sb;
	sb.in = &w, sb.mi = &H, sb.bloom = d.cpu->bloom;
	wmh::map_batch(&sb, &H, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
#else
	map_batch_splice(&d, mi, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
#endif
}
const bool g_aln_mapping = (g_map_batch = map_batch_aln, true);
} // namespace

extern "C" int64_t wmt_splice_aln_n_exts2(void) { return g_n_exts2; }
// the next runs' single index carries junction intervals (what wm_gpu_idx_upload_flag records from WM_IDX_JUNC)
static bool g_junc = false;
extern "C" void wmt_splice_aln_set_junc(int on) { g_junc = on != 0; }

// winnowmap [-W kmers] -x preset [--splice] [-G N] (-c | -a) [flags] [-C noncan] [--cap-sw-mem N] [-H] [-I part_bases [--split-prefix]]
// ref.fa reads.fa: set_flags / clear_flags are the MM_F_* bits the other options set or clear (--cs, --MD, --eqx, -Y, -u,
// --splice-flank), noncan < 0 keeps the preset's -C.  The number of index parts, or what the run returned when it failed.
extern "C" int wmt_map_file_splice_aln(const char *ref_fn, const char *kmer_fn, const char *preset, int splice, int max_intron_len, int sam,
                                       int64_t set_flags, int64_t clear_flags, int noncan, int64_t max_sw_mat, const char *reads_fn,
                                       const char *out_fn, int n_threads, uint64_t part_bases, int split)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	wmh::set_opt(0, &io, &mo);
	if (wmh::set_opt(preset, &io, &mo) < 0) return -1;
	if (splice) mo.flag |= WM_F_SPLICE;
	wmh::mapopt_max_intron_len(&mo, max_intron_len);
	mo.flag |= sam ? WM_F_OUT_SAM | WM_F_CIGAR : WM_F_OUT_CG | WM_F_CIGAR;
	mo.flag = (mo.flag | set_flags) & ~clear_flags;
	if (noncan >= 0) mo.noncan = noncan;
	mo.max_sw_mat = max_sw_mat;
	if ((mo.flag & WM_F_SPLICE_FOR) || (mo.flag & WM_F_SPLICE_REV)) mo.flag |= WM_F_SPLICE; // mm_mapopt_update (src/options.c:73)
	const int chk = wmh::check_opt(&io, &mo);
	if (chk < 0 && chk != -8) return -2;
	int rc;
	if (!part_bases) {
		OracleIndex X;
		if ((rc = load_oracle_index(ref_fn, kmer_fn, io.k, io.w, X)) < 0) return rc;
		X.H.junc = g_junc;
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
	OracleIndex F;
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
