// TEST INFRASTRUCTURE ONLY: spliced base-level alignment with junction annotation (--junc-bed) through the product's host
// orchestration on the oracle backend.  splice_aln_backend.cpp is compiled unchanged into this file (with its splice harness and
// its entry point wmt_map_file_splice_aln); what this file adds is a DP backend in front of its SpliceDp that gives every splice
// DP the oracle's annotation of the job's target window (wmo_bed_junc, oracle/wm_oracle_junc.c, compiled in here).  The intervals
// are what the product's BED reader (read_bed_junc, as wm_idx_bed_read runs it) reads for the names of the index part the job
// maps against; wmt_map_file_junc_aln names the BED for one run.
#include <map>
#include <mutex>
#include "splice_aln_backend.cpp"
extern "C" {
#include "../../oracle/wm_oracle_junc.c"
}

namespace {
std::string g_bed;                                       // the BED of the run in progress (empty: none)
std::mutex g_iv_mu;
std::map<const wm_host_idx*, wm_host_idx> g_iv;          // per index part of the run: its names and the intervals read for them

const wm_host_idx *intervals_of(const wm_host_idx *H)
{
	if (g_bed.empty()) return 0;
	std::lock_guard<std::mutex> lk(g_iv_mu);
	auto it = g_iv.find(H);
	if (it == g_iv.end()) {
		wm_host_idx &J = g_iv[H];
		J.name = H->name;
		if (wmh::read_bed_junc(&J, g_bed.c_str()) < 0) { fprintf(stderr, "[ERROR] cannot read %s\n", g_bed.c_str()); exit(1); }
		return &J;
	}
	return &it->second;
}

struct JuncDp : SpliceDp {
	void run_dp(const std::vector<wmh::DpJob> &jobs, const std::vector<wmh::MapWin> &wins, const wmh::DpScoring &sc, std::vector<wmh::DpRes> &res) override
	{
		const wm_host_idx *I = sc.splice ? intervals_of(cpu->hidx) : 0;
		if (!I) { SpliceDp::run_dp(jobs, wins, sc, res); return; }
		const int n = (int)jobs.size();
		res.assign(n, wmh::DpRes()); cigs.assign(n, {});
		g_n_exts2 += n;
		#pragma omp parallel for schedule(dynamic, 8)
		for (int i = 0; i < n; ++i) {
			const wmh::DpJob &J = jobs[i];
			std::vector<uint8_t> q, t, jn;
			cpu->fetch(J.q, wins[J.task], q); cpu->fetch(J.t, wins[J.task], t);
			if (J.t.kind == wmh::SEQ_REF) { // src/align.c:688-794: the target window of this DP, reversed with it
				const int64_t o = I->junc_off[J.t.rid], n_iv = I->junc_off[J.t.rid + 1] - o;
				jn.resize(J.t.len + 1);
				(J.t.reversed ? wmo_bed_junc_rev : wmo_bed_junc)((const wmo_intv1_t*)I->junc_iv.data() + o, (int)n_iv, (int32_t)J.t.off,
				                                                (int32_t)(J.t.off + J.t.len), jn.data());
			}
			wmo_ez_t ez;
			cigs[i].resize(J.q.len + J.t.len + 2);
			wmo_ksw_exts2(J.q.len, q.data(), J.t.len, t.data(), sc.mat, sc.q, sc.e, sc.q2, sc.noncan, J.zdrop, sc.junc_bonus, J.flag & 0xffff,
			              jn.empty() ? 0 : jn.data(), &ez, cigs[i].data(), (int)cigs[i].size());
			wmh::DpRes &r = res[i];
			r.max = ez.max, r.zdropped = ez.zdropped, r.max_q = ez.max_q, r.max_t = ez.max_t, r.mqe = ez.mqe, r.mqe_t = ez.mqe_t, r.mte = ez.mte, r.mte_q = ez.mte_q;
			r.score = ez.score, r.reach_end = ez.reach_end, r.n_cigar = ez.n_cigar, r.cigar = cigs[i].data();
		}
	}
};

// map_batch_aln of splice_aln_backend.cpp with JuncDp in place of SpliceDp
void map_batch_junc(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                    std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, wmh::MapStats *stats)
{
	JuncDp d;
	d.cpu = static_cast<CpuBackend*>(be);
#if defined(WMT_SPLICE_HPC)
	CdnaFromParams w;
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
const bool g_junc_mapping = (g_map_batch = map_batch_junc, true);
} // namespace

// wmt_map_file_splice_aln (its arguments first) with the junction intervals of the BED bed_fn (null: none) on every index part
extern "C" int wmt_map_file_junc_aln(const char *ref_fn, const char *kmer_fn, const char *preset, int splice, int max_intron_len, int sam,
                                     int64_t set_flags, int64_t clear_flags, int noncan, int64_t max_sw_mat, const char *reads_fn,
                                     const char *out_fn, int n_threads, uint64_t part_bases, int split, const char *bed_fn)
{
	g_bed = bed_fn ? bed_fn : "";
	g_iv.clear();
	const int rc = wmt_map_file_splice_aln(ref_fn, kmer_fn, preset, splice, max_intron_len, sam, set_flags, clear_flags, noncan, max_sw_mat,
	                                       reads_fn, out_fn, n_threads, part_bases, split);
	g_bed.clear();
	g_iv.clear();
	return rc;
}

// the product's BED reader (read_bed_junc) on an index with these sequence names: the raw 16-byte records of every sequence, in
// order (at most cap of them into recs), their per-sequence offsets into off[0..n]; the number of records, or -1
extern "C" int64_t wmt_bed_read(int n, const char *const *names, const char *fn, void *recs, int64_t *off, int64_t cap)
{
	wm_host_idx H;
	for (int i = 0; i < n; ++i) H.name.push_back(names[i]);
	if (wmh::read_bed_junc(&H, fn) < 0) return -1;
	const int64_t m = (int64_t)H.junc_iv.size();
	memcpy(recs, H.junc_iv.data(), sizeof(wm_idx_intv1_t) * (size_t)(m < cap ? m : cap));
	for (int i = 0; i <= n; ++i) off[i] = H.junc_off[i];
	return m;
}
