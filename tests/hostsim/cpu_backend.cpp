// TEST INFRASTRUCTURE ONLY (lives under tests/, never shipped): a Backend whose three device operations are
// served by the CPU oracle (oracle/wm_oracle.c).  Linked with the product's *host* sources it lets the CPU-only
// test-suite drive the whole orchestration (host_driver / host_map / host_align / host_glue / host_format) end to end
// and compare the PAF with the reference goldens -- the product library itself never contains or loads this.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../winnowmap_b200/csrc/host_backend.h"
#include "../../winnowmap_b200/csrc/host_driver.h"
#include "../../winnowmap_b200/csrc/host_index.h"
#include "../../winnowmap_b200/csrc/host_io.h"

extern "C" {
// oracle/wm_oracle.c
typedef struct wmo_bloom_s wmo_bloom_t;
typedef struct wmo_idx_s wmo_idx_t;
void *wmo_bloom_init(uint64_t n_kmers);
void wmo_bloom_insert(void *b, uint64_t key);
void wmo_bloom_free(void *b);
long wmo_sketch(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
void *wmo_idx_build(const uint64_t *mz_xy, long n);
void wmo_idx_free(void *ix);
long wmo_collect_seed_hits(const void *ix, int max_occ, const uint64_t *mv_xy, long n_mv, int qlen, uint64_t *a_xy, long max_a, int *rep_len_, uint64_t *mini_pos, int *n_mini_pos_);
void wmo_radix_sort_128x(void *beg, long n);
int wmo_chain_dp(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc, float gap_scale, long n,
                 uint64_t *a_xy, uint64_t *u_out, uint64_t *b_xy, long *n_b);
typedef struct { int max, zdropped, max_q, max_t, mqe, mqe_t, mte, mte_q, score, reach_end, n_cigar; } wmo_ez_t;
int wmo_ksw_extd2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, const int8_t *mat, int q, int e, int q2, int e2, int w, int zdrop,
                  int end_bonus, int flag, wmo_ez_t *ez, uint32_t *cigar_out, int max_cigar);
int wmo_ksw_extz2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, const int8_t *mat, int q, int e, int w, int zdrop,
                  int end_bonus, int flag, wmo_ez_t *ez, uint32_t *cigar_out, int max_cigar);
int wmo_ksw_ll(int qlen, const uint8_t *query, int tlen, const uint8_t *target, const int8_t *mat, int gapo, int gape, int *qe_, int *te_);
}

using namespace wmh;

static inline uint8_t code_of(char c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': case 'U': case 'u': return 3; default: return 4; }
}

class CpuBackend : public Backend {
public:
	const wm_host_idx *hidx; void *bloom; void *idx;
	std::vector<const wm_read*> reads;
	// result storage
	std::vector<std::vector<uint32_t>> mz_pos; std::vector<std::vector<uint64_t>> us; std::vector<std::vector<wm_pair_t>> bs;
	std::vector<std::vector<uint32_t>> cigs;
	std::vector<int64_t> n_anchors; // per task of the last seed_chain call: the anchors it chained (stage-1 and seeds)
	void begin_batch(const std::vector<const wm_read*> &r) override { reads = r; }
	void end_batch() override {}

	void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) override
	{
		const int n = (int)tasks.size();
		out.assign(n, SeedOut());
		mz_pos.assign(n, {}); us.assign(n, {}); bs.assign(n, {}); n_anchors.assign(n, 0);
		#pragma omp parallel for schedule(dynamic, 4)
		for (int i = 0; i < n; ++i) {
			const SeedTask &t = tasks[i];
			std::vector<wm_pair_t> a;
			int rep_len = 0;
			if (!(t.flags & SEED_NO_SKETCH)) {
				std::string s(reads[t.win.read]->seq.data() + t.win.wb, t.win.wl);
				if (t.flags & SEED_MASKED)
					for (int m = 0; m < t.n_mask; ++m)
						for (int p = mask_pool[2 * (t.mask_off + m)]; p < mask_pool[2 * (t.mask_off + m) + 1]; ++p) s[p] = 'N';
				std::vector<uint64_t> mv((size_t)2 * (s.size() / 2 + 64));
				long nm = wmo_sketch(s.data(), (int)s.size(), hidx->w, hidx->k, 0, bloom, mv.data(), (long)mv.size() / 2);
				long cap = 1 << 14, na;
				std::vector<uint64_t> mp(nm + 1);
				int nmp = 0;
				for (;;) {
					a.resize(cap);
					na = wmo_collect_seed_hits(idx, max_occ, mv.data(), nm, t.win.wl, (uint64_t*)a.data(), cap, &rep_len, mp.data(), &nmp);
					if (na <= cap) break;
					cap = na;
				}
				a.resize(na);
				// per-minimizer "position | kept << 31" in sketch order, as the GPU backend reports it
				mz_pos[i].resize(nm);
				{
					int kk = 0;
					for (long m = 0; m < nm; ++m) {
						uint32_t pos = (uint32_t)mv[2 * m + 1] >> 1;
						bool kept = kk < nmp && (uint32_t)mp[kk] == pos;
						if (kept) ++kk;
						mz_pos[i][m] = pos | (kept ? 0x80000000u : 0);
					}
				}
			}
			if (t.n_pre > 0) { // [pre ; seeds] then the unstable sort again (src/map.c:818-831)
				std::vector<wm_pair_t> w(pre_pool + t.pre_off, pre_pool + t.pre_off + t.n_pre);
				w.insert(w.end(), a.begin(), a.end());
				if (!a.empty()) wmo_radix_sort_128x(w.data(), (long)w.size());
				a.swap(w);
			}
			n_anchors[i] = (int64_t)a.size();
			const ChainParams &c = cp[t.chain_set];
			us[i].resize(a.size() + 1); bs[i].resize(a.size() + 1);
			long nb = 0;
			int nu = wmo_chain_dp(c.max_dist_x, c.min_dist_x, c.max_dist_y, c.bw, c.max_skip, c.max_iter, c.min_cnt, c.min_sc, c.gap_scale, (long)a.size(),
			                      (uint64_t*)a.data(), us[i].data(), (uint64_t*)bs[i].data(), &nb);
			SeedOut &o = out[i];
			o.rep_len = (t.flags & SEED_NO_SKETCH) ? 0 : rep_len;
			o.n_mz = (int32_t)mz_pos[i].size(); o.mz_pos = mz_pos[i].data();
			o.n_u = nu; o.u = us[i].data(); o.n_b = nb; o.b = bs[i].data();
		}
	}

	void fetch(const SeqRef &s, const MapWin &w, std::vector<uint8_t> &out) const
	{
		out.resize(s.len);
		if (s.kind == SEQ_REF) hidx->getseq(s.rid, (uint32_t)s.off, (uint32_t)(s.off + s.len), out.data());
		else {
			const std::string &rd = reads[w.read]->seq;
			for (int i = 0; i < s.len; ++i) {
				if (s.kind == SEQ_Q0) out[i] = code_of(rd[w.wb + s.off + i]);
				else { uint8_t c = code_of(rd[w.wb + w.wl - 1 - (s.off + i)]); out[i] = c < 4 ? 3 - c : 4; }
			}
		}
		if (s.reversed) std::reverse(out.begin(), out.end());
	}

	void run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res) override
	{
		const int n = (int)jobs.size();
		res.assign(n, DpRes()); cigs.assign(n, {});
		#pragma omp parallel for schedule(dynamic, 8)
		for (int i = 0; i < n; ++i) {
			const DpJob &J = jobs[i];
			std::vector<uint8_t> q, t;
			fetch(J.q, wins[J.task], q); fetch(J.t, wins[J.task], t);
			wmo_ez_t ez;
			cigs[i].resize(J.q.len + J.t.len + 2);
			if (sc.q == sc.q2 && sc.e == sc.e2) // src/align.c:328-331
				wmo_ksw_extz2(J.q.len, q.data(), J.t.len, t.data(), sc.mat, sc.q, sc.e, J.w, J.zdrop, J.end_bonus, J.flag, &ez, cigs[i].data(), (int)cigs[i].size());
			else
				wmo_ksw_extd2(J.q.len, q.data(), J.t.len, t.data(), sc.mat, sc.q, sc.e, sc.q2, sc.e2, J.w, J.zdrop, J.end_bonus, J.flag, &ez, cigs[i].data(), (int)cigs[i].size());
			DpRes &r = res[i];
			r.max = ez.max, r.zdropped = ez.zdropped, r.max_q = ez.max_q, r.max_t = ez.max_t, r.mqe = ez.mqe, r.mqe_t = ez.mqe_t, r.mte = ez.mte, r.mte_q = ez.mte_q;
			r.score = ez.score, r.reach_end = ez.reach_end, r.n_cigar = ez.n_cigar, r.cigar = cigs[i].data();
		}
	}

	void run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res) override
	{
		const int n = (int)jobs.size();
		res.assign(n, LlRes());
		for (int i = 0; i < n; ++i) {
			std::vector<uint8_t> q, t;
			fetch(jobs[i].q, wins[jobs[i].task], q); fetch(jobs[i].t, wins[jobs[i].task], t);
			res[i].score = wmo_ksw_ll((int)q.size(), q.data(), (int)t.size(), t.data(), sc.mat, sc.q, sc.e, &res[i].qe, &res[i].te);
		}
	}
};

// -A / -B / --score-N / -O / -E of the next run; a negative entry keeps the preset's value
static int g_scoring_override[7] = {-1, -1, -1, -1, -1, -1, -1};
extern "C" void wmt_set_scoring(int a, int b, int sc_ambi, int q, int e, int q2, int e2)
{
	const int v[7] = {a, b, sc_ambi, q, e, q2, e2};
	memcpy(g_scoring_override, v, sizeof(v));
}
extern "C" void wmt_set_gap(int q, int e, int q2, int e2) { wmt_set_scoring(-1, -1, -1, q > 0 ? q : -1, e > 0 ? e : -1, q2 > 0 ? q2 : -1, e2 > 0 ? e2 : -1); }

// the options of one run: preset, -c or -a, extra output flags and the one-shot scoring override
static int run_opts(const char *preset, int sam, int64_t extra_flags, wm_idxopt_t &io, wm_mapopt_t &mo)
{
	set_opt(0, &io, &mo);
	if (preset && set_opt(preset, &io, &mo) < 0) return -1;
	if (sam) mo.flag |= WM_F_OUT_SAM | WM_F_CIGAR; // -a (src/main.c)
	else mo.flag |= WM_F_OUT_CG | WM_F_CIGAR;      // -c
	mo.flag |= extra_flags;                        // --cs / --cs=long / --MD (src/main.c:227,249-266)
	int *const field[7] = {&mo.a, &mo.b, &mo.sc_ambi, &mo.q, &mo.e, &mo.q2, &mo.e2}; // src/main.c: -A, -B, --score-N, -O, -E
	for (int i = 0; i < 7; ++i) if (g_scoring_override[i] >= 0) *field[i] = g_scoring_override[i];
	for (int i = 0; i < 7; ++i) g_scoring_override[i] = -1; // one shot
	return check_opt(&io, &mo) < 0 ? -2 : 0;
}

// The host index of a reference: names, lengths, 4-bit packed bases, the down-weight filter of the k-mer list and the
// oracle's minimizers of every sequence (in position order, as wmo_sketch emits them).
struct OracleIndex {
	wm_host_idx H;
	std::vector<uint64_t> kmers; // the -W list, canonical k-mers
	std::vector<uint64_t> mz;    // x, y pairs
	void *bloom = 0;
	~OracleIndex() { if (bloom) wmo_bloom_free(bloom); }
};

// the -W list of kmer_fn and its down-weight filter
static int load_kmer_filter(const char *kmer_fn, int k, OracleIndex &X)
{
	if (read_kmer_list(kmer_fn, k, X.kmers) < 0) return -3;
	X.bloom = wmo_bloom_init(X.kmers.size());
	for (uint64_t km : X.kmers) wmo_bloom_insert(X.bloom, km);
	return 0;
}

// The sequences of index part `part` of ref_fn, cut as mm_idx_gen cuts it (PartCutter; the defaults give one part), sketched
// with the filter `bloom`: the number of parts of the file, or < 0 when it cannot be read
static int load_oracle_seqs(const char *ref_fn, int k, int w, const void *bloom, OracleIndex &X, uint64_t part_bases = UINT64_MAX,
                            int mini_batch_size = 0, int part = 0)
{
	wm_host_idx &H = X.H;
	H.k = k, H.w = w;
	SeqReader rd;
	if (!rd.open(ref_fn)) return -4;
	PartCutter cut(part_bases, mini_batch_size);
	int n_parts = 0;
	wm_read r; uint64_t sum_len = 0;
	while (rd.next(r)) {
		n_parts = cut.next(r.seq.size()) + 1;
		if (n_parts - 1 != part) continue;
		const uint32_t rid = (uint32_t)H.name.size();
		H.name.push_back(r.name); H.len.push_back((uint32_t)r.seq.size()); H.offset.push_back(sum_len);
		H.S.resize((sum_len + r.seq.size() + 7) / 8, 0);
		pack_seq4(H.S.data(), sum_len, r.seq.data(), r.seq.size());
		sum_len += r.seq.size();
		if (r.seq.empty()) continue;
		std::vector<uint64_t> tmp((size_t)2 * (r.seq.size() / 2 + 64));
		long n = wmo_sketch(r.seq.data(), (int)r.seq.size(), w, k, rid, bloom, tmp.data(), (long)tmp.size() / 2);
		X.mz.insert(X.mz.end(), tmp.begin(), tmp.begin() + 2 * n);
	}
	set_name_order(&H);
	return n_parts;
}

static int load_oracle_index(const char *ref_fn, const char *kmer_fn, int k, int w, OracleIndex &X)
{
	int rc = load_kmer_filter(kmer_fn, k, X);
	if (rc == 0) rc = load_oracle_seqs(ref_fn, k, w, X.bloom, X);
	return rc < 0 ? rc : 0;
}

typedef void (*MapBatchFn)(Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                           std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads, MapStats *stats);
// how a batch is mapped on an oracle backend: the product's map_batch (hpc_backend.cpp maps through an HPC index instead)
static MapBatchFn g_map_batch = map_batch;

// The file driver's view (host_driver.h) of indexes served by oracle backends, one per part.  Under --cs / --MD every hit
// mapped is formatted and its tag compared with what mm_gen_cs / mm_gen_MD give (gen_cs_or_MD).
struct OracleParts : IndexParts {
	std::vector<Backend*> be; std::vector<const wm_host_idx*> H;
	wm_host_idx merged_H;           // the sequence table of all parts
	std::vector<int32_t> f_mid_occ; // per part: mid_occ of the run's -f, -1 where the selection is refused
	std::vector<int32_t> mid_occ;   // per part: the mid_occ it mapped with (-1: not mapped)
	int n_gen_mismatch = 0;
	void add(Backend *b, const wm_host_idx *h)
	{
		be.push_back(b), H.push_back(h), mid_occ.push_back(-1);
		merged_H.k = h->k, merged_H.w = h->w, merged_H.flag = h->flag;
		merged_H.name.insert(merged_H.name.end(), h->name.begin(), h->name.end());
		merged_H.len.insert(merged_H.len.end(), h->len.begin(), h->len.end());
	}
	int n_parts() const override { return (int)H.size(); }
	const wm_host_idx *part(int p) const override { return H[p]; }
	const wm_host_idx *all() const override { return H.size() == 1 ? H[0] : &merged_H; }
	bool part_opt(int p, const wm_mapopt_t *opt, wm_mapopt_t *o) override
	{
		*o = *opt;
		if (opt->mid_occ_frac >= 0 && opt->mid_occ_frac < 1) { // -f: what mm_mapopt_update sets per part
			if (p >= (int)f_mid_occ.size() || f_mid_occ[p] < 0) return false;
			o->mid_occ = std::max(f_mid_occ[p], opt->min_mid_occ), o->mid_occ_frac = -1.0f;
		}
		mid_occ[p] = o->mid_occ;
		return true;
	}
	void map(int p, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
	         std::vector<int> &rl, int n_threads) override
	{
		std::vector<int> fg;
		g_map_batch(be[p], H[p], opt, reads, regs, rl, fg, n_threads, 0);
		if (!(opt->flag & (WM_F_OUT_CS | WM_F_OUT_MD))) return;
		const bool md = (opt->flag & WM_F_OUT_MD) != 0;
		std::string line, g;
		for (size_t i = 0; i < reads.size(); ++i)
			for (size_t j = 0; j < regs[i].size(); ++j) {
				if (!regs[i][j].p) continue;
				if (opt->flag & WM_F_OUT_SAM) write_sam(line, H[p], reads[i], (int)j, (int)regs[i].size(), regs[i].data(), opt->flag, rl[i], "");
				else write_paf(line, H[p], reads[i], &regs[i][j], opt->flag, rl[i]);
				gen_cs_or_MD(g, H[p], &regs[i][j], reads[i]->seq.data(), md, !(opt->flag & WM_F_OUT_CS_LONG));
				const size_t at = line.find(md ? "\tMD:Z:" : "\tcs:Z:");
				if (at == std::string::npos || line.compare(at + 6, g.size(), g) != 0 || (at + 6 + g.size() < line.size() && line[at + 6 + g.size()] != '\t')) ++n_gen_mismatch;
			}
	}
	// the whole read file in one batch (the golden inputs are far below the mini-batch of mapopt_init), rank 0 of 1
	int run(const wm_mapopt_t &mo, const char *reads_fn, const char *out_fn, int n_threads)
	{
		const int rc = map_file(*this, &mo, reads_fn, out_fn, "", n_threads, 0, 1, 0, INT64_MAX);
		return n_gen_mismatch ? -100 - n_gen_mismatch : rc;
	}
};

// Maps every read of `reads_fn` through `be` with the product's file driver and writes PAF or SAM to `out_fn`
static int map_file_on(Backend *be, const wm_host_idx &H, const wm_mapopt_t &mo, const char *reads_fn, const char *out_fn, int n_threads)
{
	OracleParts ix;
	ix.add(be, &H);
	return ix.run(mo, reads_fn, out_fn, n_threads);
}

static int map_file_impl(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads, int sam, int64_t extra_flags = 0)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	int rc = run_opts(preset, sam, extra_flags, io, mo);
	if (rc < 0) return rc;
	OracleIndex X;
	if ((rc = load_oracle_index(ref_fn, kmer_fn, io.k, io.w, X)) < 0) return rc;
	CpuBackend be;
	be.hidx = &X.H; be.bloom = X.bloom; be.idx = wmo_idx_build(X.mz.data(), (long)X.mz.size() / 2);
	rc = map_file_on(&be, X.H, mo, reads_fn, out_fn, n_threads);
	wmo_idx_free(be.idx);
	return rc;
}

// winnowmap [-W kmers] -x preset -c ref.fa reads.fa > out.paf, host orchestration on the oracle backend
extern "C" int wmt_map_file(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads)
{
	return map_file_impl(ref_fn, kmer_fn, preset, reads_fn, out_fn, n_threads, 0);
}
// -c or -a plus extra MM_F_* output flags
extern "C" int wmt_map_file_flags(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads,
                                  int sam, int64_t extra_flags)
{
	return map_file_impl(ref_fn, kmer_fn, preset, reads_fn, out_fn, n_threads, sam, extra_flags);
}
// the same with -a: SAM
extern "C" int wmt_map_file_sam(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads)
{
	return map_file_impl(ref_fn, kmer_fn, preset, reads_fn, out_fn, n_threads, 1);
}

#include "../../winnowmap_b200/csrc/host_timers.h"
// tuning aid: the orchestration's phase timers (WM_SUBTIMING=1 adds the per-task breakdown)
extern "C" void wmt_dump_timers(void) { wmh::g_timers.dump(stderr); wmh::g_timers.reset(); }

// unit hook: the index builder's 4-bit packing of a sequence placed at base offset o0 (S: zeroed words)
extern "C" void wmt_pack_seq4(uint32_t *S, uint64_t o0, const char *seq, uint64_t L) { wmh::pack_seq4(S, o0, seq, L); }
// unit hook: the index builder's parallel (hash, position) sort on an interleaved x,y array
extern "C" void wmt_sort_index_pairs(uint64_t *xy, int64_t n, int n_threads)
{
	std::vector<wm_pair_t> a((size_t)n);
	for (int64_t i = 0; i < n; ++i) a[i].x = xy[2 * i], a[i].y = xy[2 * i + 1];
	wmh::sort_index_pairs(a, n_threads);
	for (int64_t i = 0; i < n; ++i) xy[2 * i] = a[i].x, xy[2 * i + 1] = a[i].y;
}
