// Batch orchestration of Winnowmap's two-stage mapper (reference src/map.c:279-974, mm_map_frag with one
// segment), re-organised for the GPU: instead of one thread running a read from start to end, the whole
// batch advances in waves.  A wave is the set of mini-mappings that are runnable now: for stage 1 one window
// (read, start point, level, direction) per start point (levels of one start point are sequential, because
// each level is only tried if the previous one failed, src/map.c:343,513,685), for stage 2 one whole-read
// mapping per read.  Inside a wave the GPU does sketch/seed/sort/chain, then the DP jobs of all hits in
// rounds; the small, branchy, libm-dependent glue runs on host threads.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <tuple>
#include "host_backend.h"
#include "host_glue.h"
#include "host_sort.h"
#include "host_timers.h"

namespace wmh {

Timers g_timers;

static inline uint32_t x31_hash(const char *s)
{ // __ac_X31_hash_string (src/khash.h:383-388)
	uint32_t h = (uint32_t)*s;
	if (h) for (++s; *s; ++s) h = (h << 5) - h + (uint32_t)*s;
	return h;
}
static inline uint32_t wang_hash(uint32_t key)
{ // __ac_Wang_hash (src/khash.h:400-409)
	key += ~(key << 15); key ^= (key >> 10); key += (key << 3);
	key ^= (key >> 6); key += ~(key << 11); key ^= (key >> 16);
	return key;
}

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

namespace {

struct MiniMap { // one sketch -> seed -> chain -> align -> mapq instance
	MapWin win;
	const wm_mapopt_t *opt;
	int chain_set;
	bool est_err;
	uint32_t hash;
	int rep_len;
	int max_chain_gap_ref;
	std::vector<wm_pair_t> a;
	std::vector<uint64_t> u;
	std::vector<uint64_t> mini_pos;
	std::vector<wm_reg1_t> regs;
	AlignTask at;
	bool aligning;
	JobSink sink;
	size_t base_dp, base_ll;
};

struct Cursor { // one start point of stage 1 (the body of the loop at src/map.c:334)
	int read, suffix_id, sub_begin;
	std::vector<std::pair<int, int>> steps; // (sub_len, dir) in the order the reference tries them; dir 0 = right, 1 = left
	size_t step;
	bool done;
};

struct ReadState {
	int qlen;
	bool stage1;
	std::vector<std::vector<wm_pair_t>> collect_a; // per start point (src/map.c:486-496)
	std::vector<uint8_t> mapped;                   // seqMapped (src/map.c:310)
};

// chaining parameters as computed at src/map.c:374-389 (non-SR, max_gap_ref <= 0 unless set, no max_frag_len)
void chain_gaps(const wm_mapopt_t *o, int qlen_sum, int *max_qry, int *max_ref, int *min_ref)
{
	*max_qry = o->max_gap;
	if (o->max_gap_ref > 0) *max_ref = o->max_gap_ref;
	else if (o->max_frag_len > 0) {
		*max_ref = o->max_frag_len - qlen_sum;
		if (*max_ref < o->max_gap) *max_ref = o->max_gap;
	} else *max_ref = o->max_gap;
	*min_ref = o->min_gap_ref < *max_ref ? o->min_gap_ref : *max_ref;
}

ChainParams chain_params(const wm_mapopt_t *o, const wm_mapopt_t *base, int qlen_sum)
{
	ChainParams c;
	int mq, mr, mn;
	chain_gaps(o, qlen_sum, &mq, &mr, &mn);
	c.max_dist_x = mr, c.min_dist_x = mn, c.max_dist_y = mq, c.bw = o->bw;
	c.max_skip = o->max_chain_skip, c.max_iter = o->max_chain_iter, c.min_cnt = o->min_cnt, c.min_sc = o->min_chain_score;
	c.gap_scale = base->chain_gap_scale;
	return c;
}

} // namespace

void set_name_order(wm_host_idx *mi)
{ // strcmp compares bytes as unsigned char, as std::string::compare does: equal names get equal ranks
	const uint32_t n = (uint32_t)mi->name.size();
	std::vector<uint32_t> &s = mi->name_sorted, &rank = mi->name_rank;
	s.resize(n), rank.resize(n);
	for (uint32_t i = 0; i < n; ++i) s[i] = i;
	std::stable_sort(s.begin(), s.end(), [&](uint32_t a, uint32_t b) { return strcmp(mi->name[a].c_str(), mi->name[b].c_str()) < 0; });
	for (uint32_t i = 0; i < n; ++i)
		rank[s[i]] = i > 0 && mi->name[s[i]] == mi->name[s[i - 1]] ? rank[s[i - 1]] : i;
}

uint32_t skip_bits(const wm_host_idx *mi, int64_t flag, const wm_read *rd, uint32_t *name_lt)
{ // skip_seed (src/map.c:132-154), the parts that depend on the read only
	uint32_t b = 0;
	*name_lt = 0;
	if (flag & WM_F_FOR_ONLY) b |= SKIP_FOR_ONLY;
	if (flag & WM_F_REV_ONLY) b |= SKIP_REV_ONLY;
	if (!rd->has_name || !(flag & (WM_F_NO_DIAG | WM_F_NO_DUAL))) return b;
	if (mi->name_sorted.size() != mi->name.size()) {
		fprintf(stderr, "[ERROR] winnowmap-b200: the index's name order is not set (set_name_order)\n");
		exit(1);
	}
	if (flag & WM_F_NO_DIAG) b |= SKIP_NO_DIAG;
	if (flag & WM_F_NO_DUAL) b |= SKIP_NO_DUAL;
	const char *q = rd->name.c_str();
	const std::vector<uint32_t> &s = mi->name_sorted;
	const size_t lt = std::partition_point(s.begin(), s.end(), [&](uint32_t r) { return strcmp(mi->name[r].c_str(), q) < 0; }) - s.begin();
	if (lt < s.size() && mi->name[s[lt]] == rd->name) b |= SKIP_NAME_EQ;
	*name_lt = (uint32_t)lt;
	return b;
}

void map_batch(Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
               std::vector<std::vector<wm_reg1_t>> &regs_out, std::vector<int> &rep_len_out, std::vector<int> &frag_gap_out, int n_threads, MapStats *st)
{
	const int n_reads = (int)reads.size();
	regs_out.assign(n_reads, std::vector<wm_reg1_t>());
	rep_len_out.assign(n_reads, 0);
	frag_gap_out.assign(n_reads, 0);
	if (n_reads == 0) return;
	if (n_threads < 1) n_threads = 1;
	if (opt->flag & (WM_F_SPLICE | WM_F_SR | WM_F_HEAP_SORT)) {
		fprintf(stderr, "[ERROR] winnowmap-b200: splice/sr/heap-sort modes are outside the accelerated path\n");
		exit(1);
	}
	// options the reference honours on this path that are not implemented here are refused, not silently ignored
	if (opt->max_occ > opt->mid_occ) { // re-chaining with a higher occurrence threshold (src/map.c:391-415, :563-590, :892-915)
		fprintf(stderr, "[ERROR] winnowmap-b200: max_occ > mid_occ (re-chaining of repetitive reads) is not implemented; the CLI cannot set it either (src/main.c:278)\n");
		exit(1);
	}
	if (opt->max_qlen > 0) { // stage-1 / stage-2 length cut-off (src/map.c:356, :528, :725)
		fprintf(stderr, "[ERROR] winnowmap-b200: max_qlen is not implemented\n");
		exit(1);
	}
	if (opt->mid_occ_frac >= 0.0f && opt->mid_occ_frac < 1.0f) { // -f: the C ABI resolves it per index (wm_mapopt_update) before mapping
		fprintf(stderr, "[ERROR] winnowmap-b200: mid_occ_frac (-f) reached the batch unresolved: set mid_occ from the index first (wm_mapopt_update)\n");
		exit(1);
	}
	const double t_batch0 = Timers::now();
	be->begin_batch(reads);
	g_timers.add("batch.begin_upload", Timers::now() - t_batch0);
	const double t_enc0 = Timers::now();
	// 0..4 codes of every read, both strands, once per batch: the alignment tasks of all windows of a read slice them
	std::vector<int64_t> code_off(n_reads + 1, 0);
	for (int i = 0; i < n_reads; ++i) code_off[i + 1] = code_off[i] + (int64_t)reads[i]->seq.size();
	std::vector<uint8_t> codes_fwd((size_t)code_off[n_reads] + 1), codes_rev((size_t)code_off[n_reads] + 1);
	#pragma omp parallel for schedule(dynamic, 8) num_threads(n_threads)
	for (int i = 0; i < n_reads; ++i)
		encode_strands(reads[i]->seq.data(), (int)reads[i]->seq.size(), codes_fwd.data() + code_off[i], codes_rev.data() + code_off[i]);
	g_timers.add("batch.encode_strands", Timers::now() - t_enc0);

	// the three option sets of mm_map_frag: stage 1 (src/map.c:300-302), stage 2 (:711-717), fallback (= user options, :857)
	wm_mapopt_t opt2 = *opt, opt3 = *opt;
	opt2.best_n = std::max(5, opt2.best_n);
	opt3.zdrop_inv = std::min(opt->zdrop_inv, opt->stage2_zdrop_inv);
	opt3.bw = std::max(opt->bw, opt->stage2_bw);
	opt3.max_gap = std::max(opt->max_gap, opt->stage2_max_gap);
	DpScoring sc;
	gen_simple_mat(sc.mat, (int8_t)opt->a, (int8_t)opt->b, (int8_t)opt->sc_ambi);
	sc.q = opt->q, sc.e = opt->e, sc.q2 = opt->q2, sc.e2 = opt->e2;

	std::vector<ReadState> rs(n_reads);
	std::vector<uint32_t> skip(n_reads, 0), name_lt(n_reads, 0); // the seed filter of every read (-D, --dual=no, --for-only, --rev-only)
	if (opt->flag & (WM_F_NO_DIAG | WM_F_NO_DUAL | WM_F_FOR_ONLY | WM_F_REV_ONLY)) {
		#pragma omp parallel for schedule(static) num_threads(n_threads)
		for (int i = 0; i < n_reads; ++i) skip[i] = skip_bits(mi, opt->flag, reads[i], &name_lt[i]);
	}
	std::vector<Cursor> cursors;
	std::vector<int> levels;
	for (int sub_len = opt2.minPrefixLength; sub_len <= opt2.maxPrefixLength; sub_len = (int)((float)sub_len * opt2.prefixIncrementFactor)) {
		levels.push_back(sub_len); // src/map.c:343: "sub_len *= factor" is an int <- float round trip
		if ((int)((float)sub_len * opt2.prefixIncrementFactor) <= sub_len) break; // a factor <= 1 would never terminate in the reference either
	}
	for (int i = 0; i < n_reads; ++i) {
		ReadState &R = rs[i];
		R.qlen = (int)reads[i]->seq.size();
		R.stage1 = opt2.SVaware && R.qlen >= opt2.SVawareMinReadLength && R.qlen > 0;
		if (!R.stage1) continue;
		const int off = opt2.suffixSampleOffset;
		const int n_start = 1 + (int)ceil(R.qlen * 1.0 / off); // src/map.c:304
		R.collect_a.resize(n_start);
		R.mapped.assign(R.qlen, 0);
		for (int sb = 0; sb < R.qlen + off - 1; sb += off) { // src/map.c:334-340
			Cursor c;
			c.read = i, c.suffix_id = sb / off, c.sub_begin = sb >= R.qlen ? R.qlen - 1 : sb, c.step = 0, c.done = false;
			for (int sub_len : levels) {
				if (c.sub_begin + sub_len <= R.qlen) c.steps.push_back(std::make_pair(sub_len, 0));
				if (c.sub_begin - sub_len + 1 >= 0) c.steps.push_back(std::make_pair(sub_len, 1));
			}
			if (c.steps.empty()) c.done = true;
			cursors.push_back(c);
			if (sb >= R.qlen) break;
		}
	}

	std::vector<MiniMap> mm;
	std::vector<int32_t> mask_pool;
	std::vector<wm_pair_t> pre_pool;
	std::vector<SeedTask> tasks;
	std::vector<SeedOut> sout;
	std::vector<MapWin> wins;
	std::vector<DpJob> dp_jobs; std::vector<LlJob> ll_jobs;
	std::vector<DpRes> dp_res; std::vector<LlRes> ll_res;

	// Runs every MiniMap of `mm` (tasks[] prepared by the caller) through seed/chain, glue, alignment and MAPQ.
	auto run_wave = [&](int stage) {
		const int n = (int)mm.size();
		if (n == 0) return;
		double t0 = now_s();
		ChainParams cp[2];
		// window length does not enter the chaining parameters unless max_frag_len is set (never by the CLI presets)
		cp[0] = chain_params(stage == 1 ? &opt2 : opt, opt, 0);
		cp[1] = chain_params(&opt3, opt, 0);
		{ WM_TIMED("wave.seed_chain"); be->seed_chain(tasks, mask_pool.data(), pre_pool.data(), cp, opt->mid_occ, sout); }
		double t1 = now_s();
		if (st) st->t_seed += t1 - t0, st->n_minimaps += n;
		wins.resize(n);
		double tg0 = Timers::now();
		#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads)
		for (int i = 0; i < n; ++i) {
			MiniMap &M = mm[i];
			const SeedOut &o = sout[i];
			const wm_read *rd = reads[M.win.read];
			wins[i] = M.win;
			M.rep_len = o.rep_len;
			static const bool sub_t = getenv("WM_SUBTIMING") != 0;
			double q0 = sub_t ? Timers::now() : 0;
			M.a.assign(o.b, o.b + o.n_b);
			M.u.assign(o.u, o.u + o.n_u);
			M.mini_pos.clear();
			if (M.est_err)
				for (int k = 0; k < o.n_mz; ++k)
					if (o.mz_pos[k] >> 31) M.mini_pos.push_back((uint64_t)(o.mz_span ? o.mz_span[k] : mi->k) << 32 | (o.mz_pos[k] & 0x7fffffffu));
			M.hash = rd->name.empty() ? 0 : x31_hash(rd->name.c_str()); // src/map.c:358-360
			M.hash ^= wang_hash((uint32_t)M.win.wl) + wang_hash((uint32_t)M.opt->seed);
			M.hash = wang_hash(M.hash);
			if (sub_t) { double q1 = Timers::now(); g_timers.add("glue.copy", q1 - q0); q0 = q1; }
			gen_regs(M.hash, M.win.wl, (int)M.u.size(), M.u.data(), M.a.data(), M.regs);
			if (sub_t) { double q1 = Timers::now(); g_timers.add("glue.gen_regs", q1 - q0); q0 = q1; }
			chain_post(M.opt, mi->k, M.win.wl, M.regs, M.a.data());
			if (sub_t) { double q1 = Timers::now(); g_timers.add("glue.chain_post", q1 - q0); q0 = q1; }
			if (M.est_err) est_err(mi, M.win.wl, M.regs, M.a.data(), (int32_t)M.mini_pos.size(), M.mini_pos.data());
			if (sub_t) { double q1 = Timers::now(); g_timers.add("glue.est_err", q1 - q0); q0 = q1; }
			M.aligning = (M.opt->flag & WM_F_CIGAR) != 0;
			if (M.aligning) {
				const int64_t L = (int64_t)rd->seq.size(), o = code_off[M.win.read];
				// strand 1 of the window [wb, wb+wl) is a slice of strand 1 of the read
				M.at.init(M.opt, mi, i, M.win.wl, rd->seq.data() + M.win.wb, M.regs, M.a.data(),
				          codes_fwd.data() + o + M.win.wb, codes_rev.data() + o + (L - M.win.wb - M.win.wl));
			}
			M.sink.dp.clear(), M.sink.ll.clear();
			if (sub_t) { double q1 = Timers::now(); g_timers.add("glue.at_init", q1 - q0); q0 = q1; }
		}
		g_timers.add("wave.glue_pre_align", Timers::now() - tg0);
		if (st) for (int i = 0; i < n; ++i) st->n_chained += (int64_t)mm[i].a.size();
		// alignment rounds (align_regs, src/map.c:267-277 -> mm_align_skeleton)
		std::vector<int> active;
		for (int i = 0; i < n; ++i) if (mm[i].aligning) active.push_back(i);
		dp_res.clear(), ll_res.clear();
		double t_dp_wave = 0;
		while (!active.empty()) {
			double ta0 = Timers::now();
			#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads)
			for (size_t k = 0; k < active.size(); ++k) {
				MiniMap &M = mm[active[k]];
				const DpRes *dpp = dp_res.empty() ? 0 : dp_res.data() + M.base_dp;
				const LlRes *llp = ll_res.empty() ? 0 : ll_res.data() + M.base_ll;
				M.sink.dp.clear(), M.sink.ll.clear();
				M.aligning = !M.at.advance(dpp, llp, M.sink);
			}
			g_timers.add("round.advance", Timers::now() - ta0);
			double tm0 = Timers::now();
			std::vector<int> next;
			size_t n_dp = 0, n_ll = 0;
			for (int i : active) {
				MiniMap &M = mm[i];
				if (!M.aligning) { M.regs.swap(M.at.regs); continue; }
				M.base_dp = n_dp, M.base_ll = n_ll;
				n_dp += M.sink.dp.size(), n_ll += M.sink.ll.size();
				next.push_back(i);
			}
			dp_jobs.resize(n_dp), ll_jobs.resize(n_ll);
			#pragma omp parallel for schedule(static) num_threads(n_threads)
			for (size_t k = 0; k < next.size(); ++k) {
				const MiniMap &M = mm[next[k]];
				std::copy(M.sink.dp.begin(), M.sink.dp.end(), dp_jobs.begin() + M.base_dp);
				std::copy(M.sink.ll.begin(), M.sink.ll.end(), ll_jobs.begin() + M.base_ll);
			}
			active.swap(next);
			g_timers.add("round.merge_jobs", Timers::now() - tm0);
			if (active.empty()) break;
			double t2 = now_s();
			{ WM_TIMED("round.run_dp"); be->run_dp(dp_jobs, wins, sc, dp_res); }
			{ WM_TIMED("round.run_ll"); be->run_ll(ll_jobs, wins, sc, ll_res); }
			t_dp_wave += now_s() - t2;
			if (st) {
				st->t_dp += now_s() - t2, st->n_dp_jobs += (int64_t)dp_jobs.size(), st->n_ll_jobs += (int64_t)ll_jobs.size(), ++st->n_rounds;
			}
		}
		double tf0 = Timers::now();
		#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads)
		for (int i = 0; i < n; ++i) {
			MiniMap &M = mm[i];
			if (M.opt->flag & WM_F_CIGAR) { // tail of align_regs (src/map.c:271-275)
				if (!(M.opt->flag & WM_F_ALL_CHAINS)) {
					set_parent(M.opt->mask_level, M.opt->mask_len, (int)M.regs.size(), M.regs.data(), M.opt->a * 2 + M.opt->b, (int)(M.opt->flag & WM_F_HARD_MLEVEL), M.opt->alt_drop);
					select_sub(M.opt->pri_ratio, mi->k * 2, M.opt->best_n, M.regs);
					set_sam_pri((int)M.regs.size(), M.regs.data());
				}
			}
			set_mapq(M.regs, M.opt->min_chain_score, M.opt->a, M.rep_len, 0);
		}
		g_timers.add("wave.final_mapq", Timers::now() - tf0);
		if (st) st->t_host += now_s() - t1 - t_dp_wave; // the host's own share: the DP rounds are counted in t_dp
	};

	// ---------------- stage 1: minimal confidently-alignable substrings (src/map.c:314-700) ----------------
	for (;;) {
		double tb0 = Timers::now();
		tasks.clear(), mask_pool.clear(), pre_pool.clear();
		std::vector<int> cur_ids;
		for (size_t c = 0; c < cursors.size(); ++c) if (!cursors[c].done) cur_ids.push_back((int)c);
		{ // (re)build the wave's mini-mappings in parallel: they own many small vectors
			const int n_new = (int)cur_ids.size();
			mm.resize(n_new); // objects are reused wave after wave: their vectors keep their capacity (no malloc/free churn)
			tasks.resize(n_new);
			#pragma omp parallel for schedule(static) num_threads(n_threads)
			for (int k = 0; k < n_new; ++k) {
				const Cursor &C = cursors[cur_ids[k]];
				const int sub_len = C.steps[C.step].first, dir = C.steps[C.step].second;
				MiniMap &M = mm[k];
				M.win.read = C.read, M.win.wl = sub_len, M.win.wb = dir == 0 ? C.sub_begin : C.sub_begin - sub_len + 1;
				M.opt = &opt2, M.chain_set = 0, M.est_err = true;
				SeedTask t;
				t.win = M.win, t.flags = 0, t.chain_set = 0, t.n_mask = 0, t.mask_off = 0, t.n_pre = 0, t.pre_off = 0;
				t.skip = skip[C.read], t.name_lt = name_lt[C.read];
				tasks[k] = t;
			}
		}
		g_timers.add("stage1.build_wave", Timers::now() - tb0);
		if (mm.empty()) break;
		run_wave(1);
		double tk0 = Timers::now();
		#pragma omp parallel for schedule(dynamic, 32) num_threads(n_threads)
		for (int k = 0; k < (int)mm.size(); ++k) { // acceptance test and bookkeeping (src/map.c:440-515, :612-687)
			MiniMap &M = mm[k];
			Cursor &C = cursors[cur_ids[k]];
			ReadState &R = rs[C.read];
			const int sub_len = C.steps[C.step].first, dir = C.steps[C.step].second;
			const int n_regs0 = (int)M.regs.size();
			int found = -1;
			for (int j = 0; j < n_regs0; ++j)
				if ((int)M.regs[j].mapq >= opt2.min_mapq && M.regs[j].blen >= opt2.min_qcov * sub_len && M.regs[j].cnt > 0) { found = j; break; }
			if (found >= 0) {
				const wm_reg1_t &r = M.regs[found];
				std::vector<wm_pair_t> &dst = R.collect_a[C.suffix_id];
				dst.resize(r.cnt);
				for (int i = 0; i < r.cnt; ++i) {
					wm_pair_t p = M.a[i + r.as];
					if (dir == 0) { // src/map.c:491-494
						if (p.x >> 63) p.y += (uint64_t)(R.qlen - C.sub_begin - sub_len);
						else p.y += (uint64_t)C.sub_begin;
					} else { // src/map.c:663-666
						if (p.x >> 63) p.y += (uint64_t)((R.qlen - 1) - C.sub_begin);
						else p.y += (uint64_t)(C.sub_begin - sub_len + 1);
					}
					dst[i] = p;
				}
				for (int i = M.win.wb; i < M.win.wb + M.win.wl; ++i) R.mapped[i] = 1;
			}
			for (auto &r : M.regs) free(r.p);
			M.regs.clear();
			if (found >= 0 || !n_regs0) C.done = true;
			else if (++C.step >= C.steps.size()) C.done = true;
		}
		g_timers.add("stage1.bookkeeping", Timers::now() - tk0);
	}

	// ---------------- stage 2: re-map with the selected anchors (src/map.c:709-954) ----------------
	tasks.clear(), mask_pool.clear(), pre_pool.clear();
	size_t n_mm2 = 0; // stage 2 reuses the mini-mapping objects of stage 1
	std::vector<int> mm_read;
	double ts0 = Timers::now();
	std::vector<std::vector<wm_pair_t>> stage2_a(n_reads);
	#pragma omp parallel for schedule(dynamic, 8) num_threads(n_threads)
	for (int i = 0; i < n_reads; ++i) { // gather, de-duplicate and sort the stage-1 anchors of every read (src/map.c:742-774)
		ReadState &R = rs[i];
		std::vector<wm_pair_t> &a = stage2_a[i];
		if (!R.stage1) continue;
		for (auto &v : R.collect_a) a.insert(a.end(), v.begin(), v.end());
		if (!a.empty()) { // src/map.c:752-773
			std::sort(a.begin(), a.end(), [](const wm_pair_t &p, const wm_pair_t &q) { return std::tie(p.x, p.y) < std::tie(q.x, q.y); });
			a.erase(std::unique(a.begin(), a.end(), [](const wm_pair_t &p, const wm_pair_t &q) { return p.x == q.x && p.y == q.y; }), a.end());
			radix_sort(a.data(), a.data() + a.size());
			if ((int64_t)a.size() < opt3.min_cnt) a.clear();
		}
	}
	for (int i = 0; i < n_reads; ++i) {
		ReadState &R = rs[i];
		if (R.qlen == 0) continue; // src/map.c:724
		if (opt3.max_qlen > 0 && R.qlen > opt3.max_qlen) continue;
		std::vector<wm_pair_t> &a = stage2_a[i];
		if (n_mm2 >= mm.size()) mm.emplace_back();
		MiniMap &M = mm[n_mm2++];
		M.win.read = i, M.win.wb = 0, M.win.wl = R.qlen;
		M.est_err = false;
		SeedTask t;
		t.win = M.win, t.n_mask = 0, t.mask_off = 0, t.n_pre = 0, t.pre_off = 0;
		t.skip = skip[i], t.name_lt = name_lt[i];
		if (!a.empty()) {
			int unmapped = 0;
			for (int k = 0; k < R.qlen; ++k) unmapped += R.mapped[k] == 0;
			M.opt = &opt3, M.chain_set = 1;
			t.chain_set = 1;
			t.n_pre = (int32_t)a.size(), t.pre_off = (int64_t)pre_pool.size();
			pre_pool.insert(pre_pool.end(), a.begin(), a.end());
			if (unmapped > 0) { // src/map.c:786-846: seed the uncovered bases too
				t.flags = SEED_MASKED;
				t.mask_off = (int64_t)mask_pool.size() / 2;
				for (int k = 0; k < R.qlen;) {
					if (!R.mapped[k]) { ++k; continue; }
					int e = k;
					while (e < R.qlen && R.mapped[e]) ++e;
					mask_pool.push_back(k), mask_pool.push_back(e);
					++t.n_mask;
					k = e;
				}
			} else t.flags = SEED_NO_SKETCH;
		} else { // src/map.c:849-865: the default route with the user's own options
			M.opt = opt, M.chain_set = 0;
			t.chain_set = 0, t.flags = 0;
		}
		tasks.push_back(t);
		mm_read.push_back(i);
	}
	mm.resize(n_mm2);
	g_timers.add("stage2.prep", Timers::now() - ts0);
	run_wave(2);
	for (size_t k = 0; k < mm.size(); ++k) {
		MiniMap &M = mm[k];
		const int i = mm_read[k];
		regs_out[i].swap(M.regs);
		// rep_len: the (patched) reference leaves it 0 unless stage 2 sketched something (src/map.c:281,810,859,917)
		rep_len_out[i] = (tasks[k].flags & SEED_NO_SKETCH) ? 0 : M.rep_len;
		int mq, mr, mn;
		chain_gaps(M.opt, M.win.wl, &mq, &mr, &mn);
		frag_gap_out[i] = mr; // src/map.c:916
	}
	if (st) {
		st->n_reads += n_reads;
		for (int i = 0; i < n_reads; ++i) st->n_bases += rs[i].qlen;
	}
	be->end_batch();
}

} // namespace wmh
