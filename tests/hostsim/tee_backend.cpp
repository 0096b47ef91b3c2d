// TEST INFRASTRUCTURE ONLY: a Backend that sends every call of the mapping path (host_backend.h) to two backends and
// compares their answers field by field.  The first backend -- the product's CUDA backend, or for the comparator's own
// check an oracle backend that may change one value on purpose -- serves the caller; the second is the oracle backend of
// cpu_backend.cpp (compiled into this file unchanged), whose answers are the expected ones.  Every mismatch is recorded
// with the call, the task or job, the field and element, both values and the task's or job's description, so a
// divergence of the GPU path reads as "seed_chain call 4 task 37: u[2]" instead of a differing output line.
//
// Both backends read one index: the oracle's minimizers of the reference, flattened for the CUDA backend into sorted
// unique keys, CSR offsets and ascending positions (the order of wmo_idx_build), with the down-weight filter of
// wm_bloom_build.  With -H the oracle sketches homopolymer-compressed sequences and adds the minimizers' spans
// (span_backend.h), and the CUDA backend gets an index flagged WM_I_HPC.
//
// Built by tests/tee_lib.py against libwinnowmap_b200.so, which provides the host orchestration and the CUDA backend.
#include <stdint.h>
#include <map>
#include <string>
#include <vector>

extern "C" {
long wmo_sketch(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
}
static int g_tee_hpc = 0; // the oracle's sketch: homopolymer-compressed (-H) or plain
extern "C" long wmt_sketch_kind(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out)
{
	return g_tee_hpc ? wmo_sketch_hpc(str, len, w, k, rid, bf, out_xy, max_out) : wmo_sketch(str, len, w, k, rid, bf, out_xy, max_out);
}

#define wmo_sketch wmt_sketch_kind
#include "cpu_backend.cpp"
#undef wmo_sketch
#include "span_backend.h"
#include "../../winnowmap_b200/csrc/gpu_backend.h"

extern "C" {
wm_bloom_t *wm_bloom_build(const uint64_t *canon_kmers, int64_t n);
uint64_t wm_bloom_bits(const wm_bloom_t *b);
const uint8_t *wm_bloom_table(const wm_bloom_t *b);
void wm_bloom_destroy(wm_bloom_t *b);
}
size_t wm_extd2_bt_bytes(int qlen, int tlen, int w); // ksw_extd2.cu: the backtrack bytes of one DP job

#define EZ_SCAN_ZDROP 0x10000

// The score walk of mm_test_zdrop (src/align.c:32-70) over a CIGAR: max_zdrop and the most-dropped region {t0, t1, q0, q1}.
static int zdrop_walk(int q, int e, const int8_t *mat, const uint8_t *qs, const uint8_t *ts, int n_cigar, const uint32_t *cigar, int pos[4])
{
	int32_t score = 0, max = INT32_MIN, max_i = -1, max_j = -1, i = 0, j = 0, max_zdrop = 0;
	pos[0] = pos[1] = pos[2] = pos[3] = -1;
	auto upd = [&](int ii, int jj) {
		if (score < max) {
			const int li = ii - max_i, lj = jj - max_j, diff = li > lj ? li - lj : lj - li;
			const int z = max - score - diff * e;
			if (z > max_zdrop) max_zdrop = z, pos[0] = max_i, pos[1] = ii, pos[2] = max_j, pos[3] = jj;
		} else max = score, max_i = ii, max_j = jj;
	};
	for (int k = 0; k < n_cigar; ++k) {
		const uint32_t op = cigar[k] & 0xf, len = cigar[k] >> 4;
		if (op == 0) {
			for (uint32_t l = 0; l < len; ++l) { score += mat[ts[i + l] * 5 + qs[j + l]]; upd(i + l, j + l); }
			i += len, j += len;
		} else if (op == 1 || op == 2 || op == 3) {
			score -= q + e * (int)len;
			if (op == 1) j += len; else i += len;
			upd(i, j);
		}
	}
	return max_zdrop;
}

// The host's rule for the CTA-cooperative DP sweep (wm_dp_is_coop in wm_common.cuh), for the counters
static bool dp_is_coop(int qlen, int tlen, int w)
{
	const char *env = getenv("WM_DP_COOP_MIN_CELLS");
	const long long min_cells = env && atoll(env) > 0 ? atoll(env) : 300000;
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	const int diag = std::min(std::min(qlen, tlen), w + 1);
	return diag >= 384 && (long long)tlen * std::min(qlen, 2 * w + 1) >= min_cells;
}

static int env_int(const char *name, int dflt) { const char *e = getenv(name); return e && atoi(e) > 0 ? atoi(e) : dflt; }

class TeeBackend : public Backend {
public:
	Backend *dev = 0, *ora = 0; // served / expected
	CpuBackend *fetcher = 0;    // slices of the batch's reads and of the reference, for the Z-drop walk
	bool hpc = false;
	size_t budget = 0;          // the CUDA backend's backtrack budget: DP chunks per round are counted with it (0: not counted)
	int64_t n_mismatch = 0;
	std::vector<std::string> lines;
	std::map<std::string, int64_t> cnt;
	int64_t calls[3] = {0, 0, 0};
	std::vector<const wm_read*> reads;

	void add(const std::string &k, int64_t v = 1) { cnt[k] += v; }
	void peak(const std::string &k, int64_t v) { int64_t &c = cnt[k]; if (v > c) c = v; }
	void bad(const char *kind, int64_t call, int64_t idx, const char *field, int64_t elem, const std::string &exp, const std::string &got, const std::string &desc)
	{
		++n_mismatch;
		if (lines.size() >= 200) return;
		char b[256];
		snprintf(b, sizeof(b), "mismatch\t%s\t%lld\t%lld\t%s\t%lld\t", kind, (long long)call, (long long)idx, field, (long long)elem);
		lines.push_back(b + exp + "\t" + got + "\t" + desc);
	}
	static std::string hex(uint64_t v) { char b[32]; snprintf(b, sizeof(b), "0x%llx", (unsigned long long)v); return b; }
	static std::string dec(int64_t v) { return std::to_string(v); }
	template<class T, class F>
	void cmp_arr(const char *kind, int64_t call, int64_t idx, const char *field, const T *e, const T *g, int64_t n, F str, const std::string &desc)
	{ // the first differing element, with the number of differing ones
		int64_t first = -1, n_diff = 0;
		for (int64_t i = 0; i < n; ++i)
			if (memcmp(&e[i], &g[i], sizeof(T)) != 0) { if (first < 0) first = i; ++n_diff; }
		if (first >= 0) bad(kind, call, idx, field, first, str(e[first]), str(g[first]), desc + " (" + dec(n_diff) + " of " + dec(n) + " differ)");
	}

	void begin_batch(const std::vector<const wm_read*> &r) override { reads = r; dev->begin_batch(r); ora->begin_batch(r); }
	void end_batch() override { dev->end_batch(); ora->end_batch(); }

	void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) override
	{
		const int64_t call = calls[0]++;
		std::vector<SeedOut> eo;
		ora->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, eo);
		dev->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out);
		const int n = (int)tasks.size();
		bool set_used[2] = {false, false};
		add("seed.calls"); add("seed.tasks", n);
		// tasks of this call per worker class of the CTA kernels, as peaks over calls: above 1, some worker of a class whose
		// grid is capped at one CTA (WM_SORT_MEDIUM_CTAS / WM_SORT_GIANT_CTAS / WM_CHAIN_TILE_CTAS = 1) took a second task
		const int64_t tile_min = env_int("WM_CHAIN_TILE_MIN", 2048), bt_cta_min = env_int("WM_CHAIN_BT_CTA_MIN", 4096);
		const int64_t giant_min = env_int("WM_SORT_GIANT_MIN", 0) >= 2048 ? env_int("WM_SORT_GIANT_MIN", 0) : 1 << 30; // seed.cu
		int64_t n_tile = 0, n_bt_cta = 0, n_sort_medium[3] = {0, 0, 0}, n_sort_giant[3] = {0, 0, 0};
		for (int i = 0; i < n; ++i) { // sort launches (gpu_backend.cu seed_chain): the seeds of the plain and of the masked pass, then sort #3
			const SeedTask &t = tasks[i];
			const int64_t n_a = fetcher->n_anchors[i], n_seed = n_a - t.n_pre;
			const int64_t sz[3] = {(t.flags & (SEED_MASKED | SEED_NO_SKETCH)) ? 0 : n_seed, (t.flags & SEED_MASKED) ? n_seed : 0,
			                       t.n_pre > 0 && n_seed > 0 ? n_a : 0};
			for (int l = 0; l < 3; ++l) { n_sort_medium[l] += sz[l] > 2048 && sz[l] <= giant_min; n_sort_giant[l] += sz[l] > giant_min; }
			n_tile += n_a > tile_min; n_bt_cta += n_a > bt_cta_min;
		}
		peak("peak.chain_tile", n_tile); peak("peak.chain_bt_cta", n_bt_cta);
		for (int l = 0; l < 3; ++l) { peak("peak.sort_medium", n_sort_medium[l]); peak("peak.sort_giant", n_sort_giant[l]); }
		for (int i = 0; i < n; ++i) {
			const SeedTask &t = tasks[i];
			const SeedOut &e = eo[i], &g = out[i];
			char d[200];
			snprintf(d, sizeof(d), "read %d wb %d wl %d flags %d set %d n_mask %d n_pre %d", t.win.read, t.win.wb, t.win.wl, t.flags, t.chain_set, t.n_mask, t.n_pre);
			const std::string desc = d;
			set_used[t.chain_set & 1] = true;
			// shapes seen (anchor counts as the oracle backend chained them)
			const int64_t n_a = fetcher->n_anchors[i], n_seed = n_a - t.n_pre;
			if (t.flags & SEED_MASKED) add("seed.masked");
			if (t.flags & SEED_NO_SKETCH) add("seed.no_sketch");
			if (t.n_pre > 0) add("seed.pre");
			if (t.n_pre > 0 && n_seed > 0) add(n_a <= 64 ? "sort3.le64" : n_a <= 2048 ? "sort3.le2048" : "sort3.gt2048");
			add(n_a <= 128 ? "chain.le128" : n_a <= 2048 ? "chain.le2048" : n_a <= 4096 ? "chain.le4096" : "chain.gt4096");
			if (n_a > env_int("WM_CHAIN_TILE_MIN", 2048)) add("chain.tile_tasks");     // chain.cu: the tile kernel
			if (n_a > env_int("WM_CHAIN_BT_CTA_MIN", 4096)) add("chain.bt_cta_tasks"); // chain.cu: the CTA backtrack
			if (g.rep_len != e.rep_len) bad("seed_chain", call, i, "rep_len", -1, dec(e.rep_len), dec(g.rep_len), desc);
			if (g.n_mz != e.n_mz) bad("seed_chain", call, i, "n_mz", -1, dec(e.n_mz), dec(g.n_mz), desc);
			cmp_arr("seed_chain", call, i, "mz_pos", e.mz_pos, g.mz_pos, std::min(e.n_mz, g.n_mz), hex, desc);
			if (hpc && !(t.flags & SEED_NO_SKETCH)) {
				if (!g.mz_span || !e.mz_span) { if (std::min(e.n_mz, g.n_mz) > 0) bad("seed_chain", call, i, "mz_span", -1, e.mz_span ? "set" : "null", g.mz_span ? "set" : "null", desc); }
				else cmp_arr("seed_chain", call, i, "mz_span", e.mz_span, g.mz_span, std::min(e.n_mz, g.n_mz), [](uint8_t v) { return dec(v); }, desc);
			}
			if (g.n_u != e.n_u) bad("seed_chain", call, i, "n_u", -1, dec(e.n_u), dec(g.n_u), desc);
			cmp_arr("seed_chain", call, i, "u", e.u, g.u, std::min(e.n_u, g.n_u), hex, desc);
			if (g.n_b != e.n_b) bad("seed_chain", call, i, "n_b", -1, dec(e.n_b), dec(g.n_b), desc);
			cmp_arr("seed_chain", call, i, "b", e.b, g.b, std::min(e.n_b, g.n_b), [](const wm_pair_t &p) { return hex(p.x) + "," + hex(p.y); }, desc);
		}
		if (set_used[0] && set_used[1]) add("seed.mixed_set_calls");
	}

	void run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res) override
	{
		const int64_t call = calls[1]++;
		std::vector<DpRes> er;
		ora->run_dp(jobs, wins, sc, er);
		dev->run_dp(jobs, wins, sc, res);
		const int n = (int)jobs.size();
		const bool single = sc.q == sc.q2 && sc.e == sc.e2; // ksw_extz2 (src/align.c:328-331)
		add("dp.calls"); add("dp.jobs", n); if (single) add("dp.extz2_jobs", n);
		if (budget > 0 && n > 0) { // the chunks the CUDA backend cuts this round into (gpu_backend.cu run_dp)
			int64_t chunks = 0; size_t b = 0;
			for (int i = 0; i < n; ++i) {
				const size_t x = wm_extd2_bt_bytes(jobs[i].q.len, jobs[i].t.len, jobs[i].w);
				if (i == 0 || b + x > budget) ++chunks, b = 0;
				b += x;
			}
			peak("dp.max_chunks", chunks);
			if (chunks >= 3) add("dp.rounds_3plus_chunks");
		}
		for (int i = 0; i < n; ++i) {
			const DpJob &J = jobs[i];
			const DpRes &e = er[i], &g = res[i];
			char d[240];
			snprintf(d, sizeof(d), "task %d q %d/%lld+%d%s t %d:%d/%lld+%d%s w %d zdrop %d end_bonus %d flag 0x%x", J.task, J.q.kind, (long long)J.q.off, J.q.len, J.q.reversed ? "r" : "",
			         J.t.kind, J.t.rid, (long long)J.t.off, J.t.len, J.t.reversed ? "r" : "", J.w, J.zdrop, J.end_bonus, J.flag);
			const std::string desc = d;
			char fk[32]; snprintf(fk, sizeof(fk), "dp.flag_0x%x", J.flag); add(fk);
			if (!single && J.q.len + J.t.len >= 1600 && dp_is_coop(J.q.len, J.t.len, J.w)) add("dp.coop_jobs");
			static const char *names[11] = {"max", "zdropped", "max_q", "max_t", "mqe", "mqe_t", "mte", "mte_q", "score", "reach_end", "n_cigar"};
			const int32_t ev[11] = {e.max, e.zdropped, e.max_q, e.max_t, e.mqe, e.mqe_t, e.mte, e.mte_q, e.score, e.reach_end, e.n_cigar};
			const int32_t gv[11] = {g.max, g.zdropped, g.max_q, g.max_t, g.mqe, g.mqe_t, g.mte, g.mte_q, g.score, g.reach_end, g.n_cigar};
			for (int f = 0; f < 11; ++f)
				if (ev[f] != gv[f]) bad("run_dp", call, i, names[f], -1, dec(ev[f]), dec(gv[f]), desc);
			const int nc = std::min(e.n_cigar, g.n_cigar);
			if (nc > 0) cmp_arr("run_dp", call, i, "cigar", e.cigar, g.cigar, nc, [](uint32_t c) { return dec(c >> 4) + "MIDN"[c & 3]; }, desc);
			if (!(J.flag & EZ_SCAN_ZDROP)) continue;
			add("dp.scan_zdrop_jobs");
			// nothing aligned (an empty input, or a scoring the reference returns on before the sweep): no walk on the device,
			// host_align.cpp walks the empty CIGAR itself
			if (J.q.len <= 0 || J.t.len <= 0 || (e.n_cigar == 0 && !g.has_zd)) continue;
			if (!g.has_zd) { bad("run_dp", call, i, "has_zd", -1, "1", dec(g.has_zd), desc); continue; }
			std::vector<uint8_t> qs, ts;
			fetcher->fetch(J.q, wins[J.task], qs); fetcher->fetch(J.t, wins[J.task], ts);
			int pos[4];
			const int zmax = zdrop_walk(sc.q, sc.e, sc.mat, qs.data(), ts.data(), e.n_cigar, e.cigar, pos);
			if (g.zd_max != zmax) bad("run_dp", call, i, "zd_max", -1, dec(zmax), dec(g.zd_max), desc);
			for (int f = 0; f < 4; ++f)
				if (g.zd_pos[f] != pos[f]) bad("run_dp", call, i, "zd_pos", f, dec(pos[f]), dec(g.zd_pos[f]), desc);
		}
	}

	void run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res) override
	{
		const int64_t call = calls[2]++;
		std::vector<LlRes> er;
		ora->run_ll(jobs, wins, sc, er);
		dev->run_ll(jobs, wins, sc, res);
		add("ll.calls"); add("ll.jobs", (int64_t)jobs.size());
		for (size_t i = 0; i < jobs.size(); ++i) {
			const LlJob &J = jobs[i];
			char d[160];
			snprintf(d, sizeof(d), "task %d q %d/%lld+%d t %d:%d/%lld+%d", J.task, J.q.kind, (long long)J.q.off, J.q.len, J.t.kind, J.t.rid, (long long)J.t.off, J.t.len);
			if (res[i].score != er[i].score) bad("run_ll", call, i, "score", -1, dec(er[i].score), dec(res[i].score), d);
			if (res[i].qe != er[i].qe) bad("run_ll", call, i, "qe", -1, dec(er[i].qe), dec(res[i].qe), d);
			if (res[i].te != er[i].te) bad("run_ll", call, i, "te", -1, dec(er[i].te), dec(res[i].te), d);
		}
	}

	int write_report(const char *fn) const
	{
		FILE *f = fopen(fn, "w");
		if (!f) return -1;
		fprintf(f, "count\tmismatches\t%lld\n", (long long)n_mismatch);
		for (auto &kv : cnt) fprintf(f, "count\t%s\t%lld\n", kv.first.c_str(), (long long)kv.second);
		for (auto &l : lines) fprintf(f, "%s\n", l.c_str());
		fclose(f);
		return 0;
	}
};

// The comparator's own check: an oracle backend that imitates the CUDA backend's Z-drop walk and changes exactly one value
// of one kind (the first one it meets), and says where.
enum { MUT_NONE, MUT_REP_LEN, MUT_KEPT, MUT_U, MUT_B, MUT_CIGAR, MUT_ZD_POS, MUT_LL };

class MutantBackend : public Backend {
public:
	Backend *in = 0; CpuBackend *fetcher = 0;
	int mut = MUT_NONE; bool done = false;
	int64_t calls[3] = {0, 0, 0};
	std::string where; // "kind\tcall\tindex\tfield\telem" of the change
	void note(const char *kind, int64_t call, int64_t idx, const char *field, int64_t elem)
	{
		char b[160]; snprintf(b, sizeof(b), "%s\t%lld\t%lld\t%s\t%lld", kind, (long long)call, (long long)idx, field, (long long)elem);
		where = b; done = true;
	}
	void begin_batch(const std::vector<const wm_read*> &r) override { in->begin_batch(r); }
	void end_batch() override { in->end_batch(); }
	void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) override
	{
		const int64_t call = calls[0]++;
		in->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out);
		for (size_t i = 0; i < out.size() && !done; ++i) {
			SeedOut &o = out[i];
			if (mut == MUT_REP_LEN && !(tasks[i].flags & SEED_NO_SKETCH)) { o.rep_len += 1; note("seed_chain", call, i, "rep_len", -1); }
			else if (mut == MUT_KEPT && o.n_mz > 2) { const_cast<uint32_t*>(o.mz_pos)[2] ^= 0x80000000u; note("seed_chain", call, i, "mz_pos", 2); }
			else if (mut == MUT_U && o.n_u > 0) { const_cast<uint64_t*>(o.u)[o.n_u - 1] += 1ULL << 32; note("seed_chain", call, i, "u", o.n_u - 1); }
			else if (mut == MUT_B && o.n_b > 1) { const_cast<wm_pair_t*>(o.b)[1].y += 1; note("seed_chain", call, i, "b", 1); }
		}
	}
	void run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res) override
	{
		const int64_t call = calls[1]++;
		in->run_dp(jobs, wins, sc, res);
		for (size_t i = 0; i < jobs.size(); ++i) {
			DpRes &r = res[i];
			const DpJob &J = jobs[i];
			r.has_zd = 0;
			if ((J.flag & EZ_SCAN_ZDROP) && J.q.len > 0 && J.t.len > 0) {
				std::vector<uint8_t> qs, ts;
				fetcher->fetch(J.q, wins[J.task], qs); fetcher->fetch(J.t, wins[J.task], ts);
				r.zd_max = zdrop_walk(sc.q, sc.e, sc.mat, qs.data(), ts.data(), r.n_cigar, r.cigar, r.zd_pos);
				r.has_zd = 1;
			}
			if (done) continue;
			if (mut == MUT_CIGAR && r.n_cigar > 1) { const_cast<uint32_t*>(r.cigar)[1] ^= 1; note("run_dp", call, i, "cigar", 1); }
			else if (mut == MUT_ZD_POS && r.has_zd) { r.zd_pos[3] += 1; note("run_dp", call, i, "zd_pos", 3); }
		}
	}
	void run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res) override
	{
		const int64_t call = calls[2]++;
		in->run_ll(jobs, wins, sc, res);
		if (mut == MUT_LL && !done && !res.empty()) { res.back().te += 1; note("run_ll", call, (int64_t)res.size() - 1, "te", -1); }
	}
};

// One comparison run: the shared index, the oracle side, and the served side (dev_kind 0: the CUDA backend on device 0;
// 1: a second oracle backend; 2: a second oracle backend changed by `mutation`).
struct TeeRun {
	OracleIndex X;
	CpuBackend cpu_e, cpu_d;
	SpanBackend span_e, span_d;
	MutantBackend mutant;
	Backend *gpu = 0;
	TeeBackend tee;
	TeeRun() { cpu_e.idx = cpu_d.idx = 0; }
	~TeeRun()
	{
		if (gpu) gpu_backend_destroy(gpu);
		wmo_idx_free(cpu_e.idx);
	}
	int init(const char *ref_fn, const char *kmer_fn, int k, int w, int hpc, int dev_kind, int mutation, int64_t budget)
	{
		g_tee_hpc = hpc;
		int rc = load_oracle_index(ref_fn, kmer_fn, k, w, X);
		if (rc < 0) return rc;
		X.H.flag = hpc ? WM_I_HPC : 0;
		void *idx = wmo_idx_build(X.mz.data(), (long)X.mz.size() / 2);
		for (CpuBackend *c : {&cpu_e, &cpu_d}) c->hidx = &X.H, c->bloom = X.bloom, c->idx = idx;
		span_e.in = &cpu_e, span_d.in = &cpu_d;
		for (SpanBackend *s : {&span_e, &span_d}) s->mi = &X.H, s->bloom = X.bloom;
		tee.ora = hpc ? (Backend*)&span_e : &cpu_e;
		tee.fetcher = &cpu_e;
		tee.hpc = hpc != 0;
		if (dev_kind == 0) {
			// sorted unique keys, CSR offsets, ascending positions: the order of wmo_idx_build
			const int64_t n = (int64_t)X.mz.size() / 2;
			std::vector<std::pair<uint64_t, uint64_t>> p(n);
			for (int64_t i = 0; i < n; ++i) p[i] = std::make_pair(X.mz[2 * i] >> 8, X.mz[2 * i + 1]);
			std::sort(p.begin(), p.end());
			std::vector<uint64_t> keys, poff, pos(n);
			for (int64_t i = 0; i < n; ++i) {
				if (i == 0 || p[i].first != p[i - 1].first) keys.push_back(p[i].first), poff.push_back(i);
				pos[i] = p[i].second;
			}
			poff.push_back(n);
			wm_bloom_t *bl = wm_bloom_build(X.kmers.empty() ? 0 : X.kmers.data(), (int64_t)X.kmers.size());
			gpu = gpu_backend_create(&X.H, keys.data(), (int64_t)keys.size(), poff.data(), pos.data(), wm_bloom_bits(bl), wm_bloom_table(bl), 0);
			wm_bloom_destroy(bl);
			if (budget > 0) gpu_backend_set_budget(gpu, (size_t)budget);
			tee.dev = gpu;
			tee.budget = gpu_backend_get_budget(gpu);
		} else {
			mutant.in = hpc ? (Backend*)&span_d : &cpu_d;
			mutant.fetcher = &cpu_d;
			mutant.mut = dev_kind == 2 ? mutation : MUT_NONE;
			tee.dev = &mutant;
			tee.budget = budget > 0 ? (size_t)budget : 0;
		}
		return 0;
	}
	int finish(const char *report_fn)
	{
		if (!mutant.where.empty()) tee.lines.insert(tee.lines.begin(), "mutated\t" + mutant.where);
		return tee.write_report(report_fn);
	}
};

// winnowmap [-H] -x preset -c ref.fa reads.fa through the tee: writes the PAF of the served backend and the report
extern "C" int wmt_tee_map_file(const char *ref_fn, const char *kmer_fn, const char *preset, const char *reads_fn, const char *out_fn, int n_threads,
                                int hpc, int64_t budget, int dev_kind, int mutation, const char *report_fn)
{
	wm_idxopt_t io; wm_mapopt_t mo;
	int rc = run_opts(preset, 0, 0, io, mo);
	if (rc < 0) return rc;
	TeeRun R;
	if ((rc = R.init(ref_fn, kmer_fn, io.k, io.w, hpc, dev_kind, mutation, budget)) < 0) return rc;
	rc = map_file_on(&R.tee, R.X.H, mo, reads_fn, out_fn, n_threads);
	if (R.finish(report_fn) < 0) return -6;
	return rc;
}

// Crafted seed_chain batches, in the two shapes host_map.cpp sends.  Call 1 is a stage-1 wave: windows (rows1: read, wb,
// wl, source) on chain set 0, plain.  Call 2 is the stage-2 call over whole reads (reads2), built as host_map.cpp builds it
// (src/map.c:742-846): a read's stage-1 anchors are the top chain of every call-1 window flagged `source` that chained
// something, moved into read coordinates, de-duplicated and sorted; such a read is chained on set 1, sketched with its
// mapped windows masked, or not sketched when they cover it.  A read without stage-1 anchors takes the default route: set 0.
// cp_i: two rows of max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc; cp_f: the two gap_scale.
extern "C" int wmt_tee_seed_chain(const char *ref_fn, const char *kmer_fn, int k, int w, int hpc, int dev_kind, int mutation,
                                  int n_reads, const char *seq, const int64_t *read_off, int n1, const int32_t *rows1, int n2, const int32_t *reads2,
                                  const int32_t *cp_i, const float *cp_f, int max_occ, const char *report_fn)
{
	TeeRun R;
	int rc = R.init(ref_fn, kmer_fn, k, w, hpc, dev_kind, mutation, 0);
	if (rc < 0) return rc;
	std::vector<wm_read> rs(n_reads);
	std::vector<const wm_read*> rp(n_reads);
	for (int i = 0; i < n_reads; ++i) rs[i].name = "r" + std::to_string(i), rs[i].seq.assign(seq + read_off[i], read_off[i + 1] - read_off[i]), rp[i] = &rs[i];
	ChainParams cp[2];
	for (int s = 0; s < 2; ++s) {
		const int32_t *c = cp_i + 8 * s;
		cp[s].max_dist_x = c[0], cp[s].min_dist_x = c[1], cp[s].max_dist_y = c[2], cp[s].bw = c[3];
		cp[s].max_skip = c[4], cp[s].max_iter = c[5], cp[s].min_cnt = c[6], cp[s].min_sc = c[7], cp[s].gap_scale = cp_f[s];
	}
	R.tee.begin_batch(rp);
	std::vector<SeedTask> t1(n1);
	for (int i = 0; i < n1; ++i) {
		const int32_t *r = rows1 + 4 * i;
		SeedTask &t = t1[i];
		t.win = MapWin{ r[0], r[1], r[2] }, t.flags = 0, t.chain_set = 0, t.n_mask = 0, t.mask_off = 0, t.n_pre = 0, t.pre_off = 0;
	}
	std::vector<SeedOut> o1, o2;
	int32_t no_mask[2] = {0, 0};
	R.tee.seed_chain(t1, no_mask, 0, cp, max_occ, o1);
	std::vector<SeedTask> t2(n2);
	std::vector<wm_pair_t> pre;
	std::vector<int32_t> masks;
	for (int i = 0; i < n2; ++i) {
		const int rd = reads2[i], qlen = (int)rs[rd].seq.size();
		std::vector<wm_pair_t> a;
		std::vector<char> mapped(qlen, 0);
		for (int j = 0; j < n1; ++j) {
			const int32_t *r = rows1 + 4 * j;
			if (r[0] != rd || !r[3] || o1[j].n_u == 0) continue;
			const int wb = r[1], wl = r[2], cnt = (int)(uint32_t)o1[j].u[0]; // the top chain (src/map.c:491-494, :663-666)
			for (int c = 0; c < cnt; ++c) {
				wm_pair_t p = o1[j].b[c];
				p.y += (p.x >> 63) ? (uint64_t)(qlen - wb - wl) : (uint64_t)wb;
				a.push_back(p);
			}
			for (int q = wb; q < wb + wl; ++q) mapped[q] = 1;
		}
		std::sort(a.begin(), a.end(), [](const wm_pair_t &p, const wm_pair_t &q) { return p.x != q.x ? p.x < q.x : p.y < q.y; });
		a.erase(std::unique(a.begin(), a.end(), [](const wm_pair_t &p, const wm_pair_t &q) { return p.x == q.x && p.y == q.y; }), a.end());
		if ((int)a.size() < cp[1].min_cnt) a.clear();
		if (!a.empty()) wmo_radix_sort_128x(a.data(), (long)a.size());
		SeedTask &t = t2[i];
		t.win = MapWin{ rd, 0, qlen }, t.n_mask = 0, t.mask_off = (int64_t)masks.size() / 2, t.n_pre = 0, t.pre_off = 0;
		if (a.empty()) { t.chain_set = 0, t.flags = 0; continue; }
		t.chain_set = 1, t.n_pre = (int32_t)a.size(), t.pre_off = (int64_t)pre.size();
		pre.insert(pre.end(), a.begin(), a.end());
		for (int q = 0; q < qlen;) { // the mapped intervals, sorted and disjoint
			if (!mapped[q]) { ++q; continue; }
			int e = q;
			while (e < qlen && mapped[e]) ++e;
			masks.push_back(q), masks.push_back(e), ++t.n_mask;
			q = e;
		}
		t.flags = t.n_mask == 1 && masks[masks.size() - 2] == 0 && masks.back() == qlen ? SEED_NO_SKETCH : SEED_MASKED;
		if (t.flags == SEED_NO_SKETCH) masks.resize(masks.size() - 2), t.n_mask = 0;
	}
	pre.push_back(wm_pair_t()), masks.push_back(0), masks.push_back(0);
	if (n2 > 0) R.tee.seed_chain(t2, masks.data(), pre.data(), cp, max_occ, o2);
	R.tee.end_batch();
	return R.finish(report_fn);
}

// Crafted run_dp / run_ll batches over query windows of the given reads (win rows: read, wb, wl).  Job rows (int64):
// task, q.kind, q.rid, q.off, q.len, q.reversed, t.kind, t.rid, t.off, t.len, t.reversed, w, zdrop, end_bonus, flag;
// ll rows: the first eleven.  sc_i: q, e, q2, e2.  budget: the CUDA backend's backtrack budget in bytes (0: its default).
extern "C" int wmt_tee_align(const char *ref_fn, int k, int w, int dev_kind, int mutation, int64_t budget, int n_reads, const char *seq, const int64_t *read_off,
                             int n_win, const int32_t *win_rows, int n_dp, const int64_t *dp_rows, int n_ll, const int64_t *ll_rows,
                             const int8_t *mat, const int32_t *sc_i, const char *report_fn)
{
	TeeRun R;
	int rc = R.init(ref_fn, 0, k, w, 0, dev_kind, mutation, budget);
	if (rc < 0) return rc;
	std::vector<wm_read> rs(n_reads);
	std::vector<const wm_read*> rp(n_reads);
	for (int i = 0; i < n_reads; ++i) rs[i].name = "r" + std::to_string(i), rs[i].seq.assign(seq + read_off[i], read_off[i + 1] - read_off[i]), rp[i] = &rs[i];
	std::vector<MapWin> wins(n_win);
	for (int i = 0; i < n_win; ++i) wins[i] = MapWin{ win_rows[3 * i], win_rows[3 * i + 1], win_rows[3 * i + 2] };
	auto ref_of = [](const int64_t *r) { return SeqRef{ (int32_t)r[0], (int32_t)r[1], r[2], (int32_t)r[3], (int32_t)r[4] }; };
	std::vector<DpJob> dj(n_dp);
	for (int i = 0; i < n_dp; ++i) {
		const int64_t *r = dp_rows + 15 * i;
		dj[i].task = (int32_t)r[0], dj[i].q = ref_of(r + 1), dj[i].t = ref_of(r + 6);
		dj[i].w = (int32_t)r[11], dj[i].zdrop = (int32_t)r[12], dj[i].end_bonus = (int32_t)r[13], dj[i].flag = (int32_t)r[14];
	}
	std::vector<LlJob> lj(n_ll);
	for (int i = 0; i < n_ll; ++i) {
		const int64_t *r = ll_rows + 11 * i;
		lj[i].task = (int32_t)r[0], lj[i].q = ref_of(r + 1), lj[i].t = ref_of(r + 6);
	}
	DpScoring sc;
	memcpy(sc.mat, mat, 25); sc.q = sc_i[0], sc.e = sc_i[1], sc.q2 = sc_i[2], sc.e2 = sc_i[3];
	R.tee.begin_batch(rp);
	std::vector<DpRes> dr; std::vector<LlRes> lr;
	if (n_dp > 0) R.tee.run_dp(dj, wins, sc, dr);
	if (n_ll > 0) R.tee.run_ll(lj, wins, sc, lr);
	R.tee.end_batch();
	return R.finish(report_fn);
}
