// C-ABI of the drop-in boundary (include/winnowmap_b200.h): the CUDA context, its lanes, index upload / construction and
// batch mapping (the replacement of kt_for(worker_for), reference src/map.c:1162-1165).  The file-level driver
// (host_driver.cpp) runs over a context through CtxParts.
#include <stddef.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "wm_common.cuh"
#include "sketch.cuh"
#include "index_dev.cuh"
#include "topfreq.cuh"
#include "occ_select.cuh"
#include "gpu_backend.h"
#include "host_cli.h"
#include "host_driver.h"
#include "host_io.h"
#include "host_index.h"
#include "host_timers.h"
#include "host_glue.h"

using namespace wmh;


struct wm_gpu_ctx_s {
	wm_host_idx hidx;
	Backend *be;
	int device;
	MapStats stats;
	double t_index, t_map;
	int64_t n_keys, n_pos;
	std::vector<wm_read> resident; // bench: reads already uploaded by wm_bench_upload ...
	char *d_resident = 0;          // ... their bases, one device pool (wm_read::dev_off)
	std::vector<std::vector<wm_reg1_t>> res_regs; std::vector<int> res_rl; // records of the last wm_bench_map_resident pass (wm_bench_write)
	int64_t n_topfreq = 0; uint64_t topfreq_thr = 0; double t_topfreq = 0; // the -W list counted by wm_index_build_topfreq
	std::string sam_cl;            // command line recorded in the @PG line of SAM output (wm_set_sam_cl)
	std::vector<Backend*> lanes;   // lanes[0] == be; further lanes share the index and own a stream + workspaces
	// host copy of the flattened index, kept for the one-time fan-out to the other GPUs (wm_idx_blob_*)
	std::vector<uint64_t> keys, pos_off, pos;
	std::vector<uint8_t> bloom;
	uint64_t bloom_bits;
	// A multi-part index (wm_index_build_parts): the root owns the parts and the lanes, and its hidx is the sequence table
	// of all parts (names and lengths, no sequence); be is parts[0]->be.  A part is a borrowed context whose root is set:
	// it maps with the root's lanes, bound to its own index arrays.
	std::vector<wm_gpu_ctx_s*> parts;
	wm_gpu_ctx_s *root = 0;
	std::mutex occ_mu; std::vector<std::pair<float, int32_t>> occ_cache; // mid_occ of each mid_occ_frac asked for (wm_idx_cal_max_occ)
};

static bool is_multi(const wm_gpu_ctx_s *c) { return c->parts.size() > 1; }
static wm_gpu_ctx_s *root_of(wm_gpu_ctx_s *c) { return c->root ? c->root : c; }

static void free_reg_vectors(std::vector<std::vector<wm_reg1_t>> &regs);
static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static void require_device(const char *who)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
		fprintf(stderr, "[ERROR] %s: no CUDA device visible; winnowmap-b200 has no CPU fallback\n", who);
		exit(1);
	}
}

// Orchestration lanes: the reads of a call are cut into chunks that L lanes pull from a shared counter and run through
// map_batch concurrently, each lane on its own host thread and CUDA stream, so that one lane's host glue overlaps the
// other lanes' kernels.  Results do not depend on the grouping (reads never interact, src/map.c:1008-1048).
static int n_lanes_wanted(int n_threads)
{ // eight lanes unless WM_LANES says otherwise: a lane mostly waits for the GPU, so lanes pay even with one host thread each
  // (measured with 8 host threads on the tandem-repeat workload: 2 lanes 53, 8 lanes 69 Mbase/s)
	const char *e = getenv("WM_LANES");
	int n = e ? atoi(e) : 8;
	if (!e && n > n_threads) n = n_threads < 2 ? 2 : n_threads;
	return n < 1 ? 1 : n > 16 ? 16 : n;
}

static void ensure_lanes(wm_gpu_ctx_s *c, int n_threads)
{
	if (!c->lanes.empty()) return;
	const int L = n_lanes_wanted(n_threads);
	c->lanes.push_back(c->be);
	const size_t budget = gpu_backend_get_budget(c->be) / (size_t)L;
	for (int i = 1; i < L; ++i) c->lanes.push_back(gpu_backend_clone(c->be, L));
	for (int i = 0; i < L; ++i) { gpu_backend_set_budget(c->lanes[i], budget); c->lanes[i]->set_resident_pool(c->d_resident); }
}

static void map_lanes(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
                      std::vector<int> &rl, std::vector<int> &fg, int n_threads)
{
	wm_gpu_ctx_s *r = root_of(c);
	ensure_lanes(r, n_threads);
	for (Backend *lane : r->lanes) gpu_backend_bind(lane, c->be); // a part of a multi-part index maps with the root's lanes
	MapStats &stats = r->stats;
	const std::vector<Backend*> &lanes = r->lanes;
	const int n = (int)reads.size();
	regs.assign(n, std::vector<wm_reg1_t>()); rl.assign(n, 0); fg.assign(n, 0);
	if (n == 0) return;
	// The reads are cut into chunks of about chunk_bases bases (in input order) that the lanes pull from a shared counter:
	// a lane that finishes early takes the next chunk, and lanes drift out of phase so that one lane's host glue
	// overlaps the other lanes' kernels.
	std::vector<int> cb(1, 0);
	{
		// large chunks amortise the per-wave latencies of a batch; two chunks per lane leave room for the lanes to drift apart
		const char *e = getenv("WM_CHUNK_BASES");
		int64_t total = 0, acc = 0;
		for (int i = 0; i < n; ++i) total += (int64_t)reads[i]->seq.size();
		int64_t chunk_bases = total / (2 * (int64_t)lanes.size()) + 1;
		if (chunk_bases < 4000000) chunk_bases = 4000000;
		if (chunk_bases > 16000000) chunk_bases = 16000000; // eight lanes' workspaces for chunks of this size fit an 80 GB H100
		if (e && atoll(e) > 0) chunk_bases = atoll(e);
		// whole rounds: the latency of a chunk grows much more slowly than its size (it is set by the serial giant tasks of
		// its waves), so a lone chunk left over after the last full round costs almost a whole round.  The chunk size is
		// therefore adjusted (up to +35 %) so that the chunks fill a whole number of rounds of the lanes.
		const int64_t n_lanes = (int64_t)lanes.size();
		int64_t rounds = (int64_t)((double)total / (double)(n_lanes * chunk_bases) + 0.35);
		if (rounds < 1) rounds = 1;
		if (total > n_lanes * chunk_bases * 13 / 20) chunk_bases = (total + n_lanes * rounds - 1) / (n_lanes * rounds);
		else if (total / n_lanes >= 2000000) chunk_bases = (total + n_lanes - 1) / n_lanes; // less than a round: one chunk per lane
		for (int i = 0; i < n; ++i) {
			acc += (int64_t)reads[i]->seq.size();
			if (acc >= chunk_bases || i == n - 1) { cb.push_back(i + 1); acc = 0; }
		}
	}
	const int n_chunks = (int)cb.size() - 1;
	int L = (int)lanes.size();
	if (L > n_chunks) L = n_chunks;
	if (L == 1 && n_chunks == 1) {
		map_batch(lanes[0], &c->hidx, opt, reads, regs, rl, fg, n_threads, &stats);
		wm_dbuf_async = false; // the caller's thread may go on to the one-shot kernel entry points, which allocate synchronously
		return;
	}
	std::vector<MapStats> st(L);
	std::vector<double> lane_end(L, 0.0);
	std::vector<std::thread> th;
	std::atomic<int> next(0);
	const int thr = n_threads / L > 0 ? n_threads / L : 1;
	for (int l = 0; l < L; ++l) {
		memset(&st[l], 0, sizeof(MapStats));
		th.emplace_back([&, l]() {
			for (;;) {
				const int j = next.fetch_add(1);
				if (j >= n_chunks) break;
				std::vector<const wm_read*> sub(reads.begin() + cb[j], reads.begin() + cb[j + 1]);
				std::vector<std::vector<wm_reg1_t>> r2; std::vector<int> rl2, fg2;
				const double tb0 = wmh::Timers::now();
				map_batch(lanes[l], &c->hidx, opt, sub, r2, rl2, fg2, thr, &st[l]);
				wmh::g_timers.add("lane.map_batch", wmh::Timers::now() - tb0);
				for (size_t k = 0; k < sub.size(); ++k) { const int i = cb[j] + (int)k; regs[i].swap(r2[k]); rl[i] = rl2[k]; fg[i] = fg2[k]; }
			}
			lane_end[l] = wmh::Timers::now();
		});
	}
	for (auto &t : th) t.join();
	{ // what the lanes that finished early waited for the last one (tuning aid)
		const double t_end = wmh::Timers::now();
		for (int l = 0; l < L; ++l) wmh::g_timers.add("lane.idle_tail", t_end - lane_end[l]);
	}
	for (int l = 0; l < L; ++l) {
		MapStats &a = stats; const MapStats &b = st[l];
		a.n_reads += b.n_reads, a.n_bases += b.n_bases, a.n_minimaps += b.n_minimaps, a.n_chained += b.n_chained, a.n_dp_jobs += b.n_dp_jobs;
		a.n_ll_jobs += b.n_ll_jobs, a.n_rounds += b.n_rounds, a.t_seed += b.t_seed, a.t_dp += b.t_dp, a.t_host += b.t_host;
	}
}

// the sketch kernels size their shared arrays for the reference's own limits (assert at src/sketch.c:140)
static bool kw_ok(const char *who, int k, int w)
{
	if (w > 0 && w < 256 && k > 0 && k <= 28) return true;
	fprintf(stderr, "[ERROR] %s: k = %d, w = %d outside the supported range (0 < w < 256, 0 < k <= 28; src/sketch.c:140)\n", who, k, w);
	return false;
}

// the index flags the mapping path honours (mm_idx_t::flag, src/minimap.h:41-43): only MM_I_HPC
static bool idx_flag_ok(const char *who, int flag)
{
	if ((flag & ~WM_I_HPC) == 0) return true;
	fprintf(stderr, "[ERROR] %s: index flag 0x%x not supported (only MM_I_HPC = 0x%x)\n", who, flag, WM_I_HPC);
	return false;
}

extern "C" wm_gpu_ctx_s *wm_gpu_idx_upload_flag(const wm_idx_view_t *v, int idx_flag, int device)
{
	require_device("wm_gpu_idx_upload");
	if (!kw_ok("wm_gpu_idx_upload", v->k, v->w) || !idx_flag_ok("wm_gpu_idx_upload", idx_flag & ~WM_I_JUNC)) return 0;
	wm_gpu_ctx_s *c = new wm_gpu_ctx_s();
	memset(&c->stats, 0, sizeof(c->stats));
	c->device = device; c->t_index = c->t_map = 0;
	c->hidx.k = v->k, c->hidx.w = v->w, c->hidx.flag = idx_flag & ~WM_I_JUNC, c->hidx.junc = (idx_flag & WM_I_JUNC) != 0;
	for (int i = 0; i < v->n_seq; ++i) {
		c->hidx.name.push_back(v->seq_name && v->seq_name[i] ? v->seq_name[i] : std::to_string(i));
		c->hidx.len.push_back(v->seq_len[i]);
		c->hidx.offset.push_back(v->seq_offset[i]);
	}
	c->hidx.S.assign(v->S, v->S + v->S_words);
	set_name_order(&c->hidx);
	c->n_keys = v->n_keys, c->n_pos = (int64_t)v->pos_off[v->n_keys];
	c->keys.assign(v->keys, v->keys + v->n_keys);
	c->pos_off.assign(v->pos_off, v->pos_off + v->n_keys + 1);
	c->pos.assign(v->pos, v->pos + v->pos_off[v->n_keys]);
	c->bloom.assign(v->bloom_table, v->bloom_table + v->bloom_bits / 8);
	c->bloom_bits = v->bloom_bits;
	c->be = gpu_backend_create(&c->hidx, v->keys, v->n_keys, v->pos_off, v->pos, v->bloom_bits, v->bloom_table, device);
	return c;
}

extern "C" wm_gpu_ctx_s *wm_gpu_idx_upload(const wm_idx_view_t *v, int device) { return wm_gpu_idx_upload_flag(v, 0, device); }
extern "C" int wm_idx_flag(const wm_gpu_ctx_s *c) { return c->hidx.flag; }

extern "C" void wm_gpu_destroy(wm_gpu_ctx_s *c)
{
	if (!c || c->root) return; // a part belongs to its root
	for (size_t i = 1; i < c->lanes.size(); ++i) gpu_backend_destroy(c->lanes[i]); // clones first: they borrow the owner's index
	if (is_multi(c)) {
		for (wm_gpu_ctx_s *p : c->parts) { gpu_backend_destroy(p->be); delete p; } // lanes[0] is parts[0]->be
	} else gpu_backend_destroy(c->be);
	if (c->d_resident) cudaFree(c->d_resident);
	gpu_backend_trim_pool(c->device);
	free_reg_vectors(c->res_regs);
	delete c;
}

// The reference read once and packed on the device (mm_seq4_set's 2-bit form, pkseq.cuh), about 1 Gbase of ASCII per group:
// the pools stay resident (0.375 bytes per base) until the index is sketched, so that the -W list can be counted from them
// first.  With H, the sequence table and the 4-bit host copy S are filled as well.
struct ref_pools {
	struct group {
		uint32_t *pk = 0, *nm = 0; int64_t *d_off = 0; std::vector<wm_sk_task> tasks; int part = 0;
		void release() { cudaFree(pk); cudaFree(nm); cudaFree(d_off); pk = nm = 0; d_off = 0; }
	};
	std::vector<group> g;
	~ref_pools() { release(); }
	void release() { for (auto &x : g) x.release(); g.clear(); }
	std::vector<wm_tf_group> tf() const
	{
		std::vector<wm_tf_group> v;
		for (auto &x : g) v.push_back(wm_tf_group{ x.pk, x.nm, x.d_off, (int)x.tasks.size() });
		return v;
	}
};

// The reference is cut into index parts by PartCutter (host_driver.h); H (if not null) gets one sequence table per part:
// rid and offset restart at 0 in every part
static bool read_ref_pools(const char *ref_fn, std::vector<wm_host_idx> *H, uint64_t batch_size, int mini_batch_size, ref_pools &P)
{
	SeqReader rd;
	if (!rd.open(ref_fn)) { fprintf(stderr, "ERROR: failed to open file '%s'\n", ref_fn); return false; }
	std::vector<wm_sk_task> tasks; std::string group; uint64_t sum_len = 0; uint32_t n_seq = 0;
	PartCutter cut(batch_size, mini_batch_size);
	int part = -1;
	wm_dbuf d_ascii;
	auto flush = [&]() {
		if (tasks.empty()) return;
		ref_pools::group G;
		G.part = part;
		const int64_t n = (int64_t)group.size();
		char *da = (char*)d_ascii.need(group.size() + 16);
		G.pk = wm_dev_alloc<uint32_t>(wm_pk_words(n)), G.nm = wm_dev_alloc<uint32_t>(wm_nm_words(n));
		WM_CUDA_CHECK(cudaMemcpy(da, group.data(), group.size(), cudaMemcpyHostToDevice));
		wm_pack_ascii(da, n, G.pk, G.nm, 0);
		std::vector<int64_t> off;
		for (auto &t : tasks) off.push_back(t.seq_off);
		off.push_back(n);
		G.d_off = wm_dev_alloc<int64_t>(off.size());
		WM_CUDA_CHECK(cudaMemcpy(G.d_off, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice));
		G.tasks.swap(tasks);
		P.g.push_back(std::move(G));
		tasks.clear(); group.clear();
	};
	wm_read r;
	while (rd.next(r)) {
		const int p = cut.next(r.seq.size());
		if (p != part) {
			flush();
			part = p, sum_len = 0, n_seq = 0;
			if (H) H->emplace_back();
		}
		const uint32_t rid = n_seq++;
		if (H) {
			wm_host_idx *h = &H->back();
			h->name.push_back(r.name); h->len.push_back((uint32_t)r.seq.size()); h->offset.push_back(sum_len);
			const uint64_t need_words = (sum_len + r.seq.size() + 7) / 8;
			if (h->S.size() < need_words) h->S.resize(need_words, 0);
			pack_seq4(h->S.data(), sum_len, r.seq.data(), r.seq.size());
		}
		sum_len += r.seq.size();
		if (!r.seq.empty()) {
			wm_sk_task t; t.seq_off = (int64_t)group.size(); t.len = (int32_t)r.seq.size(); t.rid = rid;
			tasks.push_back(t); group += r.seq;
		}
		if (group.size() >= ((size_t)1 << 30)) flush();
	}
	flush();
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	return true;
}

// the meryl option distinct=D (merylOp-nextMer.C:103-115): a fraction of the distinct k-mers, 0 < D <= 1
static bool distinct_ok(const char *who, double d)
{
	if (d > 0.0 && d <= 1.0) return true;
	fprintf(stderr, "[ERROR] %s: distinct = %g outside (0, 1]\n", who, d);
	return false;
}

static wm_gpu_ctx_s *new_ctx(int device)
{
	wm_gpu_ctx_s *c = new wm_gpu_ctx_s();
	memset(&c->stats, 0, sizeof(c->stats));
	c->device = device; c->t_index = c->t_map = 0;
	return c;
}

// One index from the groups of part `part` of P (the groups are freed once sketched): the minimizers stay on the device,
// where they are sorted and cut into the CSR (index_dev.cu).
static wm_gpu_ctx_s *build_part(wm_host_idx &&H, ref_pools &P, int part, const wm_bloom_dev &bf, wm_bloom_s *bloom, int device)
{
	wm_gpu_ctx_s *c = new_ctx(device);
	c->hidx = std::move(H);
	const int k = c->hidx.k, w = c->hidx.w;
	std::vector<std::pair<wm128_dev*, int64_t>> sk; int64_t n_mz_total = 0;
	{
		wm_sketch_ws ws;
		for (auto &G : P.g) {
			if (G.part != part) continue;
			wm_pkseq pks; pks.pk = G.pk, pks.nm = G.nm;
			int64_t n_mz = 0;
			if (c->hidx.flag & WM_I_HPC) wm_sketch_run_hpc(&ws, bf, pks, G.tasks.data(), (int)G.tasks.size(), w, k, &n_mz, 0);
			else wm_sketch_run(&ws, bf, pks, G.tasks.data(), (int)G.tasks.size(), w, k, &n_mz, 0);
			WM_CUDA_CHECK(cudaDeviceSynchronize());
			if (n_mz > 0) {
				wm128_dev *d = wm_dev_alloc<wm128_dev>(n_mz);
				WM_CUDA_CHECK(cudaMemcpy(d, ws.mz.p, sizeof(wm128_dev) * n_mz, cudaMemcpyDeviceToDevice));
				sk.push_back(std::make_pair(d, n_mz)); n_mz_total += n_mz;
			}
			G.release();
		}
	}
	set_name_order(&c->hidx);
	// one array in position order, then sort + CSR on the device
	wm128_dev *d_all = wm_dev_alloc<wm128_dev>(n_mz_total + 1);
	{
		int64_t o = 0;
		for (auto &pp : sk) { WM_CUDA_CHECK(cudaMemcpy(d_all + o, pp.first, sizeof(wm128_dev) * pp.second, cudaMemcpyDeviceToDevice)); o += pp.second; cudaFree(pp.first); }
	}
	uint64_t *d_keys = 0, *d_poff = 0, *d_pos = 0; int64_t n_keys = 0;
	wm_index_build_dev(d_all, n_mz_total, k, &d_keys, &d_poff, &d_pos, &n_keys, 0);
	c->n_keys = n_keys, c->n_pos = n_mz_total;
	c->be = gpu_backend_create_dev(&c->hidx, d_keys, n_keys, d_poff, d_pos, wm_bloom_bits(bloom), wm_bloom_table(bloom), device);
	c->bloom_bits = wm_bloom_bits(bloom);
	c->bloom.assign(wm_bloom_table(bloom), wm_bloom_table(bloom) + c->bloom_bits / 8);
	return c;
}

// Index construction from a FASTA file (mm_idx_gen, src/index.c:378-449): same minimizers as the reference
// because the reference sequences go through the same sketch kernel as the reads.  With WM_I_HPC the minimizers are
// those of the homopolymer-compressed sequences (mm_sketch with is_hpc, src/index.c:347); S stays uncompressed.
// The -W list comes from kmer_freq_fn, or, with distinct > 0, is counted on the device from the packed reference itself
// (uncompressed also under WM_I_HPC: the list a user gets from meryl on ref.fa).  The reference is cut into parts of about
// batch_size bases as mm_idx_gen cuts it (PartCutter); UINT64_MAX gives one index whatever the size.  The FASTA is read,
// the -W list counted and the filter built once for all parts.
static wm_gpu_ctx_s *index_build(const char *who, const char *ref_fn, const char *kmer_freq_fn, double distinct, int k, int w, int idx_flag,
                                 uint64_t batch_size, int mini_batch_size, int device)
{
	require_device(who);
	if (!kw_ok(who, k, w) || !idx_flag_ok(who, idx_flag) || (distinct != 0.0 && !distinct_ok(who, distinct))) return 0;
	WM_CUDA_CHECK(cudaSetDevice(device));
	const double t0 = now_s();
	std::vector<wm_host_idx> Hs;
	ref_pools P;
	if (!read_ref_pools(ref_fn, &Hs, batch_size, mini_batch_size, P)) return 0;
	if (Hs.empty()) Hs.emplace_back(); // an empty reference: one empty index
	for (auto &H : Hs) H.k = k, H.w = w, H.flag = idx_flag;
	std::vector<uint64_t> kmers;
	int64_t n_topfreq = 0; uint64_t topfreq_thr = 0; double t_topfreq = 0;
	if (distinct != 0.0) {
		const double tc = now_s();
		wm_tf_list L;
		wm_topfreq_dev(P.tf(), k, distinct, &L, 0);
		kmers.swap(L.codes);
		n_topfreq = (int64_t)kmers.size(), topfreq_thr = L.threshold, t_topfreq = now_s() - tc;
	} else if (read_kmer_list(kmer_freq_fn, k, kmers) < 0) abort();
	wm_bloom_s *bloom = wm_bloom_build(kmers.empty() ? 0 : kmers.data(), (int64_t)kmers.size());
	uint8_t *d_table = wm_dev_alloc<uint8_t>(wm_bloom_bits(bloom) / 8 + 16);
	WM_CUDA_CHECK(cudaMemcpy(d_table, wm_bloom_table(bloom), wm_bloom_bits(bloom) / 8, cudaMemcpyHostToDevice));
	wm_bloom_dev bf; wm_bloom_dev_from_table(&bf, d_table, wm_bloom_bits(bloom));
	std::vector<wm_gpu_ctx_s*> parts;
	for (size_t p = 0; p < Hs.size(); ++p) parts.push_back(build_part(std::move(Hs[p]), P, (int)p, bf, bloom, device));
	P.release(); cudaFree(d_table);
	wm_bloom_destroy(bloom);
	wm_gpu_ctx_s *c = parts[0];
	if (parts.size() > 1) { // the root: the sequence table of all parts, in part order (the merged index of mm_split_merge_prep)
		c = new_ctx(device);
		c->hidx.k = k, c->hidx.w = w, c->hidx.flag = idx_flag;
		c->n_keys = c->n_pos = 0;
		for (wm_gpu_ctx_s *p : parts) {
			c->hidx.name.insert(c->hidx.name.end(), p->hidx.name.begin(), p->hidx.name.end());
			c->hidx.len.insert(c->hidx.len.end(), p->hidx.len.begin(), p->hidx.len.end());
			c->n_keys += p->n_keys, c->n_pos += p->n_pos;
			p->root = c;
		}
		c->parts = parts;
		c->be = parts[0]->be;
	}
	c->n_topfreq = n_topfreq, c->topfreq_thr = topfreq_thr, c->t_topfreq = t_topfreq;
	c->t_index = now_s() - t0;
	return c;
}

extern "C" wm_gpu_ctx_s *wm_index_build(const char *ref_fn, const char *kmer_freq_fn, int k, int w, int device)
{
	return index_build("wm_index_build", ref_fn, kmer_freq_fn, 0.0, k, w, 0, UINT64_MAX, 0, device);
}

extern "C" wm_gpu_ctx_s *wm_index_build_opt(const char *ref_fn, const char *kmer_freq_fn, const wm_idxopt_t *io, int device)
{
	return index_build("wm_index_build_opt", ref_fn, kmer_freq_fn, 0.0, io->k, io->w, io->flag, UINT64_MAX, 0, device);
}

extern "C" wm_gpu_ctx_s *wm_index_build_topfreq(const char *ref_fn, const wm_idxopt_t *io, double distinct, int device)
{
	if (!distinct_ok("wm_index_build_topfreq", distinct)) return 0;
	return index_build("wm_index_build_topfreq", ref_fn, 0, distinct, io->k, io->w, io->flag, UINT64_MAX, 0, device);
}

extern "C" wm_gpu_ctx_s *wm_index_build_parts(const char *ref_fn, const char *kmer_freq_fn, const wm_idxopt_t *io, double distinct, int device)
{
	if (distinct != 0.0 && kmer_freq_fn) { fprintf(stderr, "[ERROR] wm_index_build_parts: give either a -W file or distinct, not both\n"); return 0; }
	return index_build("wm_index_build_parts", ref_fn, kmer_freq_fn, distinct, io->k, io->w, io->flag, io->batch_size, io->mini_batch_size, device);
}

extern "C" int wm_part_plan(const char *ref_fn, uint64_t batch_size, int mini_batch_size, int32_t *n_seq, int cap)
{
	SeqReader rd;
	if (!rd.open(ref_fn)) { fprintf(stderr, "ERROR: failed to open file '%s'\n", ref_fn); return -1; }
	PartCutter cut(batch_size, mini_batch_size);
	std::vector<int32_t> n;
	wm_read r;
	while (rd.next(r)) {
		const int p = cut.next(r.seq.size());
		if (p >= (int)n.size()) n.push_back(0);
		++n[p];
	}
	for (int i = 0; i < (int)n.size() && i < cap; ++i) n_seq[i] = n[i];
	return (int)n.size();
}

extern "C" int wm_idx_n_parts(const wm_gpu_ctx_s *c) { return is_multi(c) ? (int)c->parts.size() : 1; }
extern "C" wm_gpu_ctx_s *wm_idx_part(wm_gpu_ctx_s *c, int i)
{
	if (is_multi(c)) return i >= 0 && (size_t)i < c->parts.size() ? c->parts[i] : 0;
	return i == 0 ? c : 0;
}

// meryl count k=K + meryl print greater-than distinct=D on ref_fn: the list's length; up to cap (code, count) pairs into
// kmers / counts (NULL with cap = 0: count only), the threshold into *threshold; -1 when k or distinct is refused
extern "C" int64_t wm_topfreq(const char *ref_fn, int k, double distinct, uint64_t *kmers, uint32_t *counts, int64_t cap, uint64_t *threshold, int device)
{
	require_device("wm_topfreq");
	if (k < 1 || k > 28) { fprintf(stderr, "[ERROR] wm_topfreq: k = %d outside the supported range (0 < k <= 28; src/sketch.c:140)\n", k); return -1; }
	if (!distinct_ok("wm_topfreq", distinct)) return -1;
	WM_CUDA_CHECK(cudaSetDevice(device));
	ref_pools P;
	if (!read_ref_pools(ref_fn, 0, UINT64_MAX, 0, P)) return -1;
	wm_tf_list L;
	wm_topfreq_dev(P.tf(), k, distinct, &L, 0);
	const int64_t n = (int64_t)L.codes.size(), m = std::min<int64_t>(n, cap > 0 ? cap : 0);
	if (m > 0) { memcpy(kmers, L.codes.data(), sizeof(uint64_t) * m); memcpy(counts, L.counts.data(), sizeof(uint32_t) * m); }
	if (threshold) *threshold = L.threshold;
	return n;
}

extern "C" int wm_set_opt(const char *preset, wm_idxopt_t *io, wm_mapopt_t *mo) { return set_opt(preset, io, mo); }
extern "C" int wm_check_opt(const wm_idxopt_t *io, const wm_mapopt_t *mo) { return check_opt(io, mo); }
extern "C" void wm_mapopt_max_intron_len(wm_mapopt_t *opt, int max_intron_len) { mapopt_max_intron_len(opt, max_intron_len); }
// mm_idx_cal_max_occ (src/index.c:173-194) of one index: INT32_MAX for f <= 0, else the ((1 - f) * n)-th smallest occurrence
// count over the n keys, plus one, selected on the device (occ_select.cu) and remembered per f.  -1, with a message, where
// the reference would read past its array (the rank reaches n: f too small for the number of keys, or no key at all) and
// on a multi-part context, whose parts each have their own value.
extern "C" int32_t wm_idx_cal_max_occ(const wm_gpu_ctx_s *c_, float f)
{
	wm_gpu_ctx_s *c = const_cast<wm_gpu_ctx_s*>(c_);
	if (f <= 0.) return INT32_MAX;
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_idx_cal_max_occ: a multi-part index has one value per part (wm_idx_part)\n"); return -1; }
	std::lock_guard<std::mutex> lk(c->occ_mu);
	for (auto &e : c->occ_cache) if (e.first == f) return e.second;
	const uint64_t n = (uint64_t)c->n_keys, rank = (uint32_t)((1. - f) * n);
	if (rank >= n) {
		fprintf(stderr, "[ERROR] wm_idx_cal_max_occ: f = %g selects rank %llu of %llu occurrence counts; the reference reads past its array here\n",
		        (double)f, (unsigned long long)rank, (unsigned long long)n);
		return -1;
	}
	WM_CUDA_CHECK(cudaSetDevice(c->device));
	const uint64_t *dk, *dpo, *dp;
	gpu_backend_index_arrays(c->be, &dk, &dpo, &dp);
	const int32_t v = (int32_t)(wm_occ_select_dev(dpo, (int64_t)n, rank, 0) + 1);
	c->occ_cache.push_back(std::make_pair(f, v));
	return v;
}

// mm_mapopt_update (src/options.c:71-81) against one index; 0, or -1 when wm_idx_cal_max_occ refuses
extern "C" int wm_mapopt_update(wm_mapopt_t *opt, const wm_gpu_ctx_s *c)
{
	if ((opt->flag & WM_F_SPLICE_FOR) || (opt->flag & WM_F_SPLICE_REV)) opt->flag |= WM_F_SPLICE;
	if (opt->mid_occ_frac >= 0 && opt->mid_occ_frac < 1) {
		const int32_t m = wm_idx_cal_max_occ(c, opt->mid_occ_frac);
		if (m < 0) return -1;
		opt->mid_occ = m;
	}
	if (opt->mid_occ < opt->min_mid_occ) opt->mid_occ = opt->min_mid_occ;
	return 0;
}

// The options one index maps with: under -f, mid_occ of that index (what mm_mapopt_update sets per part, src/main.c:403);
// without -f, opt unchanged.  false when the selection is refused.
static bool part_opt(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, wm_mapopt_t *o)
{
	*o = *opt;
	if (!(opt->mid_occ_frac >= 0 && opt->mid_occ_frac < 1)) return true;
	if (wm_mapopt_update(o, c) < 0) return false;
	o->mid_occ_frac = -1.0f; // resolved
	return true;
}

extern "C" int wm_sizeof_mapopt(void) { return (int)sizeof(wm_mapopt_t); }
extern "C" int wm_sizeof_reg1(void) { return (int)sizeof(wm_reg1_t); }
extern "C" int wm_abi_layout(int64_t *out, int cap)
{
	int n = 0;
#define PUT(v) do { if (n < cap) out[n] = (int64_t)(v); ++n; } while (0)
	PUT(sizeof(wm_mapopt_t)); PUT(sizeof(wm_reg1_t)); PUT(sizeof(wm_extra_t)); PUT(sizeof(wm_idxopt_t));
#define MO(f) PUT(offsetof(wm_mapopt_t, f))
	MO(flag); MO(seed); MO(sdust_thres); MO(max_qlen); MO(bw); MO(max_gap); MO(max_gap_ref); MO(min_gap_ref); MO(max_frag_len); MO(max_chain_skip);
	MO(max_chain_iter); MO(min_cnt); MO(min_chain_score); MO(chain_gap_scale); MO(SVaware); MO(SVawareMinReadLength); MO(suffixSampleOffset);
	MO(min_mapq); MO(min_qcov); MO(minPrefixLength); MO(maxPrefixLength); MO(prefixIncrementFactor); MO(stage2_bw); MO(stage2_zdrop_inv);
	MO(stage2_max_gap); MO(stage2_extension_inc); MO(mask_level); MO(mask_len); MO(pri_ratio); MO(best_n); MO(max_join_long); MO(max_join_short);
	MO(min_join_flank_sc); MO(min_join_flank_ratio); MO(alt_drop); MO(a); MO(b); MO(q); MO(e); MO(q2); MO(e2); MO(sc_ambi); MO(noncan); MO(junc_bonus);
	MO(zdrop); MO(zdrop_inv); MO(end_bonus); MO(min_dp_max); MO(min_ksw_len); MO(anchor_ext_len); MO(anchor_ext_shift); MO(max_clip_ratio);
	MO(pe_ori); MO(pe_bonus); MO(mid_occ_frac); MO(min_mid_occ); MO(mid_occ); MO(max_occ); MO(mini_batch_size); MO(max_sw_mat);
	MO(kmer_freq_filename); MO(split_prefix);
#define RG(f) PUT(offsetof(wm_reg1_t, f))
	RG(id); RG(cnt); RG(rid); RG(score); RG(qs); RG(qe); RG(rs); RG(re); RG(parent); RG(subsc); RG(as); RG(mlen); RG(blen); RG(n_sub); RG(score0); RG(hash); RG(div); RG(p);
#define EX(f) PUT(offsetof(wm_extra_t, f))
	EX(capacity); EX(dp_score); EX(dp_max); EX(dp_max2); EX(n_cigar); EX(cigar);
#define IO(f) PUT(offsetof(wm_idxopt_t, f))
	IO(k); IO(w); IO(flag); IO(bucket_bits); IO(mini_batch_size); IO(batch_size);
#undef PUT
#undef MO
#undef RG
#undef EX
#undef IO
	return n;
}

// The parts of a context in order: its own index for a single one
static std::vector<wm_gpu_ctx_s*> parts_of(wm_gpu_ctx_s *c) { return is_multi(c) ? c->parts : std::vector<wm_gpu_ctx_s*>(1, c); }

// The file driver's view of a context (host_driver.h): its parts, each mapped with the root's lanes, and -f resolved per
// part by part_opt with the occurrence cache
struct CtxParts : IndexParts {
	wm_gpu_ctx_s *c; std::vector<wm_gpu_ctx_s*> parts;
	explicit CtxParts(wm_gpu_ctx_s *c) : c(c), parts(parts_of(c)) {}
	int n_parts() const override { return (int)parts.size(); }
	const wm_host_idx *part(int p) const override { return &parts[p]->hidx; }
	const wm_host_idx *all() const override { return &c->hidx; }
	bool part_opt(int p, const wm_mapopt_t *opt, wm_mapopt_t *o) override { return ::part_opt(parts[p], opt, o); }
	void map(int p, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
	         std::vector<int> &rep_len, int n_threads) override
	{
		std::vector<int> fg;
		map_lanes(parts[p], opt, reads, regs, rep_len, fg, n_threads);
	}
};

// The GPU replacement of kt_for(n_threads, worker_for, ...) (src/map.c:1164): fills n_reg/reg/rep_len/frag_gap of
// every sequence exactly as worker_for does (:1025-1034).  reg[i] and each reg[i][j].p are malloc()ed; the caller
// frees them (src/minimap.h:355-356).
extern "C" int wm_gpu_map_batch(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, int n_seq, const char *const *names, const char *const *seqs,
                                const int32_t *lens, int32_t *n_reg, wm_reg1_t **reg, int32_t *rep_len, int32_t *frag_gap, int n_threads)
{
	require_device("wm_gpu_map_batch");
	std::vector<wm_read> store(n_seq);
	std::vector<const wm_read*> reads(n_seq);
	#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads > 0 ? n_threads : 1)
	for (int i = 0; i < n_seq; ++i) {
		store[i].name = names && names[i] ? names[i] : "";
		store[i].has_name = names && names[i];
		store[i].seq.assign(seqs[i], lens[i]);
		reads[i] = &store[i];
	}
	std::vector<std::vector<wm_reg1_t>> regs; std::vector<int> rl, fg;
	if (is_multi(c)) {
		if (!opt->split_prefix) {
			fprintf(stderr, "[ERROR] wm_gpu_map_batch: a multi-part index maps part by part (wm_idx_part) unless split_prefix asks for merged hits\n");
			return -1;
		}
		CtxParts ix(c);
		if (!map_merged(ix, opt, reads, regs, n_threads)) return -1;
		rl.assign(n_seq, 0), fg.assign(n_seq, 0);
	} else {
		wm_mapopt_t o;
		if (!part_opt(c, opt, &o)) return -1;
		map_lanes(c, &o, reads, regs, rl, fg, n_threads);
	}
	for (int i = 0; i < n_seq; ++i) {
		n_reg[i] = (int32_t)regs[i].size();
		reg[i] = 0;
		if (n_reg[i] > 0) {
			reg[i] = (wm_reg1_t*)malloc(sizeof(wm_reg1_t) * n_reg[i]);
			memcpy(reg[i], regs[i].data(), sizeof(wm_reg1_t) * n_reg[i]);
		}
		rep_len[i] = rl[i], frag_gap[i] = fg[i];
	}
	return 0;
}

// mm_tbuf_t / mm_map (src/map.c:18-38, :976-984): the per-thread buffer only carries rep_len and frag_gap of the last call here
// (device workspaces belong to the context's lanes).  One read = a batch of one through the same path as wm_gpu_map_batch.
struct wm_tbuf_s { int rep_len, frag_gap; };
extern "C" wm_tbuf_s *wm_tbuf_init(void) { return (wm_tbuf_s*)calloc(1, sizeof(wm_tbuf_s)); }
extern "C" void wm_tbuf_destroy(wm_tbuf_s *b) { free(b); }
extern "C" int wm_tbuf_rep_len(const wm_tbuf_s *b) { return b->rep_len; }
extern "C" int wm_tbuf_frag_gap(const wm_tbuf_s *b) { return b->frag_gap; }
extern "C" wm_reg1_t *wm_map(wm_gpu_ctx_s *c, int l_seq, const char *seq, int *n_regs, wm_tbuf_s *b, const wm_mapopt_t *opt, const char *name)
{
	int32_t n_reg = 0, rl = 0, fg = 0, len = l_seq;
	wm_reg1_t *reg = 0;
	wm_gpu_map_batch(c, opt, 1, &name, &seq, &len, &n_reg, &reg, &rl, &fg, 1); // name == NULL: qname == 0
	if (b) b->rep_len = rl, b->frag_gap = fg;
	*n_regs = n_reg;
	return reg;
}

// mm_map_file (src/map.c:1244-1276) over the parts of c: the driver of host_driver.cpp with the context's lanes
extern "C" int wm_map_file(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, const char *reads_fn, const char *out_fn, int n_threads, int rank, int world,
                           int tag_order, int64_t max_batch_bases)
{
	require_device("wm_map_file");
	const double t0 = now_s();
	CtxParts ix(c);
	const int rc = map_file(ix, opt, reads_fn, out_fn, c->sam_cl.c_str(), n_threads, rank, world, tag_order, max_batch_bases);
	c->t_map += now_s() - t0;
	return rc;
}

extern "C" void wm_set_sam_cl(wm_gpu_ctx_s *c, const char *cl) { c->sam_cl = cl ? cl : ""; }

// The winnowmap command line (host_cli.h) over an index built on device 0, cut into parts under -I
extern "C" int wm_cli_main(int argc, char **argv)
{
	struct OwnedParts : CtxParts {
		explicit OwnedParts(wm_gpu_ctx_s *c) : CtxParts(c) {}
		~OwnedParts() override { wm_gpu_destroy(c); }
	};
	return cli_main(argc, argv, [](const CliArgs &a) -> std::unique_ptr<IndexParts> {
		require_device("winnowmap-b200");
		wm_idxopt_t io = a.ipt;
		io.flag &= WM_I_HPC; // the other index flags only drop what a prebuilt index stores
		wm_gpu_ctx_s *c = wm_index_build_parts(a.files[0].c_str(), a.has_kmer ? a.kmer_fn.c_str() : 0, &io, 0.0, 0);
		if (!c) return nullptr;
		return std::unique_ptr<IndexParts>(new OwnedParts(c));
	});
}

// mm_gen_cs / mm_gen_MD (src/minimap.h:389-390, src/format.c:245-266): *buf is (re)allocated with realloc() when it is too
// small, *max_len is its capacity; the string is NUL terminated; returns its length
static int gen_cs_or_md_c(const wm_gpu_ctx_s *c, char **buf, int *max_len, const wm_reg1_t *r, const char *seq, int is_MD, int no_iden)
{
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_gen_cs / wm_gen_MD: the reference sequence is held by the parts of a multi-part index (wm_idx_part)\n"); return -1; }
	std::string s;
	gen_cs_or_MD(s, &c->hidx, r, seq, is_MD, no_iden);
	if ((int)s.size() + 1 > *max_len) {
		int m = (int)s.size() + 1;
		m += m >> 1; // kroundup-like slack
		*buf = (char*)realloc(*buf, (size_t)m);
		*max_len = m;
	}
	memcpy(*buf, s.data(), s.size());
	(*buf)[s.size()] = 0;
	return (int)s.size();
}
// mm_idx_getseq / mm_idx_name2id (src/index.c:161-171, :131-140) and the sequence table of the index (mm_idx_seq_t)
extern "C" int wm_idx_getseq(const wm_gpu_ctx_s *c, uint32_t rid, uint32_t st, uint32_t en, uint8_t *seq)
{
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_idx_getseq: the reference sequence is held by the parts of a multi-part index (wm_idx_part)\n"); return -1; }
	return c->hidx.getseq(rid, st, en, seq);
}
extern "C" int wm_idx_name2id(const wm_gpu_ctx_s *c, const char *name)
{
	for (size_t i = 0; i < c->hidx.name.size(); ++i) if (c->hidx.name[i] == name) return (int)i;
	return -1;
}
// mm_idx_bed_read(mi, fn, 1) once per index part (src/main.c:416 runs it on every part the index reader returns), each part
// with its own names; then the intervals go to that part's device index
extern "C" int wm_idx_bed_read(wm_gpu_ctx_s *c, const char *fn)
{
	for (wm_gpu_ctx_s *p : parts_of(c)) {
		if (read_bed_junc(&p->hidx, fn) < 0) return -1;
		gpu_backend_set_junc(p->be, &p->hidx);
	}
	return 0;
}
extern "C" int wm_idx_set_junc(wm_gpu_ctx_s *c, const wm_idx_intv_t *I)
{
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_idx_set_junc: a multi-part index takes the intervals of each part (wm_idx_part)\n"); return -1; }
	set_junc(&c->hidx, I);
	gpu_backend_set_junc(c->be, &c->hidx);
	return 0;
}
extern "C" int wm_idx_n_seq(const wm_gpu_ctx_s *c) { return (int)c->hidx.name.size(); }
extern "C" const char *wm_idx_seq_name(const wm_gpu_ctx_s *c, int rid) { return rid >= 0 && (size_t)rid < c->hidx.name.size() ? c->hidx.name[rid].c_str() : 0; }
extern "C" uint32_t wm_idx_seq_len(const wm_gpu_ctx_s *c, int rid) { return rid >= 0 && (size_t)rid < c->hidx.len.size() ? c->hidx.len[rid] : 0; }

extern "C" int wm_gen_cs(const wm_gpu_ctx_s *c, char **buf, int *max_len, const wm_reg1_t *r, const char *seq, int no_iden)
{ return gen_cs_or_md_c(c, buf, max_len, r, seq, 0, no_iden); }
extern "C" int wm_gen_MD(const wm_gpu_ctx_s *c, char **buf, int *max_len, const wm_reg1_t *r, const char *seq)
{ return gen_cs_or_md_c(c, buf, max_len, r, seq, 1, 0); }

extern "C" void wm_get_stats(wm_gpu_ctx_s *c, double *o, int n)
{
	const MapStats &s = c->stats;
	double v[] = { (double)s.n_reads, (double)s.n_bases, (double)s.n_minimaps, (double)s.n_chained, (double)s.n_dp_jobs, (double)s.n_ll_jobs,
	               (double)s.n_rounds, s.t_seed, s.t_dp, s.t_host, c->t_index, c->t_map, (double)c->n_keys, (double)c->n_pos,
	               (double)c->n_topfreq, (double)c->topfreq_thr, c->t_topfreq };
	for (int i = 0; i < n && i < (int)(sizeof(v) / sizeof(v[0])); ++i) o[i] = v[i];
}
extern "C" void wm_reset_stats(wm_gpu_ctx_s *c) { memset(&c->stats, 0, sizeof(c->stats)); c->t_map = 0; }

// ---- bench instrumentation ----
extern "C" void wm_prof_enable(int on) { g_wm_prof.enabled = on; }
extern "C" void wm_prof_reset(void) { int e = g_wm_prof.enabled; memset(&g_wm_prof, 0, sizeof(g_wm_prof)); g_wm_prof.enabled = e; wm_prof_region_begin(); }
extern "C" void wm_prof_get(double *o)
{ // o[0]: kernel launches; then per kernel class (0 = DP fill at o[1..6], 1 = chaining forward pass at o[7..12]):
  // sum of launch ms, union of launch intervals ms, launches, algorithmic bytes, units (block cells / anchors), units2 (DP jobs)
	wm_prof_collect();
	o[0] = (double)g_wm_prof.n_launches;
	for (int k = 0; k < WM_PK_N; ++k) {
		const wm_prof_kind &K = g_wm_prof.k[k];
		double *q = o + 1 + 6 * k;
		q[0] = K.ms, q[1] = K.union_ms, q[2] = (double)K.launches, q[3] = K.alg_bytes, q[4] = K.units, q[5] = K.units2;
	}
}
// host<->device traffic of the mapping path since wm_prof_reset: o[0] = host-to-device bytes, o[1] = device-to-host bytes
extern "C" void wm_prof_get_copies(double *o) { o[0] = (double)g_wm_prof.h2d_bytes; o[1] = (double)g_wm_prof.d2h_bytes; }
extern "C" int wm_device_synchronize(void) { WM_CUDA_CHECK(cudaDeviceSynchronize()); return 0; }
// free / total bytes of the current device (bench: with the stream-ordered pool never trimmed while mapping, total - free after a
// pass is the high-water mark of the library's footprint)
extern "C" int wm_device_mem(double *free_bytes, double *total_bytes)
{
	size_t f = 0, t = 0;
	WM_CUDA_CHECK(cudaMemGetInfo(&f, &t));
	*free_bytes = (double)f, *total_bytes = (double)t;
	return 0;
}

extern "C" void wm_free_regs(int n, const int32_t *n_reg, wm_reg1_t **reg)
{ // what the reference's output step does after printing (src/map.c:1210-1211)
	for (int i = 0; i < n; ++i) {
		for (int j = 0; j < n_reg[i]; ++j) free(reg[i][j].p);
		free(reg[i]);
	}
}

// bench: put a batch of reads into HBM (ASCII -> codes, both strands) outside the timed region ...
extern "C" int wm_bench_upload(wm_gpu_ctx_s *c, int n_seq, const char *const *names, const char *const *seqs, const int32_t *lens)
{
	if (is_multi(c) || c->root) { fprintf(stderr, "[ERROR] wm_bench_upload: resident reads are for a single index\n"); return -1; }
	c->resident.assign(n_seq, wm_read());
	int64_t tot = 0;
	for (int i = 0; i < n_seq; ++i) {
		c->resident[i].name = names && names[i] ? names[i] : "";
		c->resident[i].seq.assign(seqs[i], lens[i]);
		c->resident[i].dev_off = tot;
		tot += lens[i];
	}
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	if (c->d_resident) { WM_CUDA_CHECK(cudaFree(c->d_resident)); c->d_resident = 0; }
	WM_CUDA_CHECK(cudaMalloc((void**)&c->d_resident, (size_t)tot + 16));
	{
		std::vector<char> stage((size_t)tot + 1);
		for (int i = 0; i < n_seq; ++i) memcpy(stage.data() + c->resident[i].dev_off, seqs[i], lens[i]);
		WM_CUDA_CHECK(cudaMemcpy(c->d_resident, stage.data(), (size_t)tot, cudaMemcpyHostToDevice));
	}
	for (auto *be : c->lanes) be->set_resident_pool(c->d_resident);
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	return 0;
}

// ... and map them with the device copies already resident; *ms = device time between two events that bracket the
// whole step (recorded on the legacy default stream, which orders against the backend's blocking stream).
static void free_reg_vectors(std::vector<std::vector<wm_reg1_t>> &regs)
{
	for (auto &v : regs) for (auto &r : v) free(r.p);
	regs.clear();
}

extern "C" int wm_bench_map_resident(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, int n_threads, int group_reads, double *ms)
{ // the resident reads are submitted in groups of group_reads reads (<= 0: all at once); two events bracket the whole pass
	static cudaEvent_t e0 = 0, e1 = 0;
	if (!e0) { WM_CUDA_CHECK(cudaEventCreate(&e0)); WM_CUDA_CHECK(cudaEventCreate(&e1)); }
	const int n = (int)c->resident.size();
	free_reg_vectors(c->res_regs);
	c->res_regs.resize(n); c->res_rl.assign(n, 0);
	if (group_reads <= 0) group_reads = n > 0 ? n : 1;
	WM_CUDA_CHECK(cudaEventRecord(e0, 0));
	for (int g0 = 0; g0 < n; g0 += group_reads) {
		const int g1 = std::min(n, g0 + group_reads);
		std::vector<const wm_read*> reads(g1 - g0);
		for (int i = g0; i < g1; ++i) reads[i - g0] = &c->resident[i];
		std::vector<std::vector<wm_reg1_t>> regs; std::vector<int> rl, fg;
		map_lanes(c, opt, reads, regs, rl, fg, n_threads);
		for (int i = g0; i < g1; ++i) { c->res_regs[i].swap(regs[i - g0]); c->res_rl[i] = rl[i - g0]; }
	}
	WM_CUDA_CHECK(cudaEventRecord(e1, 0));
	WM_CUDA_CHECK(cudaEventSynchronize(e1));
	float f = 0.f;
	WM_CUDA_CHECK(cudaEventElapsedTime(&f, e0, e1));
	*ms = f;
	return 0;
}

// bench: the records of the last resident pass, formatted for the first n_first reads in input order (parity check of the timed path)
extern "C" int wm_bench_write(wm_gpu_ctx_s *c, const wm_mapopt_t *opt, int n_first, const char *out_fn)
{
	FILE *out = fopen(out_fn, "wb");
	if (!out) return -1;
	const int n = std::min<int>(n_first, (int)c->res_regs.size());
	std::string buf;
	for (int i = 0; i < n; ++i) {
		buf.clear();
		format_read(buf, &c->hidx, opt->flag, &c->resident[i], (int)c->res_regs[i].size(), c->res_regs[i].data(), c->res_rl[i]);
		fwrite(buf.data(), 1, buf.size(), out);
	}
	fclose(out);
	return n;
}

// The records wm_gpu_map_batch returned, formatted in input order with the writer wm_map_file uses (mm_write_paf3 / mm_write_sam3)
extern "C" int wm_format_batch(const wm_gpu_ctx_s *c, const wm_mapopt_t *opt, int n_seq, const char *const *names, const char *const *seqs, const int32_t *lens,
                               const int32_t *n_reg, wm_reg1_t *const *reg, const int32_t *rep_len, const char *out_fn)
{
	FILE *out = fopen(out_fn, "wb");
	if (!out) return -1;
	std::string buf;
	wm_read t;
	for (int i = 0; i < n_seq; ++i) {
		t.name = names && names[i] ? names[i] : "";
		t.seq.assign(seqs[i], lens[i]);
		buf.clear();
		format_read(buf, &c->hidx, opt->flag, &t, n_reg[i], reg[i], rep_len[i]);
		fwrite(buf.data(), 1, buf.size(), out);
	}
	fclose(out);
	return 0;
}

extern "C" void wm_dump_timers(void) { wmh::g_timers.dump(stderr); wmh::g_timers.reset(); }

// ---- one-time index fan-out: the flattened index as one relocatable blob ----
// Rank 0 builds the index, the blob travels GPU-to-GPU with one NCCL broadcast (torch.distributed in bench.py) and
// every other rank re-creates its context from it.  Layout: 8 x uint64 header, then the arrays, each 8-byte aligned.
static inline size_t pad8(size_t x) { return (x + 7) & ~(size_t)7; }

// the host copies of keys / pos_off / pos exist only when the index came through wm_gpu_idx_upload; an index built on the
// device (wm_index_build) is fetched when the blob is first asked for
static void fetch_index_arrays(wm_gpu_ctx_s *c)
{
	if (!c->keys.empty() || c->n_keys == 0) return;
	const uint64_t *dk, *dpo, *dp;
	gpu_backend_index_arrays(c->be, &dk, &dpo, &dp);
	c->keys.resize(c->n_keys); c->pos_off.resize(c->n_keys + 1); c->pos.resize(c->n_pos);
	WM_CUDA_CHECK(cudaMemcpy(c->keys.data(), dk, sizeof(uint64_t) * c->n_keys, cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(c->pos_off.data(), dpo, sizeof(uint64_t) * (c->n_keys + 1), cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(c->pos.data(), dp, sizeof(uint64_t) * c->n_pos, cudaMemcpyDeviceToHost));
}

extern "C" int64_t wm_idx_blob_size(const wm_gpu_ctx_s *c_)
{
	wm_gpu_ctx_s *c = const_cast<wm_gpu_ctx_s*>(c_);
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_idx_blob_size: the fan-out of a multi-part index is not supported\n"); return -1; }
	fetch_index_arrays(c);
	const wm_host_idx &H = c->hidx;
	size_t names = 0;
	for (auto &s : H.name) names += s.size() + 1;
	return (int64_t)(8 * 8 + pad8(H.len.size() * 4) + H.offset.size() * 8 + pad8(names) + pad8(H.S.size() * 4) + c->keys.size() * 8 +
	                 c->pos_off.size() * 8 + c->pos.size() * 8 + pad8(c->bloom.size()));
}

extern "C" int wm_idx_blob_write(const wm_gpu_ctx_s *c_, uint8_t *buf)
{
	wm_gpu_ctx_s *c = const_cast<wm_gpu_ctx_s*>(c_);
	if (is_multi(c)) { fprintf(stderr, "[ERROR] wm_idx_blob_write: the fan-out of a multi-part index is not supported\n"); return -1; }
	fetch_index_arrays(c);
	const wm_host_idx &H = c->hidx;
	size_t names = 0;
	for (auto &s : H.name) names += s.size() + 1;
	uint64_t *h = (uint64_t*)buf;
	h[0] = 0x31584449424d57ULL; /* "WMBIDX1" */ h[1] = (uint64_t)H.k << 32 | (uint64_t)(uint16_t)H.flag << 16 | (uint32_t)H.w; h[2] = H.len.size(); h[3] = names;
	h[4] = H.S.size(); h[5] = c->keys.size(); h[6] = c->pos.size(); h[7] = c->bloom_bits;
	uint8_t *p = buf + 64;
	memcpy(p, H.len.data(), H.len.size() * 4); p += pad8(H.len.size() * 4);
	memcpy(p, H.offset.data(), H.offset.size() * 8); p += H.offset.size() * 8;
	{ uint8_t *q = p; for (auto &s : H.name) { memcpy(q, s.c_str(), s.size() + 1); q += s.size() + 1; } p += pad8(names); }
	memcpy(p, H.S.data(), H.S.size() * 4); p += pad8(H.S.size() * 4);
	memcpy(p, c->keys.data(), c->keys.size() * 8); p += c->keys.size() * 8;
	memcpy(p, c->pos_off.data(), c->pos_off.size() * 8); p += c->pos_off.size() * 8;
	memcpy(p, c->pos.data(), c->pos.size() * 8); p += c->pos.size() * 8;
	memcpy(p, c->bloom.data(), c->bloom.size());
	return 0;
}

extern "C" wm_gpu_ctx_s *wm_idx_blob_load(const uint8_t *buf, int64_t size, int device)
{
	require_device("wm_idx_blob_load");
	const uint64_t *h = (const uint64_t*)buf;
	if (size < 64 || h[0] != 0x31584449424d57ULL) { fprintf(stderr, "[ERROR] wm_idx_blob_load: bad blob\n"); return 0; }
	const size_t n_seq = h[2], names = h[3], s_words = h[4], n_keys = h[5], n_pos = h[6], bloom_bytes = (size_t)(h[7] / 8);
	{ // every section length comes from the header: the total must be exactly the buffer (a truncated or foreign broadcast is refused)
		const unsigned __int128 need = (unsigned __int128)64 + pad8(n_seq * 4) + (unsigned __int128)n_seq * 8 + pad8(names) + pad8(s_words * 4) +
			(unsigned __int128)n_keys * 8 + ((unsigned __int128)n_keys + 1) * 8 + (unsigned __int128)n_pos * 8 + pad8(bloom_bytes);
		if (need != (unsigned __int128)size) { fprintf(stderr, "[ERROR] wm_idx_blob_load: blob of %lld bytes does not match its header\n", (long long)size); return 0; }
	}
	const uint8_t *p = buf + 64;
	const uint32_t *len = (const uint32_t*)p; p += pad8(n_seq * 4);
	const uint64_t *off = (const uint64_t*)p; p += n_seq * 8;
	const char *nm = (const char*)p, *nm_end = nm + names; p += pad8(names);
	const uint32_t *S = (const uint32_t*)p; p += pad8(s_words * 4);
	const uint64_t *keys = (const uint64_t*)p; p += n_keys * 8;
	const uint64_t *pos_off = (const uint64_t*)p; p += (n_keys + 1) * 8;
	const uint64_t *pos = (const uint64_t*)p; p += n_pos * 8;
	if (pos_off[n_keys] != n_pos) { fprintf(stderr, "[ERROR] wm_idx_blob_load: occurrence table does not match its header\n"); return 0; }
	std::vector<const char*> name_ptr(n_seq);
	for (size_t i = 0; i < n_seq; ++i) {
		const void *z = nm < nm_end ? memchr(nm, 0, (size_t)(nm_end - nm)) : 0;
		if (!z) { fprintf(stderr, "[ERROR] wm_idx_blob_load: sequence name table is truncated\n"); return 0; }
		name_ptr[i] = nm; nm = (const char*)z + 1;
	}
	wm_idx_view_t v;
	// h[1]: k << 32 | flag << 16 | w (w < 256; a blob without flags has zeros there)
	v.k = (int32_t)(h[1] >> 32), v.w = (int32_t)(h[1] & 0xffff), v.n_seq = (int32_t)n_seq;
	v.seq_name = name_ptr.data(), v.seq_len = len, v.seq_offset = off, v.S = S, v.S_words = s_words;
	v.n_keys = (int64_t)n_keys, v.keys = keys, v.pos_off = pos_off, v.pos = pos, v.bloom_bits = h[7], v.bloom_table = p;
	return wm_gpu_idx_upload_flag(&v, (int)(h[1] >> 16 & 0xffff), device);
}
