// CUDA implementation of the device boundary (host_backend.h) for one GPU: resident index, per-batch read
// pool, and the three coarse operations the orchestrator calls.  All buffers are grow-only pools (wm_dbuf)
// sized for a batch; nothing is allocated per read.
#include <string.h>
#include <algorithm>
#include <mutex>
#include <vector>
#include "wm_common.cuh"
#include "scan.cuh"
#include "sketch.cuh"
#include "seed.cuh"
#include "chain.cuh"
#include "bed_junc.cuh"
#include "gpu_backend.h"
#include "host_timers.h"

// from ksw_extd2.cu / ksw_ll.cu
// (wm_extd2_ws / wm_extd2_plan / wm_extd2_launch are declared in wm_common.cuh)
struct wm_ll_job { int64_t q_off, t_off; int64_t s_off; int32_t qlen, tlen; };
void wm_ksw_ll_launch(const wm_ll_job *d_jobs, int n, const uint8_t *d_seq, const int8_t *d_mat, int gapo, int gape, int32_t *d_scratch, int32_t *d_out, cudaStream_t st);

using namespace wmh;

static_assert(WM_SKIP_NO_DIAG == SKIP_NO_DIAG && WM_SKIP_NO_DUAL == SKIP_NO_DUAL && WM_SKIP_FOR_ONLY == SKIP_FOR_ONLY &&
              WM_SKIP_REV_ONLY == SKIP_REV_ONLY && WM_SKIP_NAME_EQ == SKIP_NAME_EQ, "seed filter bits");
static_assert(WM_SDUST_MAX_T == SDUST_MAX_T, "-T range");

// ---- small data-movement kernels ----
// Masked copy of a window (src/map.c:795-801: covered bases become ambiguous) as a packed sequence of its own: one thread
// per 32 bases takes the unaligned source windows and sets the flags of the covered bases.
__global__ void wm_mask_pack_kernel(const wm_pkseq seq, const wm_mask_task *__restrict__ tasks, const int64_t *__restrict__ goff, int n_tasks,
                                    const int32_t *__restrict__ mask_pool, int64_t n_groups, uint32_t *__restrict__ pk_out, uint32_t *__restrict__ nm_out)
{
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n_groups) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (goff[m] <= g) lo = m; else hi = m; }
	uint64_t v; uint32_t m;
	wm_pk_mask32(seq, tasks[lo], (int)(g - goff[lo]) * 32, mask_pool, &v, &m);
	((uint2*)pk_out)[g] = make_uint2((uint32_t)v, (uint32_t)(v >> 32));
	nm_out[g] = m;
}

struct wm_cat_task { int64_t pre_off, seed_off, dst_off; int32_t n_pre, n_seed; };

__global__ void wm_concat_kernel(const wm_cat_task *__restrict__ tasks, const int64_t *__restrict__ toff, int n_tasks, const wm128_dev *__restrict__ pre,
                                 const wm128_dev *__restrict__ seeds, wm128_dev *__restrict__ dst, int64_t n)
{ // a_whole = [a ; a_remaining] (src/map.c:818-828)
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (toff[m] <= g) lo = m; else hi = m; }
	const wm_cat_task T = tasks[lo];
	const int64_t p = g - toff[lo];
	dst[T.dst_off + p] = p < T.n_pre ? pre[T.pre_off + p] : seeds[T.seed_off + (p - T.n_pre)];
}

__global__ void wm_compact_chain_kernel(const int64_t *__restrict__ src_off, const int64_t *__restrict__ nb_off, const int64_t *__restrict__ nu_off, int n_tasks,
                                        const wm128_dev *__restrict__ a, const uint64_t *__restrict__ u, wm128_dev *__restrict__ b_out, uint64_t *__restrict__ u_out)
{ // one warp per task copies the meaningful prefix of its chain output
	const int task = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (task >= n_tasks) return;
	const int64_t so = src_off[task], bo = nb_off[task], uo = nu_off[task];
	const int64_t nb = nb_off[task + 1] - bo, nu = nu_off[task + 1] - uo;
	for (int64_t i = lane; i < nb; i += 32) b_out[bo + i] = a[so + i];
	for (int64_t i = lane; i < nu; i += 32) u_out[uo + i] = u[so + i];
}

__global__ void wm_ncigar_kernel(const wm_dp_job *__restrict__ jobs, const wm_extz_dev *__restrict__ ez, int n_jobs, int32_t *__restrict__ nc)
{ // CIGAR length of every job (what fits its buffer: an overflow is reported by the host from ez.n_cigar)
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_jobs) return;
	const int n = ez[i].n_cigar;
	nc[i] = n < jobs[i].cig_cap ? n : jobs[i].cig_cap;
}

__global__ void wm_compact_cigar_kernel(const wm_dp_job *__restrict__ jobs, const wm_extz_dev *__restrict__ ez, const int64_t *__restrict__ out_off, int n_jobs,
                                        const uint32_t *__restrict__ cig, uint32_t *__restrict__ out)
{
	const int job = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (job >= n_jobs) return;
	const int64_t o = out_off[job], n = out_off[job + 1] - o, s = jobs[job].cig_off;
	for (int64_t i = lane; i < n; i += 32) out[o + i] = cig[s + i];
}

namespace wmh {

struct GpuBackendImpl {
	int device;
	cudaStream_t st;
	wm_idx_dev ix;
	wm_bloom_dev bf;
	const wm_host_idx *hidx;
	// batch state
	std::vector<int64_t> read_off; // host
	wm_dbuf ascii, pk, nm, d_read_off, d_src_off; // the batch's reads: ASCII as uploaded, then the packed pool (pkseq.cuh)
	int64_t n_bases;
	const char *resident_pool = 0;         // device ASCII of reads that carry a dev_off (bench: inputs resident in HBM)
	char *h_stage = 0; size_t h_stage_cap = 0; // pinned staging buffer of begin_batch
	// workspaces
	wm_sketch_ws sk; wm_seed_ws sd, sd2; wm_chain_ws ch; wm_extd2_ws dpws;
	int sdust_T = 0; wm_sdust_ws sdw; // -T (0: off; sdw is then never touched)
	bool heap_sort = false;            // --heap-sort=yes
	wm_dbuf masked_pk, masked_nm, mask_tasks, mask_toff, mask_pool, qlen_buf, skip_buf, pre_buf, cat_tasks, cat_toff, cat_a, set_id, off_buf, nb_off, nu_off, b_out, u_out;
	wm_dbuf nc_buf, scan_tmp, coop_ids, g_jobs, g_joff, seq_pool, dp_jobs, bt, ez, cig, cig_off, cig_out, ll_jobs, ll_scr, ll_out, mat;
	// host result pools
	std::vector<uint32_t> h_mzpos; std::vector<int64_t> h_mz_off; std::vector<int32_t> h_rep;
	std::vector<uint8_t> h_mzspan; wm_dbuf mz_span; // HPC index only: the minimizers' spans
	wm_hbuf<uint64_t> h_u; wm_hbuf<wm_pair_t> h_b; std::vector<int32_t> h_nu; std::vector<int64_t> h_nb; // (the big ones: page-locked)
	wm_hbuf<uint32_t> h_cig; wm_hbuf<wm_extz_dev> h_ez; wm_hbuf<int32_t> h_zd; wm_dbuf zd;
	size_t bt_budget;
	bool owns_index = false; // the lane that uploaded the index frees it; clones only borrow the pointers
	// the index this backend was created with (ix / bf / hidx above are the one it maps against, which gpu_backend_bind
	// may point at another index of the same context: one part of a multi-part index)
	wm_idx_dev own_ix; wm_bloom_dev own_bf; const wm_host_idx *own_hidx;
	// junction intervals of the bound index and of the own one (n_seq 0: none; gpu_backend_set_junc), and the annotation of a
	// splice DP launch's targets, parallel to seq_pool
	wm_junc_dev jx = {}, own_jx = {};
	wm_dbuf junc_pool, junc_wins;
};

class GpuBackend : public Backend {
public:
	GpuBackendImpl g;
	GpuBackend() {}
	~GpuBackend()
	{ // workspaces (wm_dbuf members) free themselves; here: the stream, the pinned staging buffer and, for the owner lane, the index
		cudaSetDevice(g.device);
		if (g.st) { cudaStreamSynchronize(g.st); }
		if (g.dpws.fill_st) cudaStreamSynchronize(g.dpws.fill_st);
		if (g.h_stage) cudaFreeHost(g.h_stage);
		if (g.owns_index) {
			const wm_idx_dev &x = g.own_ix;
			cudaFree((void*)x.keys); cudaFree((void*)x.pos_off); cudaFree((void*)x.pos); cudaFree((void*)x.S);
			cudaFree((void*)x.ht_key); cudaFree((void*)x.ht_val); cudaFree((void*)g.own_bf.table);
			cudaFree((void*)x.seq_len); cudaFree((void*)x.name_rank);
			wm_junc_free(&g.own_jx);
		}
		if (g.st) cudaStreamDestroy(g.st);
		// this thread's workspace allocations must not go on to the stream just destroyed (wm_dbuf_use_stream)
		if (wm_dbuf_stream == g.st) wm_dbuf_stream = 0, wm_dbuf_async = false;
	}
	void begin_batch(const std::vector<const wm_read*> &reads) override;
	void set_resident_pool(const char *device_ascii) override { g.resident_pool = device_ascii; }
	bool set_sdust(int T) override { g.sdust_T = T > 0 ? T : 0; return true; }
	bool set_heap_sort(bool on) override { g.heap_sort = on; return true; }
	void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) override;
	void run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res) override;
	void run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res) override;
	void end_batch() override {}
};

void GpuBackend::begin_batch(const std::vector<const wm_read*> &reads)
{
	WM_CUDA_CHECK(cudaSetDevice(g.device));
	wm_dbuf_use_stream(g.st);
	const int n = (int)reads.size();
	g.read_off.assign(n + 1, 0);
	for (int i = 0; i < n; ++i) g.read_off[i + 1] = g.read_off[i] + (int64_t)reads[i]->seq.size();
	g.n_bases = g.read_off[n];
	uint32_t *d_pk = (uint32_t*)g.pk.need(sizeof(uint32_t) * wm_pk_words(g.n_bases)), *d_nm = (uint32_t*)g.nm.need(sizeof(uint32_t) * wm_nm_words(g.n_bases));
	int64_t *d_off = (int64_t*)g.d_read_off.need(sizeof(int64_t) * (n + 1));
	bool resident = g.resident_pool != 0;
	for (int i = 0; i < n && resident; ++i) resident = reads[i]->dev_off >= 0;
	WM_CUDA_CHECK(wm_memcpy_async(d_off, g.read_off.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, g.st));
	if (resident) { // the bases are in HBM already: gather + pack on the device
		std::vector<int64_t> src(n);
		for (int i = 0; i < n; ++i) src[i] = reads[i]->dev_off;
		int64_t *d_src = (int64_t*)g.d_src_off.need(sizeof(int64_t) * (n + 1));
		WM_CUDA_CHECK(wm_memcpy_async(d_src, src.data(), sizeof(int64_t) * n, cudaMemcpyHostToDevice, g.st));
		wm_pack_gather(g.resident_pool, d_src, d_off, n, g.n_bases, d_pk, d_nm, g.st);
		wm_stream_sync(g.st); // src[] is a local
	} else { // one host staging buffer (pinned), one copy
		if ((size_t)g.n_bases + 16 > g.h_stage_cap) {
			if (g.h_stage) WM_CUDA_CHECK(cudaFreeHost(g.h_stage));
			g.h_stage_cap = (size_t)(g.n_bases + 16) * 5 / 4;
			WM_CUDA_CHECK(cudaMallocHost((void**)&g.h_stage, g.h_stage_cap));
		}
		wm_stream_sync(g.st); // the previous batch's copy out of the staging buffer
		for (int i = 0; i < n; ++i)
			if (!reads[i]->seq.empty()) memcpy(g.h_stage + g.read_off[i], reads[i]->seq.data(), reads[i]->seq.size());
		char *d_ascii = (char*)g.ascii.need(g.n_bases + 16);
		if (g.n_bases > 0) WM_CUDA_CHECK(wm_memcpy_async(d_ascii, g.h_stage, g.n_bases, cudaMemcpyHostToDevice, g.st));
		wm_pack_ascii(d_ascii, g.n_bases, d_pk, d_nm, g.st);
	}
}

void GpuBackend::seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out)
{
	WM_CUDA_CHECK(cudaSetDevice(g.device));
	wm_dbuf_use_stream(g.st);
	cudaStream_t st = g.st;
	const int n = (int)tasks.size();
	out.assign(n, SeedOut());
	if (n == 0) return;
	wm_pkseq rd; rd.pk = (const uint32_t*)g.pk.p, rd.nm = (const uint32_t*)g.nm.p;
	double t_mark = Timers::now();
	auto lap = [&](const char *nm) { const double t = Timers::now(); g_timers.add(nm, t - t_mark); t_mark = t; };
	// 1. masked copies
	std::vector<wm_mask_task> mt; std::vector<int64_t> mtoff(1, 0); // mtoff: in groups of 32 bases
	int64_t n_mask_iv = 0, n_pre = 0;
	for (int i = 0; i < n; ++i) {
		const SeedTask &t = tasks[i];
		if (t.flags & SEED_MASKED) {
			wm_mask_task m;
			m.src_off = g.read_off[t.win.read] + t.win.wb, m.dst_off = mtoff.back() * 32, m.mask_off = t.mask_off, m.len = t.win.wl, m.n_mask = t.n_mask;
			mt.push_back(m); mtoff.push_back(mtoff.back() + (t.win.wl + 31) / 32);
			n_mask_iv = std::max<int64_t>(n_mask_iv, t.mask_off + t.n_mask);
		}
		n_pre = std::max<int64_t>(n_pre, t.pre_off + t.n_pre);
	}
	wm_pkseq rd_masked;
	{
		const int64_t nb = mtoff.back() * 32;
		uint32_t *mpk = (uint32_t*)g.masked_pk.need(sizeof(uint32_t) * wm_pk_words(nb)), *mnm = (uint32_t*)g.masked_nm.need(sizeof(uint32_t) * wm_nm_words(nb));
		rd_masked.pk = mpk, rd_masked.nm = mnm;
		if (!mt.empty()) { // the look-ahead words
			WM_CUDA_CHECK(cudaMemsetAsync(mpk + 2 * mtoff.back(), 0, sizeof(uint32_t) * WM_PK_SLACK, st));
			WM_CUDA_CHECK(cudaMemsetAsync(mnm + mtoff.back(), 0xff, sizeof(uint32_t) * WM_PK_SLACK, st));
		}
	}
	if (!mt.empty()) {
		wm_mask_task *d_mt = (wm_mask_task*)g.mask_tasks.need(sizeof(wm_mask_task) * mt.size());
		int64_t *d_mtoff = (int64_t*)g.mask_toff.need(sizeof(int64_t) * mtoff.size());
		int32_t *d_mp = (int32_t*)g.mask_pool.need(sizeof(int32_t) * 2 * (n_mask_iv + 1));
		WM_CUDA_CHECK(wm_memcpy_async(d_mt, mt.data(), sizeof(wm_mask_task) * mt.size(), cudaMemcpyHostToDevice, st));
		WM_CUDA_CHECK(wm_memcpy_async(d_mtoff, mtoff.data(), sizeof(int64_t) * mtoff.size(), cudaMemcpyHostToDevice, st));
		WM_CUDA_CHECK(wm_memcpy_async(d_mp, mask_pool, sizeof(int32_t) * 2 * n_mask_iv, cudaMemcpyHostToDevice, st));
		wm_count_launch(); wm_mask_pack_kernel<<<(unsigned)((mtoff.back() + 127) / 128), 128, 0, st>>>(rd, d_mt, d_mtoff, (int)mt.size(), d_mp, mtoff.back(), (uint32_t*)rd_masked.pk, (uint32_t*)rd_masked.nm);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	lap("seed.a_mask");
	// 2. sketch: tasks that sketch something.  The masked copies live in another buffer, so two passes.
	std::vector<int> sk_of(n, -1);       // task -> index among the sketched tasks
	std::vector<wm_sk_task> skt_plain, skt_mask;
	std::vector<int> plain_ids, mask_ids;
	{
		size_t mi_ = 0;
		for (int i = 0; i < n; ++i) {
			const SeedTask &t = tasks[i];
			if (t.flags & SEED_NO_SKETCH) continue;
			wm_sk_task s; s.len = t.win.wl, s.rid = 0;
			if (t.flags & SEED_MASKED) { s.seq_off = mt[mi_++].dst_off; skt_mask.push_back(s); mask_ids.push_back(i); }
			else { s.seq_off = g.read_off[t.win.read] + t.win.wb; skt_plain.push_back(s); plain_ids.push_back(i); }
		}
	}
	// per task results gathered into one anchor array `A` with offsets `a_off`
	const int k = g.ix.k, w = g.ix.w;
	std::vector<int64_t> seed_cnt(n, 0), seed_src(n, 0); // per task: number of seed anchors and their offset in the pass's anchor array
	std::vector<int> seed_pass(n, -1);
	std::vector<int64_t> h_mz_off_all(n + 1, 0);
	g.h_mzpos.clear(); g.h_rep.assign(n, 0);
	std::vector<int64_t> mz_cnt(n, 0), mz_src(n, 0);
	wm128_dev *d_seed_a[2] = {0, 0};
	wm_seed_ws *sdp[2] = { &g.sd, 0 };
	sdp[1] = &g.sd2; // second seed workspace for the masked pass (kept until chaining is done)
	std::vector<uint32_t> pass_mzpos[2]; std::vector<int64_t> pass_mzoff[2];
	const bool hpc = (g.hidx->flag & WM_I_HPC) != 0;
	std::vector<uint8_t> pass_mzspan[2];
	for (int pass = 0; pass < 2; ++pass) {
		std::vector<wm_sk_task> &skt = pass == 0 ? skt_plain : skt_mask;
		std::vector<int> &ids = pass == 0 ? plain_ids : mask_ids;
		const int ns = (int)skt.size();
		if (ns == 0) continue;
		int64_t n_mz = 0;
		{
			wm_dust_view dv, *dust = 0;
			if (g.sdust_T > 0) { // the regions of the sequences this pass sketches (stage-1 windows, masked copies or whole reads)
				WM_TIMED("seed.sdust");
				wm_sdust_run(&g.sdw, pass == 0 ? rd : rd_masked, skt.data(), ns, g.sdust_T, 64, &dv, st);
				dust = &dv;
			}
			WM_TIMED("seed.sketch");
			if (hpc) wm_sketch_run_hpc(&g.sk, g.bf, pass == 0 ? rd : rd_masked, skt.data(), ns, w, k, &n_mz, st, dust);
			else wm_sketch_run(&g.sk, g.bf, pass == 0 ? rd : rd_masked, skt.data(), ns, w, k, &n_mz, st, dust);
		}
		WM_TIMED("seed.lookup_sort");
		std::vector<int32_t> qlen(ns);
		for (int i = 0; i < ns; ++i) qlen[i] = skt[i].len;
		int32_t *d_qlen = (int32_t*)g.qlen_buf.need(sizeof(int32_t) * ns);
		WM_CUDA_CHECK(wm_memcpy_async(d_qlen, qlen.data(), sizeof(int32_t) * ns, cudaMemcpyHostToDevice, st));
		std::vector<uint2> skip(ns); // the seed filter of the pass' tasks; none when no task has a bit set
		bool any_skip = false;
		for (int i = 0; i < ns; ++i) { skip[i] = make_uint2(tasks[ids[i]].skip, tasks[ids[i]].name_lt); any_skip |= skip[i].x != 0; }
		uint2 *d_skip = 0;
		if (any_skip) {
			d_skip = (uint2*)g.skip_buf.need(sizeof(uint2) * ns);
			WM_CUDA_CHECK(wm_memcpy_async(d_skip, skip.data(), sizeof(uint2) * ns, cudaMemcpyHostToDevice, st));
		}
		std::vector<int64_t> a_off(ns + 1);
		wm_seed_run(sdp[pass], g.ix, (const wm128_dev*)g.sk.mz.p, (const int64_t*)g.sk.mz_off.p, n_mz, ns, d_qlen, max_occ, a_off.data(), st, d_skip, g.heap_sort);
		d_seed_a[pass] = (wm128_dev*)sdp[pass]->a.p;
		// small per-task results
		std::vector<int32_t> rep(ns);
		pass_mzoff[pass].assign(ns + 1, 0); pass_mzpos[pass].resize(n_mz);
		WM_CUDA_CHECK(wm_memcpy_async(rep.data(), sdp[pass]->rep_len.p, sizeof(int32_t) * ns, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(wm_memcpy_async(pass_mzoff[pass].data(), g.sk.mz_off.p, sizeof(int64_t) * (ns + 1), cudaMemcpyDeviceToHost, st));
		if (n_mz > 0) WM_CUDA_CHECK(wm_memcpy_async(pass_mzpos[pass].data(), sdp[pass]->mini_pos.p, sizeof(uint32_t) * n_mz, cudaMemcpyDeviceToHost, st));
		if (hpc && n_mz > 0) { // the spans vary: mm_est_err averages them (src/esterr.c:37-39)
			uint8_t *d_sp = (uint8_t*)g.mz_span.need(n_mz);
			wm_mz_spans((const wm128_dev*)g.sk.mz.p, n_mz, d_sp, st);
			pass_mzspan[pass].resize(n_mz);
			WM_CUDA_CHECK(wm_memcpy_async(pass_mzspan[pass].data(), d_sp, n_mz, cudaMemcpyDeviceToHost, st));
		}
		wm_stream_sync(st);
		if (g.sdust_T > 0) wm_sdust_check(&g.sdw);
		if (g.heap_sort) wm_seed_heap_check();
		for (int i = 0; i < ns; ++i) {
			const int t = ids[i];
			g.h_rep[t] = rep[i];
			seed_cnt[t] = a_off[i + 1] - a_off[i], seed_src[t] = a_off[i], seed_pass[t] = pass;
			mz_cnt[t] = pass_mzoff[pass][i + 1] - pass_mzoff[pass][i], mz_src[t] = pass_mzoff[pass][i];
		}
	}
	lap("seed.b_sketch_seed");
	// 3. final anchor arrays: [pre ; seeds] per task
	std::vector<int64_t> f_off(n + 1, 0);
	std::vector<wm_cat_task> ct(n);
	std::vector<uint8_t> set_id(n);
	bool any_pre = false, any_mask_pass = !skt_mask.empty();
	for (int i = 0; i < n; ++i) {
		const SeedTask &t = tasks[i];
		f_off[i + 1] = f_off[i] + t.n_pre + seed_cnt[i];
		set_id[i] = (uint8_t)t.chain_set;
		any_pre |= t.n_pre > 0;
	}
	const int64_t n_f = f_off[n];
	wm128_dev *d_A;
	int64_t *d_foff = (int64_t*)g.off_buf.need(sizeof(int64_t) * (n + 1));
	WM_CUDA_CHECK(wm_memcpy_async(d_foff, f_off.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, st));
	if (!any_pre && !any_mask_pass) {
		d_A = d_seed_a[0]; // the plain pass' array already has exactly this layout (tasks in order, no gaps)
		if (d_A == 0) d_A = (wm128_dev*)g.cat_a.need(16);
	} else {
		d_A = (wm128_dev*)g.cat_a.need(sizeof(wm128_dev) * (n_f + 1));
		wm128_dev *d_pre = (wm128_dev*)g.pre_buf.need(sizeof(wm128_dev) * (n_pre + 1));
		if (n_pre > 0) WM_CUDA_CHECK(wm_memcpy_async(d_pre, pre_pool, sizeof(wm128_dev) * n_pre, cudaMemcpyHostToDevice, st));
		// tasks fed from the plain pass and from the masked pass need different source arrays: two launches
		for (int pass = 0; pass < 2; ++pass) {
			std::vector<wm_cat_task> c2; std::vector<int64_t> toff(1, 0);
			for (int i = 0; i < n; ++i) {
				const SeedTask &t = tasks[i];
				const bool mine = seed_pass[i] == pass || (seed_pass[i] < 0 && pass == 0);
				if (!mine) continue;
				wm_cat_task c;
				c.pre_off = t.pre_off, c.n_pre = t.n_pre, c.seed_off = seed_src[i], c.n_seed = (int32_t)seed_cnt[i], c.dst_off = f_off[i];
				if (c.n_pre + c.n_seed == 0) continue;
				c2.push_back(c); toff.push_back(toff.back() + c.n_pre + c.n_seed);
			}
			if (c2.empty()) continue;
			wm_cat_task *d_ct = (wm_cat_task*)g.cat_tasks.need(sizeof(wm_cat_task) * c2.size());
			int64_t *d_toff = (int64_t*)g.cat_toff.need(sizeof(int64_t) * toff.size());
			WM_CUDA_CHECK(wm_memcpy_async(d_ct, c2.data(), sizeof(wm_cat_task) * c2.size(), cudaMemcpyHostToDevice, st));
			WM_CUDA_CHECK(wm_memcpy_async(d_toff, toff.data(), sizeof(int64_t) * toff.size(), cudaMemcpyHostToDevice, st));
			const wm128_dev *src = d_seed_a[pass] ? d_seed_a[pass] : d_A;
			wm_count_launch(); wm_concat_kernel<<<(unsigned)((toff.back() + 255) / 256), 256, 0, st>>>(d_ct, d_toff, (int)c2.size(), d_pre, src, d_A, toff.back());
			WM_CUDA_CHECK(cudaGetLastError());
			wm_stream_sync(st); // c2/toff are reused by the next pass
		}
		// sort #3 (src/map.c:831): only arrays that really merged two sorted runs can change
		std::vector<int64_t> s_off(n + 1);
		{
			// sort only the tasks with both parts (the others are already sorted), all of them in one set of launches
			std::vector<int32_t> which;
			for (int i = 0; i < n; ++i) if (tasks[i].n_pre > 0 && seed_cnt[i] > 0) which.push_back(i);
			if (!which.empty()) {
				wm_anchor_sort_run(&g.sd, d_A, d_foff, f_off.data(), n, st, which.data(), (int)which.size());
				wm_stream_sync(st);
			}
		}
	}
	lap("seed.c_concat_sort3");
	// 4. chaining
	uint8_t *d_set = (uint8_t*)g.set_id.need(n);
	WM_CUDA_CHECK(wm_memcpy_async(d_set, set_id.data(), n, cudaMemcpyHostToDevice, st));
	wm_chain_params2 PP;
	for (int s = 0; s < 2; ++s) {
		wm_chain_params &P = PP.p[s];
		P.max_dist_x = cp[s].max_dist_x, P.min_dist_x = cp[s].min_dist_x, P.max_dist_y = cp[s].max_dist_y, P.bw = cp[s].bw;
		P.max_skip = cp[s].max_skip, P.max_iter = cp[s].max_iter, P.min_cnt = cp[s].min_cnt, P.min_sc = cp[s].min_sc, P.gap_scale = cp[s].gap_scale;
	}
	PP.is_cdna = cp[0].is_cdna;
	double t_chain0 = Timers::now();
	wm_chain_run(&g.ch, d_A, d_foff, f_off.data(), n, PP, d_set, st);
	g.h_nu.assign(n, 0); g.h_nb.assign(n, 0);
	WM_CUDA_CHECK(wm_memcpy_async(g.h_nu.data(), g.ch.n_u.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
	WM_CUDA_CHECK(wm_memcpy_async(g.h_nb.data(), g.ch.n_b.p, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	g_timers.add("seed.chain", Timers::now() - t_chain0);
	lap("seed.d_chain");
	std::vector<int64_t> nb_off(n + 1, 0), nu_off(n + 1, 0);
	for (int i = 0; i < n; ++i) nb_off[i + 1] = nb_off[i] + g.h_nb[i], nu_off[i + 1] = nu_off[i] + g.h_nu[i];
	int64_t *d_nb = (int64_t*)g.nb_off.need(sizeof(int64_t) * (n + 1)), *d_nu = (int64_t*)g.nu_off.need(sizeof(int64_t) * (n + 1));
	WM_CUDA_CHECK(wm_memcpy_async(d_nb, nb_off.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_nu, nu_off.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, st));
	wm128_dev *d_bo = (wm128_dev*)g.b_out.need(sizeof(wm128_dev) * (nb_off[n] + 1));
	uint64_t *d_uo = (uint64_t*)g.u_out.need(sizeof(uint64_t) * (nu_off[n] + 1));
	wm_count_launch(); wm_compact_chain_kernel<<<(unsigned)(((int64_t)n * 32 + 127) / 128), 128, 0, st>>>(d_foff, d_nb, d_nu, n, d_A, (const uint64_t*)g.ch.u2.p, d_bo, d_uo);
	WM_CUDA_CHECK(cudaGetLastError());
	g.h_b.clear(); g.h_u.clear(); // (nothing to carry over if the pools have to grow)
	g.h_b.resize(nb_off[n] + 1); g.h_u.resize(nu_off[n] + 1);
	if (nb_off[n] > 0) WM_CUDA_CHECK(wm_memcpy_async(g.h_b.data(), d_bo, sizeof(wm128_dev) * nb_off[n], cudaMemcpyDeviceToHost, st));
	if (nu_off[n] > 0) WM_CUDA_CHECK(wm_memcpy_async(g.h_u.data(), d_uo, sizeof(uint64_t) * nu_off[n], cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	lap("seed.e_compact_d2h");
	// 5. per task views
	g.h_mz_off.assign(n + 1, 0);
	for (int i = 0; i < n; ++i) g.h_mz_off[i + 1] = g.h_mz_off[i] + mz_cnt[i];
	g.h_mzpos.resize(g.h_mz_off[n] + 1);
	for (int i = 0; i < n; ++i)
		if (mz_cnt[i] > 0) memcpy(&g.h_mzpos[g.h_mz_off[i]], &pass_mzpos[seed_pass[i]][mz_src[i]], sizeof(uint32_t) * mz_cnt[i]);
	if (hpc) {
		g.h_mzspan.resize(g.h_mz_off[n] + 1);
		for (int i = 0; i < n; ++i)
			if (mz_cnt[i] > 0) memcpy(&g.h_mzspan[g.h_mz_off[i]], &pass_mzspan[seed_pass[i]][mz_src[i]], mz_cnt[i]);
	}
	for (int i = 0; i < n; ++i) {
		SeedOut &o = out[i];
		o.rep_len = g.h_rep[i];
		o.n_mz = (int32_t)mz_cnt[i], o.mz_pos = g.h_mzpos.data() + g.h_mz_off[i];
		o.mz_span = hpc ? g.h_mzspan.data() + g.h_mz_off[i] : 0;
		o.n_u = g.h_nu[i], o.u = g.h_u.data() + nu_off[i];
		o.n_b = g.h_nb[i], o.b = g.h_b.data() + nb_off[i];
	}
	lap("seed.f_views");
}

static inline wm_gather_job make_gather(const GpuBackendImpl &g, const SeqRef &s, const MapWin &w, int64_t dst_off)
{
	wm_gather_job j;
	j.len = s.len, j.reversed = s.reversed, j.pad = 0, j.dst_off = dst_off;
	if (s.kind == SEQ_Q0) j.kind = 0, j.src_off = g.read_off[w.read] + w.wb + s.off;
	// base o of strand 1 of the window is the complement of base wl - 1 - o of its strand 0 (src/align.c:874-876)
	else if (s.kind == SEQ_Q1) j.kind = 2, j.src_off = g.read_off[w.read] + w.wb + (w.wl - 1 - s.off);
	else j.kind = 1, j.src_off = (int64_t)g.hidx->offset[s.rid] + s.off;
	return j;
}

// query / target slices of a job -> gather descriptors; every slice starts on a 16-byte boundary of the pool
static inline void add_gather(std::vector<wm_gather_job> &gj, std::vector<int64_t> &joff, const GpuBackendImpl &g, const SeqRef &s, const MapWin &w, int64_t *pool_off)
{
	gj.push_back(make_gather(g, s, w, *pool_off));
	*pool_off += (s.len + 15) & ~15;
	joff.push_back(*pool_off);
}

// DP sequences out of the packed pools: one thread writes 16 bytes of 0..4 codes (one 128-bit store) from one unaligned
// window -- 32 bits of the read pool or 64 bits of the 4-bit reference -- read forwards or backwards.  Slices start on
// 16-byte boundaries of `dst` and are zero padded to one (the fill kernel stages them with bulk copies).
__global__ void wm_gather2_kernel(const wm_gather_job *__restrict__ jobs, const int64_t *__restrict__ joff, int n_jobs, const wm_pkseq rd,
                                  const uint32_t *__restrict__ S, uint8_t *__restrict__ dst, int64_t n16)
{
	const int64_t gidx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (gidx >= n16) return;
	const int64_t byte0 = gidx * 16;
	int lo = 0, hi = n_jobs;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (joff[m] <= byte0) lo = m; else hi = m; }
	uint32_t out[4];
	wm_pk_gather16(jobs[lo], (int)(byte0 - joff[lo]), rd, S, out);
	((uint4*)dst)[gidx] = make_uint4(out[0], out[1], out[2], out[3]);
}

void GpuBackend::run_dp(const std::vector<DpJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<DpRes> &res)
{
	WM_CUDA_CHECK(cudaSetDevice(g.device));
	wm_dbuf_use_stream(g.st);
	cudaStream_t st = g.st;
	const int n = (int)jobs.size();
	const double t_setup0 = Timers::now();
	res.assign(n, DpRes());
	g.h_cig.clear();
	if (n == 0) return;
	wm_pkseq rd; rd.pk = (const uint32_t*)g.pk.p, rd.nm = (const uint32_t*)g.nm.p;
	wm_dp_params P;
	if (sc.splice) wm_dp_params_init_splice(&P, sc.mat, sc.q, sc.e, sc.q2, sc.noncan, sc.junc_bonus);
	else wm_dp_params_init(&P, sc.mat, sc.q, sc.e, sc.q2, sc.e2);
	// a splice job is ksw_exts2: unbanded (w = -1), and its global state slice, when it needs one, is its own (wm_extd2_plan)
	auto job_w = [&](const DpJob &J) { return sc.splice ? -1 : J.w; };
	auto job_bytes = [&](const DpJob &J) { return wm_extd2_bt_bytes(J.q.len, J.t.len, job_w(J)) + (sc.splice ? wm_exts2_scratch_bytes(J.t.len) : 0); };
	static int coop_on = -1; // WM_DP_COOP=0: every job on one warp (for comparison)
	if (coop_on < 0) { const char *e = getenv("WM_DP_COOP"); coop_on = (e && *e == '0') ? 0 : 1; if (getenv("WM_DP_V1") && *getenv("WM_DP_V1") == '1') coop_on = 0; }
	std::vector<int64_t> cig_base(n + 1, 0); // offsets into h_cig, by execution slot
	std::vector<int> slot_of(n, 0);           // job -> execution slot (jobs of a chunk run sorted by size)
	g.h_ez.clear(); g.h_zd.clear();
	g.h_ez.resize(n); g.h_zd.resize(5 * (size_t)n);
	std::vector<uint32_t> chunk_cig;
	g_timers.add("dp.setup", Timers::now() - t_setup0);
	int done = 0;
	while (done < n) {
		// a chunk of jobs whose backtrack matrices fit the budget
		size_t bt_bytes = 0; int end = done; int64_t cig_cap = 0, pool = 0; int max_tlen = 0, max_qlen = 0;
		while (end < n) {
			const DpJob &J = jobs[end];
			size_t b = job_bytes(J);
			if (end > done && bt_bytes + b > g.bt_budget) break;
			bt_bytes += b; cig_cap += J.q.len + J.t.len + 2; pool += J.q.len + J.t.len; max_tlen = std::max(max_tlen, J.t.len); max_qlen = std::max(max_qlen, J.q.len);
			++end;
		}
		const int m = end - done;
		double tp0 = Timers::now();
		std::vector<wm_gather_job> gj(2 * (size_t)m); std::vector<int64_t> joff(2 * (size_t)m + 1, 0); std::vector<wm_dp_job> dj(m);
		int64_t pool_off = 0, p_off = 0, c_off = 0;
		double prof_bytes = 0;
		// CTAs are dispatched in array order, four consecutive jobs each: biggest first, so that a CTA's jobs are of similar
		// size and the tail of the launch is made of small jobs
		// (stable counting sort on qlen + tlen, descending)
		std::vector<int> perm(m);
		{
			int maxk = 0;
			for (int i = 0; i < m; ++i) maxk = std::max(maxk, jobs[done + i].q.len + jobs[done + i].t.len);
			std::vector<int> pos(maxk + 2, 0);
			for (int i = 0; i < m; ++i) ++pos[jobs[done + i].q.len + jobs[done + i].t.len];
			int acc = 0;
			for (int k = maxk; k >= 0; --k) { const int c = pos[k]; pos[k] = acc; acc += c; }
			for (int i = 0; i < m; ++i) perm[pos[jobs[done + i].q.len + jobs[done + i].t.len]++] = i;
		}
		// offsets: a serial prefix over the execution order; descriptors: filled in parallel
		std::vector<int64_t> h_poff(m), h_coff(m);
		for (int i = 0; i < m; ++i) {
			const DpJob &J = jobs[done + perm[i]];
			slot_of[done + perm[i]] = done + i;
			// every sequence starts on a 16-byte boundary and is zero padded to one: the fill kernel stages it with bulk copies
			joff[2 * i] = pool_off; pool_off += (J.q.len + 15) & ~15;
			joff[2 * i + 1] = pool_off; pool_off += (J.t.len + 15) & ~15;
			h_poff[i] = p_off; p_off += (int64_t)wm_extd2_bt_bytes(J.q.len, J.t.len, job_w(J));
			h_coff[i] = c_off; c_off += J.q.len + J.t.len + 2;
			prof_bytes += 2.0 * (J.q.len + J.t.len) + 48; // SURVEY.md 8d: qlen + tlen (codes in) + (qlen + tlen) (traceback) + 48; C_block is counted on the device
		}
		joff[2 * (size_t)m] = pool_off;
		#pragma omp parallel for schedule(static) num_threads(8)
		for (int i = 0; i < m; ++i) {
			const DpJob &J = jobs[done + perm[i]];
			wm_dp_job &D = dj[i];
			D.q_off = joff[2 * i], D.t_off = joff[2 * i + 1];
			gj[2 * i] = make_gather(g, J.q, wins[J.task], D.q_off);
			gj[2 * i + 1] = make_gather(g, J.t, wins[J.task], D.t_off);
			D.qlen = J.q.len, D.tlen = J.t.len, D.w = job_w(J), D.zdrop = J.zdrop, D.end_bonus = J.end_bonus, D.flag = J.flag;
			D.p_off = h_poff[i];
			D.cig_off = h_coff[i]; D.cig_cap = J.q.len + J.t.len + 2; D.pad = -1;
		}
		const wm_extd2_plan_t plan = wm_extd2_plan(dj.data(), m, P.single != 0, P.splice != 0);
		std::vector<int32_t> coop; // the big jobs go to the CTA-cooperative sweep (not for the single-affine, splice and first-generation paths)
		if (!P.single && !P.splice && coop_on)
			for (int i = 0; i < m && dj[i].qlen + dj[i].tlen >= 1600; ++i) // (sorted by qlen + tlen, descending)
				if (dj[i].pad >= 0 && wm_dp_is_coop(dj[i].qlen, dj[i].tlen, dj[i].w)) { dj[i].flag |= WM_DP_COOP; coop.push_back(i); }
		g_timers.add("dp.host_prep", Timers::now() - tp0);
		if (getenv("WM_DP_STATS")) {
			int n_big = 0, mq = 0, mt = 0, mw = 0; double cells = 0, big_cells = 0;
			for (int i = 0; i < m; ++i) {
				const DpJob &J = jobs[done + i];
				const double c = (double)J.t.len * std::min(J.q.len, 2 * (J.w < 0 ? J.q.len : J.w) + 1);
				cells += c;
				if (J.t.len > 512 || J.q.len > 640) ++n_big, big_cells += c;
				mq = std::max(mq, J.q.len), mt = std::max(mt, J.t.len), mw = std::max(mw, J.w);
			}
			fprintf(stderr, "[dp-stats] jobs=%d big=%d max_q=%d max_t=%d max_w=%d band_cells=%.3g big_cells=%.3g bt=%.3g MB\n", m, n_big, mq, mt, mw, cells, big_cells, p_off / 1e6);
			// histogram of the longest diagonal of a job (in cells), by job count and by band cells
			const int edges[8] = {16, 32, 64, 128, 256, 512, 1024, 1 << 30};
			double hc[8] = {0}, hn[8] = {0}; int n_approx = 0;
			for (int i = 0; i < m; ++i) {
				const DpJob &J = jobs[done + i];
				const int ww = J.w < 0 ? std::max(J.q.len, J.t.len) : J.w;
				const int L = std::min(std::min(J.q.len, J.t.len), ww + 1);
				int b = 0; while (L > edges[b]) ++b;
				hn[b] += 1, hc[b] += (double)J.t.len * std::min(J.q.len, 2 * ww + 1);
				n_approx += (J.flag & 0x08) != 0;
			}
			fprintf(stderr, "[dp-hist] approx_max=%d/%d;", n_approx, m);
			for (int b = 0; b < 8; ++b) fprintf(stderr, " <=%d: %.1f%% jobs %.1f%% cells;", edges[b] > 100000 ? 99999 : edges[b], 100.0 * hn[b] / m, 100.0 * hc[b] / (cells > 0 ? cells : 1));
			fprintf(stderr, "\n");
		}
		double tq0 = Timers::now();
		wm_gather_job *d_gj = (wm_gather_job*)g.g_jobs.need(sizeof(wm_gather_job) * gj.size());
		int64_t *d_joff = (int64_t*)g.g_joff.need(sizeof(int64_t) * joff.size());
		uint8_t *d_pool = (uint8_t*)g.seq_pool.need(pool_off + 16);
		wm_dp_job *d_dj = (wm_dp_job*)g.dp_jobs.need(sizeof(wm_dp_job) * m);
		// a splice launch's state slices sit behind the traceback matrices in the same buffer: what run_dp counted against
		// bt_budget per chunk is one allocation, so the buffer's size follows the budget and not the sum of two high-water marks
		const size_t bt_end = ((size_t)p_off + 15) / 16 * 16;
		uint8_t *d_bt = (uint8_t*)g.bt.need(bt_end + (P.splice ? plan.splice_bytes : 0) + 16);
		int8_t *d_scr = P.splice ? (int8_t*)(d_bt + bt_end) : 0;
		wm_extz_dev *d_ez = (wm_extz_dev*)g.ez.need(sizeof(wm_extz_dev) * m);
		uint32_t *d_cig = (uint32_t*)g.cig.need(sizeof(uint32_t) * (c_off + 1));
		WM_CUDA_CHECK(wm_memcpy_async(d_gj, gj.data(), sizeof(wm_gather_job) * gj.size(), cudaMemcpyHostToDevice, st));
		WM_CUDA_CHECK(wm_memcpy_async(d_joff, joff.data(), sizeof(int64_t) * joff.size(), cudaMemcpyHostToDevice, st));
		WM_CUDA_CHECK(wm_memcpy_async(d_dj, dj.data(), sizeof(wm_dp_job) * m, cudaMemcpyHostToDevice, st));
		if (pool_off > 0) {
			wm_count_launch(); wm_gather2_kernel<<<(unsigned)((pool_off / 16 + 255) / 256), 256, 0, st>>>(d_gj, d_joff, (int)gj.size(), rd, g.ix.S, d_pool, pool_off / 16);
			WM_CUDA_CHECK(cudaGetLastError());
		}
		// junction annotation of every target slice (src/align.c:688-794: each DP of a spliced mm_align1 gets that of its own
		// target window), at the slice's offset in a pool parallel to d_pool
		uint8_t *d_junc = 0;
		if (P.splice && g.jx.n_seq > 0) {
			std::vector<wm_junc_win> jw(m);
			for (int i = 0; i < m; ++i) {
				const SeqRef &t = jobs[done + perm[i]].t;
				jw[i].dst_off = dj[i].t_off, jw[i].rid = t.kind == SEQ_REF ? t.rid : -1, jw[i].off = (int32_t)t.off, jw[i].len = t.len, jw[i].reversed = t.reversed;
			}
			d_junc = (uint8_t*)g.junc_pool.need(pool_off + 16);
			wm_junc_win *d_jw = (wm_junc_win*)g.junc_wins.need(sizeof(wm_junc_win) * m);
			WM_CUDA_CHECK(wm_memcpy_async(d_jw, jw.data(), sizeof(wm_junc_win) * m, cudaMemcpyHostToDevice, st));
			wm_bed_junc_run(g.jx, d_jw, m, d_junc, st);
		}
		int32_t *d_zd = (int32_t*)g.zd.need(sizeof(int32_t) * 5 * (size_t)m);
		wm_zd_params zp; memset(&zp, 0, sizeof(zp));
		zp.q = sc.q, zp.e = sc.e; memcpy(zp.mat, sc.mat, 25);
		int32_t *d_coop = 0;
		if (!coop.empty()) {
			d_coop = (int32_t*)g.coop_ids.need(sizeof(int32_t) * coop.size());
			WM_CUDA_CHECK(wm_memcpy_async(d_coop, coop.data(), sizeof(int32_t) * coop.size(), cudaMemcpyHostToDevice, st));
		}
		wm_extd2_launch(&g.dpws, d_dj, m, plan, d_pool, d_bt, d_ez, d_cig, P, st, &zp, d_zd, d_coop, (int)coop.size(), d_junc, d_scr);
		// CIGAR lengths -> offsets -> compacted CIGARs, all behind the traceback on the stream: the host then only copies
		int32_t *d_nc = (int32_t*)g.nc_buf.need(sizeof(int32_t) * (m + 1));
		int64_t *d_ooff = (int64_t*)g.cig_off.need(sizeof(int64_t) * (m + 2));
		int64_t *d_stmp = (int64_t*)g.scan_tmp.need(sizeof(int64_t) * (wm_scan_tmp_elems(m) + 1));
		uint32_t *d_cout = (uint32_t*)g.cig_out.need(sizeof(uint32_t) * (c_off + 1));
		wm_count_launch(); wm_ncigar_kernel<<<(m + 255) / 256, 256, 0, st>>>(d_dj, d_ez, m, d_nc);
		wm_exclusive_scan(d_nc, m, d_ooff, d_stmp, st);
		wm_count_launch(); wm_compact_cigar_kernel<<<(unsigned)(((int64_t)m * 32 + 127) / 128), 128, 0, st>>>(d_dj, d_ez, d_ooff, m, d_cig, d_cout);
		WM_CUDA_CHECK(cudaGetLastError());
		std::vector<int64_t> o_off(m + 1, 0);
		WM_CUDA_CHECK(wm_memcpy_async(g.h_ez.data() + done, d_ez, sizeof(wm_extz_dev) * m, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(wm_memcpy_async(g.h_zd.data() + 5 * (size_t)done, d_zd, sizeof(int32_t) * 5 * m, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(wm_memcpy_async(o_off.data(), d_ooff, sizeof(int64_t) * (m + 1), cudaMemcpyDeviceToHost, st));
		wm_stream_sync(st);
		g_timers.add("dp.gpu_fill_bt", Timers::now() - tq0);
		double tr0 = Timers::now();
		for (int i = 0; i < m; ++i) {
			int nc = g.h_ez[done + i].n_cigar;
			if (nc > dj[i].cig_cap) { fprintf(stderr, "[ERROR] winnowmap-b200: CIGAR buffer overflow (%d > %d)\n", nc, dj[i].cig_cap); exit(1); }
		}
		const size_t base = g.h_cig.size();
		g.h_cig.resize(base + o_off[m] + 1);
		if (o_off[m] > 0) WM_CUDA_CHECK(wm_memcpy_async(g.h_cig.data() + base, d_cout, sizeof(uint32_t) * o_off[m], cudaMemcpyDeviceToHost, st));
		wm_stream_sync(st);
		g.h_cig.resize(base + o_off[m]);
		for (int i = 0; i < m; ++i) cig_base[done + i] = (int64_t)base + o_off[i];
		g_timers.add("dp.cigar_d2h", Timers::now() - tr0);
		wm_prof_add(WM_PK_FILL, prof_bytes + 4.0 * (double)o_off[m], 0, m); // + 4 n_cigar
		done = end;
	}
	g.h_cig.push_back(0);
	const double t_res0 = Timers::now();
	#pragma omp parallel for schedule(static) num_threads(8)
	for (int i = 0; i < n; ++i) {
		const int s = slot_of[i]; // where job i ran
		const wm_extz_dev &e = g.h_ez[s];
		DpRes &r = res[i];
		r.max = e.max, r.zdropped = e.zdropped, r.max_q = e.max_q, r.max_t = e.max_t, r.mqe = e.mqe, r.mqe_t = e.mqe_t;
		r.mte = e.mte, r.mte_q = e.mte_q, r.score = e.score, r.reach_end = e.reach_end, r.n_cigar = e.n_cigar;
		r.cigar = g.h_cig.data() + cig_base[s];
		const int32_t *z = g.h_zd.data() + 5 * (size_t)s;
		r.has_zd = (jobs[i].flag & WM_DP_SCAN_ZDROP) && z[0] >= 0;
		if (r.has_zd) r.zd_max = z[0], r.zd_pos[0] = z[1], r.zd_pos[1] = z[2], r.zd_pos[2] = z[3], r.zd_pos[3] = z[4];
	}
	g_timers.add("dp.results", Timers::now() - t_res0);
}

void GpuBackend::run_ll(const std::vector<LlJob> &jobs, const std::vector<MapWin> &wins, const DpScoring &sc, std::vector<LlRes> &res)
{
	WM_CUDA_CHECK(cudaSetDevice(g.device));
	wm_dbuf_use_stream(g.st);
	cudaStream_t st = g.st;
	const int n = (int)jobs.size();
	res.assign(n, LlRes());
	if (n == 0) return;
	wm_pkseq rd; rd.pk = (const uint32_t*)g.pk.p, rd.nm = (const uint32_t*)g.nm.p;
	std::vector<wm_gather_job> gj; std::vector<int64_t> joff(1, 0); std::vector<wm_ll_job> lj(n);
	int64_t pool_off = 0, s_off = 0;
	for (int i = 0; i < n; ++i) {
		const LlJob &J = jobs[i];
		lj[i].q_off = pool_off; add_gather(gj, joff, g, J.q, wins[J.task], &pool_off);
		lj[i].t_off = pool_off; add_gather(gj, joff, g, J.t, wins[J.task], &pool_off);
		lj[i].qlen = J.q.len, lj[i].tlen = J.t.len, lj[i].s_off = s_off;
		s_off += 4 * (int64_t)((J.q.len + 7) / 8 * 8);
	}
	wm_gather_job *d_gj = (wm_gather_job*)g.g_jobs.need(sizeof(wm_gather_job) * gj.size());
	int64_t *d_joff = (int64_t*)g.g_joff.need(sizeof(int64_t) * joff.size());
	uint8_t *d_pool = (uint8_t*)g.seq_pool.need(pool_off + 16);
	wm_ll_job *d_lj = (wm_ll_job*)g.ll_jobs.need(sizeof(wm_ll_job) * n);
	int32_t *d_scr = (int32_t*)g.ll_scr.need(sizeof(int32_t) * (s_off + 4)), *d_out = (int32_t*)g.ll_out.need(sizeof(int32_t) * 3 * (size_t)n);
	int8_t *d_mat = (int8_t*)g.mat.need(32);
	WM_CUDA_CHECK(wm_memcpy_async(d_gj, gj.data(), sizeof(wm_gather_job) * gj.size(), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_joff, joff.data(), sizeof(int64_t) * joff.size(), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_lj, lj.data(), sizeof(wm_ll_job) * n, cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_mat, sc.mat, 25, cudaMemcpyHostToDevice, st));
	if (pool_off > 0) {
		wm_count_launch(); wm_gather2_kernel<<<(unsigned)((pool_off / 16 + 255) / 256), 256, 0, st>>>(d_gj, d_joff, (int)gj.size(), rd, g.ix.S, d_pool, pool_off / 16);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	wm_ksw_ll_launch(d_lj, n, d_pool, d_mat, sc.q, sc.e, d_scr, d_out, st);
	std::vector<int32_t> out(3 * (size_t)n);
	WM_CUDA_CHECK(wm_memcpy_async(out.data(), d_out, sizeof(int32_t) * 3 * n, cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	for (int i = 0; i < n; ++i) res[i].score = out[3 * i], res[i].qe = out[3 * i + 1], res[i].te = out[3 * i + 2];
}

// ---- construction: upload the index to one device ----
// the index arrays are device allocations handed over to the backend (which frees them when it is destroyed)
Backend *gpu_backend_create_dev(const wm_host_idx *hidx, uint64_t *d_keys, int64_t n_keys, uint64_t *d_poff, uint64_t *d_pos,
                                uint64_t bloom_bits, const uint8_t *bloom_table, int device)
{
	WM_CUDA_CHECK(cudaSetDevice(device));
	GpuBackend *be = new GpuBackend();
	GpuBackendImpl &g = be->g;
	g.device = device; g.hidx = hidx; g.n_bases = 0;
	g.st = wm_stream_create_high_priority(); // the DP fill kernels go to a lowest-priority side stream (wm_extd2_launch)
	uint32_t *d_S = wm_dev_alloc<uint32_t>(hidx->S.size() + 4);
	uint8_t *d_bt = wm_dev_alloc<uint8_t>(bloom_bits / 8 + 16);
	WM_CUDA_CHECK(cudaMemcpy(d_S, hidx->S.data(), sizeof(uint32_t) * hidx->S.size(), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_bt, bloom_table, bloom_bits / 8, cudaMemcpyHostToDevice));
	// lengths and name ranks of the sequences for the seed filter of -D / --dual=no (the ranks of hidx, or worked out here
	// from its names when a caller did not set its name order)
	const size_t n_seq = hidx->len.size();
	uint32_t *d_len = wm_dev_alloc<uint32_t>(n_seq + 1), *d_rank = wm_dev_alloc<uint32_t>(n_seq + 1);
	std::vector<uint32_t> rank = hidx->name_rank;
	if (rank.size() != n_seq) { wm_host_idx t; t.name = hidx->name; set_name_order(&t); rank.swap(t.name_rank); }
	if (n_seq) {
		WM_CUDA_CHECK(cudaMemcpy(d_len, hidx->len.data(), sizeof(uint32_t) * n_seq, cudaMemcpyHostToDevice));
		WM_CUDA_CHECK(cudaMemcpy(d_rank, rank.data(), sizeof(uint32_t) * n_seq, cudaMemcpyHostToDevice));
	}
	memset(&g.ix, 0, sizeof(g.ix));
	g.ix.seq_len = d_len, g.ix.name_rank = d_rank;
	g.ix.k = hidx->k, g.ix.w = hidx->w, g.ix.n_seq = (uint32_t)hidx->len.size();
	g.ix.n_keys = n_keys, g.ix.keys = d_keys, g.ix.pos_off = d_poff, g.ix.pos = d_pos, g.ix.S = d_S;
	wm_idx_dev_build_ht(&g.ix, g.st);
	wm_bloom_dev_from_table(&g.bf, d_bt, bloom_bits);
	g.owns_index = true;
	g.own_ix = g.ix, g.own_bf = g.bf, g.own_hidx = hidx;
	wm_stream_sync(g.st);
	size_t free_b = 0, total_b = 0;
	WM_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
	g.bt_budget = free_b / 4; // backtrack matrices of the DP launches in flight (shared by the lanes)
	if (g.bt_budget > ((size_t)32 << 30)) g.bt_budget = (size_t)32 << 30;
	if (const char *e = getenv("WM_BT_BUDGET_GB")) { // tuning: bigger budgets mean fewer, larger fill launches per DP round
		const size_t want = (size_t)atoll(e) << 30;
		if (want > 0 && want < free_b * 3 / 4) g.bt_budget = want;
	}
	{ // workspaces grow through the stream-ordered allocator (wm_dbuf): keep freed blocks in the pool for reuse
		cudaMemPool_t pool;
		uint64_t thr = ~(uint64_t)0;
		WM_CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, device));
		WM_CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
	}
	return be;
}

Backend *gpu_backend_create(const wm_host_idx *hidx, const uint64_t *keys, int64_t n_keys, const uint64_t *pos_off, const uint64_t *pos,
                            uint64_t bloom_bits, const uint8_t *bloom_table, int device)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] winnowmap-b200: no CUDA device visible; there is no CPU fallback\n");
		exit(1);
	}
	WM_CUDA_CHECK(cudaSetDevice(device));
	const uint64_t n_pos = pos_off[n_keys];
	uint64_t *d_keys = wm_dev_alloc<uint64_t>(n_keys + 1), *d_poff = wm_dev_alloc<uint64_t>(n_keys + 2), *d_pos = wm_dev_alloc<uint64_t>(n_pos + 1);
	WM_CUDA_CHECK(cudaMemcpy(d_keys, keys, sizeof(uint64_t) * n_keys, cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_poff, pos_off, sizeof(uint64_t) * (n_keys + 1), cudaMemcpyHostToDevice));
	WM_CUDA_CHECK(cudaMemcpy(d_pos, pos, sizeof(uint64_t) * n_pos, cudaMemcpyHostToDevice));
	return gpu_backend_create_dev(hidx, d_keys, n_keys, d_poff, d_pos, bloom_bits, bloom_table, device);
}

// the resident index arrays of a backend (for the one-time fan-out blob)
void gpu_backend_index_arrays(Backend *be_, const uint64_t **d_keys, const uint64_t **d_poff, const uint64_t **d_pos)
{
	GpuBackend *be = static_cast<GpuBackend*>(be_);
	*d_keys = be->g.own_ix.keys, *d_poff = be->g.own_ix.pos_off, *d_pos = be->g.own_ix.pos;
}

// Point a lane at the index `src` was created with (one part of a multi-part index): the lane keeps its stream and
// workspaces, which depend on no index.  The caller makes sure no batch of the lane is in flight.
void gpu_backend_bind(Backend *lane_, const Backend *src_)
{
	GpuBackendImpl &g = static_cast<GpuBackend*>(lane_)->g;
	const GpuBackendImpl &s = static_cast<const GpuBackend*>(src_)->g;
	g.ix = s.own_ix, g.bf = s.own_bf, g.hidx = s.own_hidx, g.jx = s.own_jx;
}

// Replace the junction intervals of the index `be_` was created with by those of hidx (none when it has no interval with a
// strand).  Lanes bound to that index see them from their next gpu_backend_bind; no batch may be in flight.
void gpu_backend_set_junc(Backend *be_, const wm_host_idx *hidx)
{
	GpuBackendImpl &g = static_cast<GpuBackend*>(be_)->g;
	WM_CUDA_CHECK(cudaSetDevice(g.device));
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	wm_junc_free(&g.own_jx);
	g.own_jx = wm_junc_upload(*hidx);
	g.jx = g.own_jx;
}

// A second orchestration lane on the same device: shares the resident index, owns its stream and workspaces.
Backend *gpu_backend_clone(Backend *base_, int n_lanes)
{
	GpuBackend *base = static_cast<GpuBackend*>(base_);
	WM_CUDA_CHECK(cudaSetDevice(base->g.device));
	GpuBackend *be = new GpuBackend();
	GpuBackendImpl &g = be->g;
	g.device = base->g.device; g.hidx = base->g.hidx; g.n_bases = 0;
	g.ix = base->g.ix; g.bf = base->g.bf;
	g.own_ix = base->g.own_ix, g.own_bf = base->g.own_bf, g.own_hidx = base->g.own_hidx;
	g.jx = base->g.jx, g.own_jx = base->g.own_jx;
	g.st = wm_stream_create_high_priority(); // the DP fill kernels go to a lowest-priority side stream (wm_extd2_launch)
	g.bt_budget = base->g.bt_budget / (size_t)(n_lanes > 0 ? n_lanes : 1);
	return be;
}

void gpu_backend_set_budget(Backend *be, size_t bytes) { static_cast<GpuBackend*>(be)->g.bt_budget = bytes; }
size_t gpu_backend_get_budget(Backend *be) { return static_cast<GpuBackend*>(be)->g.bt_budget; }

void gpu_backend_destroy(Backend *be) { delete be; }

void gpu_backend_trim_pool(int device)
{ // give the stream-ordered allocator's cached blocks back to the device (the release threshold is "never" while mapping)
	cudaMemPool_t pool;
	if (cudaSetDevice(device) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) { cudaDeviceSynchronize(); cudaMemPoolTrimTo(pool, 0); }
}

} // namespace wmh
