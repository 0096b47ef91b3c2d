// Shared helpers for the sm_90a kernels of the Winnowmap seed-chain-align path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

// Fatal-error convention of the reference (src/misc.c:123-151): message on stderr, exit(1).
#define WM_CUDA_CHECK(call) do { \
	cudaError_t wm_e_ = (call); \
	if (wm_e_ != cudaSuccess) { \
		fprintf(stderr, "[ERROR] CUDA failure at %s:%d: %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(wm_e_)); \
		exit(1); \
	} \
} while (0)

#define WM_NEG_INF (-0x40000000)

// Lightweight instrumentation used by bench.py (prof.cu): number of kernel launches and, when enabled, the device time
// and algorithmic bytes of the two kernel classes that dominate the path (the extension-DP fill kernel and the
// chaining forward pass), measured with CUDA events on the launching stream.  Nothing is synchronised inside a
// profiled region: every launch gets an event pair that is read afterwards against a common base event.
enum { WM_PK_FILL = 0, WM_PK_CHAIN = 1, WM_PK_N = 2 };
struct wm_prof_kind { double ms, union_ms, alg_bytes, units, units2; long long launches; };
struct wm_prof_t {
	long long n_launches;
	int enabled;
	wm_prof_kind k[WM_PK_N];        // units: block cells (fill) / anchors (chain); units2: DP jobs (fill)
	long long h2d_bytes, d2h_bytes; // every host<->device copy of the mapping path (wm_memcpy_async)
};
extern wm_prof_t g_wm_prof;
// cudaMemcpyAsync that also counts the bytes per direction (bench: e2e.h2d_bytes_per_step / d2h_bytes_per_step)
static inline cudaError_t wm_memcpy_async(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st)
{
	if (kind == cudaMemcpyHostToDevice) __atomic_fetch_add(&g_wm_prof.h2d_bytes, (long long)bytes, __ATOMIC_RELAXED);
	else if (kind == cudaMemcpyDeviceToHost) __atomic_fetch_add(&g_wm_prof.d2h_bytes, (long long)bytes, __ATOMIC_RELAXED);
	return cudaMemcpyAsync(dst, src, bytes, kind, st);
}
void wm_prof_region_begin(void);  // start of a profiled region (base event)
void wm_prof_collect(void);       // fold the recorded launches into g_wm_prof
// Around one launch of kind `kind` on stream `st`: begin returns a slot (-1 = not profiling) and, if ctr is non-null,
// a zeroed pair of device counters the kernel may add work units to (counted as units / algorithmic bytes at collect).
int wm_prof_launch_begin(int kind, cudaStream_t st, cudaStream_t zero_st, unsigned long long **ctr);
void wm_prof_launch_end(int slot, cudaStream_t st);
void wm_prof_add(int kind, double alg_bytes, double units, double units2);
static inline void wm_count_launch() { __atomic_fetch_add(&g_wm_prof.n_launches, 1LL, __ATOMIC_RELAXED); }

// One extension-DP job; sequences live in a device byte pool (0..4 codes).
struct wm_dp_job {
	int64_t q_off, t_off;   // byte offsets of query / target codes in the sequence pool
	int64_t p_off;          // byte offset of this job's backtrack matrix
	int64_t cig_off;        // uint32 offset of this job's CIGAR buffer
	int32_t qlen, tlen, w, zdrop, end_bonus, flag;
	int32_t cig_cap, pad;   // pad: slot of the job's state rows in the global scratch, -1 = they fit shared memory (wm_extd2_plan)
};

// Scoring parameters shared by a batch (src/ksw2_extd2_sse.c:61-97)
struct wm_dp_params {
	int32_t q, e, q2, e2;      // after the swap at :70
	int32_t qe_h;              // q+e BEFORE the swap (:61), used only for H[0]/H0 (:351,:371)
	int32_t sc_mch, sc_mis, sc_N;
	int32_t long_thres, long_diff;
	int32_t early_out;         // -min_sc > 2*(q+e) (:92)
	int32_t single;            // q == q2 && e == e2: the call is ksw_extz2_sse (src/align.c:328-331), csrc/ksw_extz2.cuh
	int32_t splice;            // the call is ksw_exts2_sse (src/align.c:326-327), csrc/ksw_exts2.cuh: q, e, q2 as given, e2 unused
	int32_t noncan, junc_bonus;
	int8_t mat[25];            // for KSW_EZ_GENERIC_SC (splice path only)
};

struct wm_extz_dev {
	int32_t max, zdropped, max_q, max_t, mqe, mqe_t, mte, mte_q, score, reach_end, n_cigar, reserved;
};

template <typename T>
static inline T *wm_dev_alloc(size_t n)
{
	T *p = 0;
	WM_CUDA_CHECK(cudaMalloc((void**)&p, (n > 0 ? n : 1) * sizeof(T)));
	return p;
}

// Growable device buffer (never shrinks): pre-sized pools instead of a per-call allocator.
// Grow-only device buffer.  Growth goes through the stream-ordered allocator on the stream the calling thread
// declared with wm_dbuf_use_stream() (each orchestration lane drives one stream): unlike cudaFree/cudaMalloc it does
// not synchronise the device, so one lane growing a workspace does not stall the kernels of the others.
extern thread_local cudaStream_t wm_dbuf_stream;
extern thread_local bool wm_dbuf_async;
static inline void wm_dbuf_use_stream(cudaStream_t st) { wm_dbuf_stream = st; wm_dbuf_async = true; }
struct wm_dbuf {
	void *p; size_t cap; bool async; cudaStream_t st;
	wm_dbuf() : p(0), cap(0), async(false), st(0) {}
	wm_dbuf(const wm_dbuf&) = delete;
	wm_dbuf &operator=(const wm_dbuf&) = delete;
	// cudaFree also takes stream-ordered allocations (it synchronises), so the owner's stream may be gone already
	~wm_dbuf() { if (p) cudaFree(p); }
	void drop() {
		if (!p) return;
		if (async) WM_CUDA_CHECK(cudaFreeAsync(p, st)); else WM_CUDA_CHECK(cudaFree(p));
		p = 0, cap = 0;
	}
	void *need(size_t bytes) {
		if (bytes > cap) {
			drop();
			size_t nc = bytes + bytes / 2 + 256;
			if (wm_dbuf_async) {
				st = wm_dbuf_stream, async = true;
				WM_CUDA_CHECK(cudaMallocAsync(&p, nc, st));
			} else { async = false; WM_CUDA_CHECK(cudaMalloc(&p, nc)); }
			cap = nc;
		}
		return p;
	}
	void release() { if (p) { if (async) cudaFreeAsync(p, st); else cudaFree(p); } p = 0; cap = 0; }
};

// Host result pool in page-locked memory, grow-only, with the small slice of std::vector's interface the backend uses.
// Device-to-host copies into pageable memory are staged by the driver through a bounce buffer, a few GB/s and one lane at
// a time; the chains and CIGARs of a wave are hundreds of MB.  Falls back to pageable memory if page-locking fails.
template <typename T> struct wm_hbuf {
	T *p; size_t n, cap; bool pinned;
	wm_hbuf() : p(0), n(0), cap(0), pinned(false) {}
	wm_hbuf(const wm_hbuf&) = delete;
	wm_hbuf &operator=(const wm_hbuf&) = delete;
	~wm_hbuf() { drop(p, pinned); }
	static void drop(T *q, bool pin) { if (q) { if (pin) cudaFreeHost(q); else free(q); } }
	T *data() { return p; }
	const T *data() const { return p; }
	size_t size() const { return n; }
	void clear() { n = 0; }
	void resize(size_t m) { // keeps the first min(n, m) elements
		if (m > cap) {
			const size_t nc = 2 * m + (1u << 16); // page-locking is slow (and serialises the lanes): grow rarely
			T *q = 0; bool pin = true;
			if (cudaMallocHost((void**)&q, nc * sizeof(T)) != cudaSuccess) { cudaGetLastError(); pin = false; q = (T*)malloc(nc * sizeof(T)); }
			if (!q) { fprintf(stderr, "[ERROR] winnowmap-b200: out of host memory (%zu bytes)\n", nc * sizeof(T)); exit(1); }
			if (n) memcpy(q, p, n * sizeof(T));
			drop(p, pinned);
			p = q, cap = nc, pinned = pin;
		}
		n = m;
	}
	void push_back(const T &v) { resize(n + 1); p[n - 1] = v; }
	T &operator[](size_t i) { return p[i]; }
};

// ---- batched ksw_extd2 on device-resident jobs (ksw_extd2.cu) ----
// The fill kernel runs on its own lowest-priority stream, ordered against the caller's stream by two events: its
// CTAs leave the SMs job group by job group, and the short kernels of the other orchestration lanes (created with
// the highest priority) take the freed slots first instead of queueing behind a whole DP launch.
struct wm_extd2_ws {
	wm_dbuf scratch;
	cudaStream_t fill_st, coop_st; cudaEvent_t ev_ready, ev_done, ev_coop; // coop_st: the CTA-cooperative sweep of the big jobs, beside the others
	wm_extd2_ws() : fill_st(0), coop_st(0), ev_ready(0), ev_done(0), ev_coop(0) {}
	~wm_extd2_ws() { if (fill_st) { cudaStreamDestroy(fill_st); cudaStreamDestroy(coop_st); cudaEventDestroy(ev_ready); cudaEventDestroy(ev_done); cudaEventDestroy(ev_coop); } }
};
struct wm_extd2_plan_t { int n_slots, max_tlen, max_qlen; size_t splice_bytes; }; // splice_bytes: the global slices of a splice launch
void wm_dp_params_init(wm_dp_params *P, const int8_t *mat, int q, int e, int q2, int e2);
void wm_dp_params_init_splice(wm_dp_params *P, const int8_t *mat, int q, int e, int q2, int noncan, int junc_bonus); // src/ksw2_exts2_sse.c:61-84
size_t wm_extd2_bt_bytes(int qlen, int tlen, int w);
// sets h_jobs[i].pad (global-scratch slot or -1) for the n jobs of one launch, in launch order; single: the jobs run the
// single-affine sweep (wm_dp_params::single), whose state slice is 9 bytes per target cell
wm_extd2_plan_t wm_extd2_plan(wm_dp_job *h_jobs, int n, bool single = false, bool splice = false); // splice: ksw_exts2.cuh, 12 bytes per cell
// splice launches size every global slice by its own job: unbanded gap fills across introns reach 200 kb of target, and one
// stride for all (the largest tlen) would multiply that by the number of jobs.  The global scratch a splice job of target
// length tlen takes (0: it fits the shared-memory slice), a multiple of WM_EXTS2_PAD_UNIT.
#define WM_EXTS2_PAD_UNIT 16
size_t wm_exts2_scratch_bytes(int tlen);
// Jobs flagged WM_DP_SCAN_ZDROP also get the score walk of mm_test_zdrop (src/align.c:32-70) over their CIGAR: five
// int32 per job in d_zd (max_zdrop, t0, t1, q0, q1; max_zdrop = -1: no result).  zp / d_zd may be null.
#define WM_DP_SCAN_ZDROP 0x10000
// Jobs flagged WM_DP_COOP are skipped by the warp-per-job kernel and swept by a whole CTA (d_coop_ids lists them): the few big
// jobs (>= 300 k band cells, diagonals of >= 384 cells) that would otherwise keep a launch waiting on one warp.  wm_dp_is_coop is the host's rule.
#define WM_DP_COOP 0x20000
static inline bool wm_dp_is_coop(int qlen, int tlen, int w)
{
	static long long min_cells = -1; // WM_DP_COOP_MIN_CELLS (tuning)
	if (min_cells < 0) { const char *e = getenv("WM_DP_COOP_MIN_CELLS"); min_cells = e && atoll(e) > 0 ? atoll(e) : 300000; }
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	const int diag = qlen < tlen ? (qlen < w + 1 ? qlen : w + 1) : (tlen < w + 1 ? tlen : w + 1);
	const long long cells = (long long)tlen * (qlen < 2 * w + 1 ? qlen : 2 * w + 1);
	return diag >= 384 && cells >= min_cells;
}
struct wm_zd_params { int32_t q, e; int8_t mat[25]; int8_t pad[3]; };
void wm_extd2_launch(wm_extd2_ws *ws, const wm_dp_job *d_jobs, int n_jobs, const wm_extd2_plan_t &plan, const uint8_t *d_seq, uint8_t *d_bt,
                     wm_extz_dev *d_ez, uint32_t *d_cigar, const wm_dp_params &P, cudaStream_t stream,
                     const wm_zd_params *zp = 0, int32_t *d_zd = 0, const int32_t *d_coop_ids = 0, int n_coop = 0,
                     const uint8_t *d_junc = 0, int8_t *d_scratch = 0); // d_junc: junction annotation parallel to d_seq (splice jobs), or
                     // null; d_scratch: the global state slices (plan.splice_bytes for a splice launch) from the caller, or null: ws->scratch
cudaStream_t wm_stream_create_high_priority(void);
// SMs of the current device: grids that hold a fixed number of CTAs per SM are sized from it
static inline int wm_sm_count(void)
{
	int dev = 0, n_sm = 0;
	WM_CUDA_CHECK(cudaGetDevice(&dev));
	WM_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	return n_sm;
}

// Wait for a stream without burning a core: an orchestration lane spends most of its time waiting for the GPU, and
// with several lanes per process and several processes per node the spinning waits of cudaStreamSynchronize compete
// with the OpenMP workers.  (WM_SPIN_SYNC=1 restores the spinning wait.)
struct wm_sync_event { // one blocking event per waiting thread, destroyed with the thread
	cudaEvent_t ev;
	wm_sync_event() : ev(0) {}
	~wm_sync_event() { if (ev) cudaEventDestroy(ev); }
};
static inline void wm_stream_sync(cudaStream_t st)
{
	static thread_local wm_sync_event h;
	static int spin = -1;
	if (spin < 0) { const char *e = getenv("WM_SPIN_SYNC"); spin = (e && *e == '1') ? 1 : 0; }
	if (spin) { WM_CUDA_CHECK(cudaStreamSynchronize(st)); return; }
	if (!h.ev) WM_CUDA_CHECK(cudaEventCreateWithFlags(&h.ev, cudaEventBlockingSync | cudaEventDisableTiming));
	WM_CUDA_CHECK(cudaEventRecord(h.ev, st));
	WM_CUDA_CHECK(cudaEventSynchronize(h.ev));
}

#ifndef WM_HOST_EMUL
// ---- bulk-asynchronous (TMA) copies: cp.async.bulk global <-> shared, completion on an mbarrier / a bulk group ----
// One thread arms an mbarrier with the byte count and issues the copy; the copy engine moves the bytes while the other
// threads do something else; everybody then waits on the barrier's phase.  Source and destination must be 16-byte aligned
// and the size a multiple of 16.  Users: the DP fill kernel (a job's target and query), the anchor sort kernels (an array
// into its shared-memory stage and back).
__device__ __forceinline__ uint32_t wm_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wm_mbar_init(uint64_t *mbar, int count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(wm_smem_u32(mbar)), "r"(count) : "memory");
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void wm_mbar_expect_tx(uint64_t *mbar, uint32_t bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(wm_smem_u32(mbar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void wm_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *mbar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
	             :: "r"(wm_smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(wm_smem_u32(mbar)) : "memory");
}
__device__ __forceinline__ void wm_mbar_wait(uint64_t *mbar, uint32_t phase)
{
	uint32_t ok = 0;
	while (!ok)
		asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
		             : "=r"(ok) : "r"(wm_smem_u32(mbar)), "r"(phase) : "memory");
}
// shared -> global, tracked by the issuing thread's bulk group
__device__ __forceinline__ void wm_bulk_s2g(void *dst_gmem, const void *src_smem, uint32_t bytes)
{
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // the generic-proxy writes of the stage must be visible to the copy engine
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst_gmem), "r"(wm_smem_u32(src_smem)), "r"(bytes) : "memory");
	asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void wm_bulk_s2g_wait(void) { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
#endif
