// The -W list on the device: count the canonical k-mers of the reference by sorting, take meryl's threshold for
// `distinct=D` and keep the k-mers above it (ext/meryl/src/meryl/merylOp-nextMer.C:103-115; DESIGN.md section 4).
//
// One algorithm for every k (1..28).  A reference of G bases has about G k-mers; two 8-byte buffers of them do not fit next
// to anything else for a human genome, so the codes are counted in partitions of the code space:
//   sweep 0   histogram of the top 12 bits of every canonical code; adjacent buckets are grouped into partitions of at most
//             `budget` k-mers (canonical codes are skewed toward small values: equal-width ranges would not balance)
//   sweep 1   per partition: the codes in its range are emitted (one slot range per warp), sorted with the stable LSD passes
//             of index_dev.cu over the bits that vary inside the range, and cut into runs (head flags + scan); the run
//             lengths go into the count histogram: exact for every value, shared-memory bins below WM_TF_SMALL and an
//             appended list above it
//   host      the threshold from the histogram (wm_topfreq_threshold, the meryl rule)
//   sweep 2   per partition again, the runs longer than the threshold, ascending by construction (a single partition keeps
//             its runs from sweep 1 and is not recounted)
#include <string.h>
#include <algorithm>
#include "wm_common.cuh"
#include "scan.cuh"
#include "index_dev.cuh"
#include "topfreq.cuh"

#define WM_TF_BUCKET_BITS 12
#define WM_TF_SMALL 2048
#define WM_TF_THREADS 256

// sweep 0 (EMIT = false): bucket histogram of the canonical codes; sweeps 1 and 2 (EMIT = true): the codes whose bucket is
// in [blo, bhi), appended to out (*n_out: slots taken).  A thread walks 32 consecutive bases per step; the loop bound is
// warp-uniform so that the whole warp takes part in the slot scan.
template <bool EMIT> __global__ void __launch_bounds__(WM_TF_THREADS)
wm_tf_walk_kernel(const uint32_t *__restrict__ pk, const uint32_t *__restrict__ nm, const int64_t *__restrict__ off, int n_tasks, int k, int sh,
                  uint32_t blo, uint32_t bhi, unsigned long long *__restrict__ hist, uint64_t *__restrict__ out, unsigned long long *__restrict__ n_out)
{
	__shared__ uint32_t cnt[EMIT ? 1 : 1 << WM_TF_BUCKET_BITS];
	if (!EMIT) {
		for (int i = threadIdx.x; i < 1 << WM_TF_BUCKET_BITS; i += blockDim.x) cnt[i] = 0;
		__syncthreads();
	}
	const int lane = threadIdx.x & 31;
	const int64_t n_chunks = (off[n_tasks] + 31) >> 5, stride = (int64_t)gridDim.x * blockDim.x;
	for (int64_t c0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); c0 < n_chunks; c0 += stride) {
		const int64_t p0 = (c0 + lane) << 5;
		uint32_t v = c0 + lane < n_chunks ? wm_tf_valid32(nm, off, n_tasks, k, p0) : 0u, keep = 0;
		for (uint32_t m = v; m; m &= m - 1) {
			const int j = __ffs(m) - 1;
			uint64_t code;
			wm_tf_kmer(pk, nm, p0 + j, k, &code);
			const uint32_t bk = (uint32_t)(code >> sh);
			if (EMIT) keep |= (bk >= blo && bk < bhi ? 1u : 0u) << j;
			else atomicAdd(&cnt[bk], 1u);
		}
		if (EMIT) {
			const int nk = __popc(keep);
			int incl = nk;
			for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
			unsigned long long base = 0;
			if (lane == 31 && incl > 0) base = atomicAdd(n_out, (unsigned long long)incl);
			base = __shfl_sync(0xffffffffu, base, 31);
			uint64_t *dst = out + base + (incl - nk);
			for (; keep; keep &= keep - 1) { uint64_t code; wm_tf_kmer(pk, nm, p0 + __ffs(keep) - 1, k, &code); *dst++ = code; }
		}
	}
	if (!EMIT) {
		__syncthreads();
		for (int i = threadIdx.x; i < 1 << WM_TF_BUCKET_BITS; i += blockDim.x)
			if (cnt[i]) atomicAdd(&hist[i], (unsigned long long)cnt[i]);
	}
}

__global__ void wm_tf_head_kernel(const uint64_t *__restrict__ s, int64_t n, int32_t *__restrict__ flag)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) flag[i] = i == 0 || s[i] != s[i - 1];
}

// start[r]: first element of run r; start[n_runs] = n
__global__ void wm_tf_start_kernel(const int32_t *__restrict__ flag, const int64_t *__restrict__ ridx, int64_t n, uint32_t *__restrict__ start)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i == n) start[ridx[n]] = (uint32_t)n;
	else if (i < n && flag[i]) start[ridx[i]] = (uint32_t)i;
}

// the count histogram: hist[c] for c < WM_TF_SMALL, every larger count appended to big
__global__ void __launch_bounds__(WM_TF_THREADS)
wm_tf_count_kernel(const uint32_t *__restrict__ start, int64_t n_runs, unsigned long long *__restrict__ hist, uint32_t *__restrict__ big, unsigned long long *__restrict__ n_big)
{
	__shared__ uint32_t cnt[WM_TF_SMALL];
	for (int i = threadIdx.x; i < WM_TF_SMALL; i += blockDim.x) cnt[i] = 0;
	__syncthreads();
	for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_runs; r += (int64_t)gridDim.x * blockDim.x) {
		const uint32_t c = start[r + 1] - start[r];
		if (c < WM_TF_SMALL) atomicAdd(&cnt[c], 1u);
		else big[atomicAdd(n_big, 1ULL)] = c;
	}
	__syncthreads();
	for (int i = threadIdx.x; i < WM_TF_SMALL; i += blockDim.x)
		if (cnt[i]) atomicAdd(&hist[i], (unsigned long long)cnt[i]);
}

__global__ void wm_tf_above_kernel(const uint32_t *__restrict__ start, int64_t n_runs, uint64_t thr, int32_t *__restrict__ flag)
{
	const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (r < n_runs) flag[r] = (uint64_t)(start[r + 1] - start[r]) > thr;
}

__global__ void wm_tf_gather_kernel(const uint64_t *__restrict__ s, const uint32_t *__restrict__ start, const int32_t *__restrict__ flag,
                                    const int64_t *__restrict__ sidx, int64_t n_runs, uint64_t *__restrict__ codes, uint32_t *__restrict__ counts)
{
	const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (r < n_runs && flag[r]) { codes[sidx[r]] = s[start[r]]; counts[sidx[r]] = start[r + 1] - start[r]; }
}

// meryl's threshold (merylOp-nextMer.C:103-115): nKmersTarget = (uint64)(D * numDistinct), a double product truncated; walk
// the count values that occur, ascending, accumulating their occurrences; the threshold is the first value at which the sum
// reaches the target.  value[] ascending, occ[] > 0.  An empty histogram gives 0 (there is nothing to list).
extern "C" uint64_t wm_topfreq_threshold(const uint64_t *value, const uint64_t *occ, int64_t n, double distinct)
{
	uint64_t n_distinct = 0, acc = 0;
	for (int64_t i = 0; i < n; ++i) n_distinct += occ[i];
	const uint64_t target = (uint64_t)(distinct * (double)n_distinct);
	for (int64_t i = 0; i < n; ++i) {
		acc += occ[i];
		if (acc >= target) return value[i];
	}
	return 0;
}

static unsigned tf_grid(int64_t n, int per_sm)
{
	const int64_t want = (n + WM_TF_THREADS - 1) / WM_TF_THREADS, cap = (int64_t)wm_sm_count() * per_sm;
	return (unsigned)std::max<int64_t>(1, std::min(want, cap));
}

// k-mers per partition: WM_TOPFREQ_PART_KMERS when set (tests force many partitions with it), else what 70 % of the free
// device memory holds at 26 bytes per k-mer (two sort buffers, head flags, run starts, the sort's tile histograms)
static int64_t tf_budget(void)
{
	const char *e = getenv("WM_TOPFREQ_PART_KMERS");
	if (e && atoll(e) > 0) return atoll(e);
	size_t f = 0, t = 0;
	WM_CUDA_CHECK(cudaMemGetInfo(&f, &t));
	return std::max<int64_t>(1 << 20, (int64_t)(0.7 * (double)f / 26.0));
}

void wm_topfreq_dev(const std::vector<wm_tf_group> &groups, int k, double distinct, wm_tf_list *out, cudaStream_t st)
{
	const int B = 2 * k < WM_TF_BUCKET_BITS ? 2 * k : WM_TF_BUCKET_BITS, sh = 2 * k - B, nb = 1 << B;
	out->codes.clear(); out->counts.clear(); out->threshold = 0; out->n_distinct = 0;
	auto walk = [&](bool emit, uint32_t blo, uint32_t bhi, unsigned long long *d_hist, uint64_t *d_out, unsigned long long *d_n) {
		for (const wm_tf_group &g : groups) {
			if (g.n_tasks <= 0) continue;
			const unsigned grid = (unsigned)wm_sm_count() * 8;
			wm_count_launch();
			if (emit) wm_tf_walk_kernel<true><<<grid, WM_TF_THREADS, 0, st>>>(g.pk, g.nm, g.d_off, g.n_tasks, k, sh, blo, bhi, d_hist, d_out, d_n);
			else wm_tf_walk_kernel<false><<<grid, WM_TF_THREADS, 0, st>>>(g.pk, g.nm, g.d_off, g.n_tasks, k, sh, blo, bhi, d_hist, d_out, d_n);
			WM_CUDA_CHECK(cudaGetLastError());
		}
	};
	// ---- sweep 0: bucket histogram, partitions ----
	std::vector<unsigned long long> bh(nb);
	{
		unsigned long long *d_bh = wm_dev_alloc<unsigned long long>(nb);
		WM_CUDA_CHECK(cudaMemsetAsync(d_bh, 0, sizeof(unsigned long long) * nb, st));
		walk(false, 0, 0, d_bh, 0, 0);
		WM_CUDA_CHECK(cudaMemcpyAsync(bh.data(), d_bh, sizeof(unsigned long long) * nb, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		cudaFree(d_bh);
	}
	const int64_t budget = tf_budget();
	std::vector<uint32_t> pb(1, 0); std::vector<int64_t> pn; // partition p: buckets [pb[p], pb[p + 1]), pn[p] k-mers
	{
		int64_t acc = 0;
		for (int b = 0; b < nb; ++b) {
			if (acc > 0 && acc + (int64_t)bh[b] > budget) { pb.push_back(b); pn.push_back(acc); acc = 0; }
			acc += (int64_t)bh[b];
		}
		pb.push_back(nb); pn.push_back(acc);
	}
	const int n_part = (int)pn.size();
	const int64_t max_n = *std::max_element(pn.begin(), pn.end());
	if (max_n == 0) return;
	if (max_n >= (int64_t)UINT32_MAX) { fprintf(stderr, "[ERROR] wm_topfreq: %lld k-mers in one partition (at most 2^32 - 1)\n", (long long)max_n); exit(1); }
	int64_t total = 0;
	for (int64_t x : pn) total += x;
	// ---- per-partition scratch, sized for the largest partition ----
	uint64_t *d_a = wm_dev_alloc<uint64_t>(max_n + 2), *d_b = wm_dev_alloc<uint64_t>(max_n + 2);
	int32_t *d_flag = wm_dev_alloc<int32_t>(max_n + 1);
	uint32_t *d_start = wm_dev_alloc<uint32_t>(max_n + 2);
	int64_t *d_tmp = wm_dev_alloc<int64_t>(wm_scan_tmp_elems(max_n) + 1);
	unsigned long long *d_ctr = wm_dev_alloc<unsigned long long>(2); // emitted k-mers, appended large counts
	unsigned long long *d_hist = wm_dev_alloc<unsigned long long>(WM_TF_SMALL);
	uint32_t *d_big = wm_dev_alloc<uint32_t>(total / WM_TF_SMALL + 1);
	WM_CUDA_CHECK(cudaMemsetAsync(d_hist, 0, sizeof(unsigned long long) * WM_TF_SMALL, st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_ctr + 1, 0, sizeof(unsigned long long), st));
	// one partition: emit, sort, runs; returns the sorted codes, d_start holds the n_runs + 1 run starts
	auto count_part = [&](int p, int64_t *n_runs) -> uint64_t* {
		const uint32_t blo = pb[p], bhi = pb[p + 1];
		WM_CUDA_CHECK(cudaMemsetAsync(d_ctr, 0, sizeof(unsigned long long), st));
		walk(true, blo, bhi, 0, d_a, d_ctr);
		unsigned long long n_emit = 0;
		WM_CUDA_CHECK(cudaMemcpyAsync(&n_emit, d_ctr, sizeof(n_emit), cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		const int64_t n = pn[p];
		if ((int64_t)n_emit != n) { fprintf(stderr, "[ERROR] wm_topfreq: partition %d emitted %llu k-mers, sweep 0 counted %lld\n", p, n_emit, (long long)n); exit(1); }
		// codes of the partition lie in [blo << sh, (bhi << sh) - 1]: only the bits below their common prefix are sorted
		const uint64_t x = ((uint64_t)blo << sh) ^ (((uint64_t)bhi << sh) - 1);
		uint64_t *s = wm_lsd_sort(d_a, d_b, n, 0, x ? 64 - __builtin_clzll(x) : 0, st);
		int64_t *d_ridx = s == d_a ? (int64_t*)d_b : (int64_t*)d_a; // the other sort buffer
		*n_runs = 0;
		if (n == 0) return s;
		wm_count_launch(); wm_tf_head_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s, n, d_flag);
		wm_exclusive_scan(d_flag, n, d_ridx, d_tmp, st);
		wm_count_launch(); wm_tf_start_kernel<<<(unsigned)((n + 1 + 255) / 256), 256, 0, st>>>(d_flag, d_ridx, n, d_start);
		WM_CUDA_CHECK(cudaGetLastError());
		WM_CUDA_CHECK(cudaMemcpyAsync(n_runs, d_ridx + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		return s;
	};
	// the runs above thr of the partition in s / d_start, appended to the list
	auto select = [&](uint64_t *s, int64_t n_runs, uint64_t thr) {
		if (n_runs == 0) return;
		int64_t *d_sidx = s == d_a ? (int64_t*)d_b : (int64_t*)d_a;
		wm_count_launch(); wm_tf_above_kernel<<<(unsigned)((n_runs + 255) / 256), 256, 0, st>>>(d_start, n_runs, thr, d_flag);
		wm_exclusive_scan(d_flag, n_runs, d_sidx, d_tmp, st);
		int64_t m = 0;
		WM_CUDA_CHECK(cudaMemcpyAsync(&m, d_sidx + n_runs, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		if (m == 0) return;
		uint64_t *d_codes = wm_dev_alloc<uint64_t>(m); uint32_t *d_counts = wm_dev_alloc<uint32_t>(m);
		wm_count_launch(); wm_tf_gather_kernel<<<(unsigned)((n_runs + 255) / 256), 256, 0, st>>>(s, d_start, d_flag, d_sidx, n_runs, d_codes, d_counts);
		WM_CUDA_CHECK(cudaGetLastError());
		const size_t o = out->codes.size();
		out->codes.resize(o + m); out->counts.resize(o + m);
		WM_CUDA_CHECK(cudaMemcpyAsync(out->codes.data() + o, d_codes, sizeof(uint64_t) * m, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaMemcpyAsync(out->counts.data() + o, d_counts, sizeof(uint32_t) * m, cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		cudaFree(d_codes); cudaFree(d_counts);
	};
	// ---- sweep 1: count every partition into the count histogram ----
	uint64_t *kept = 0; int64_t kept_runs = 0;
	for (int p = 0; p < n_part; ++p) {
		int64_t n_runs = 0;
		uint64_t *s = count_part(p, &n_runs);
		if (n_runs > 0) {
			wm_count_launch(); wm_tf_count_kernel<<<tf_grid(n_runs, 4), WM_TF_THREADS, 0, st>>>(d_start, n_runs, d_hist, d_big, d_ctr + 1);
			WM_CUDA_CHECK(cudaGetLastError());
		}
		if (n_part == 1) kept = s, kept_runs = n_runs;
	}
	// ---- the threshold on the host ----
	std::vector<unsigned long long> small(WM_TF_SMALL); unsigned long long n_big = 0;
	WM_CUDA_CHECK(cudaMemcpyAsync(small.data(), d_hist, sizeof(unsigned long long) * WM_TF_SMALL, cudaMemcpyDeviceToHost, st));
	WM_CUDA_CHECK(cudaMemcpyAsync(&n_big, d_ctr + 1, sizeof(n_big), cudaMemcpyDeviceToHost, st));
	WM_CUDA_CHECK(cudaStreamSynchronize(st));
	std::vector<uint32_t> big(n_big);
	if (n_big) WM_CUDA_CHECK(cudaMemcpy(big.data(), d_big, sizeof(uint32_t) * n_big, cudaMemcpyDeviceToHost));
	std::sort(big.begin(), big.end());
	std::vector<uint64_t> value, occ;
	for (int c = 1; c < WM_TF_SMALL; ++c) if (small[c]) value.push_back((uint64_t)c), occ.push_back(small[c]);
	for (size_t i = 0; i < big.size(); ++i) {
		if (i == 0 || big[i] != big[i - 1]) value.push_back(big[i]), occ.push_back(0);
		++occ.back();
	}
	for (uint64_t o : occ) out->n_distinct += (int64_t)o;
	out->threshold = wm_topfreq_threshold(value.data(), occ.data(), (int64_t)value.size(), distinct);
	// ---- sweep 2: the k-mers above the threshold, partition by partition (ascending codes) ----
	if (n_part == 1) select(kept, kept_runs, out->threshold);
	else
		for (int p = 0; p < n_part; ++p) {
			int64_t n_runs = 0;
			uint64_t *s = count_part(p, &n_runs);
			select(s, n_runs, out->threshold);
		}
	cudaFree(d_a); cudaFree(d_b); cudaFree(d_flag); cudaFree(d_start); cudaFree(d_tmp); cudaFree(d_ctr); cudaFree(d_hist); cudaFree(d_big);
}
