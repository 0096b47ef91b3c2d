// mm_idx_cal_max_occ (reference src/index.c:173-194) on the device: the k-th smallest occurrence count over every key of
// an index, read straight from the CSR offsets (count of key i = pos_off[i+1] - pos_off[i]; a singleton counts 1, as the
// reference's kh_key & 1 branch does).  Exact radix selection, most significant digit first: each pass histograms the
// current 8-bit digit of the counts whose higher digits equal the prefix chosen so far, and a host scan of the 256 bins
// picks the bucket that holds the rank.  Ties need no care: the selection narrows to a value, not to an element.
#include <stdio.h>
#include "wm_common.cuh"
#include "occ_select.cuh"

namespace {

constexpr int kDigitBits = 8, kBins = 1 << kDigitBits;

// bins[d] += number of keys whose count c has (c >> (shift + 8)) == (prefix >> (shift + 8)) and digit d at `shift`.
// A warp adds equal digits once (__match_any_sync): heavy ties do not serialise on one shared-memory bin.
__global__ void occ_digit_hist(const uint64_t *__restrict__ pos_off, int64_t n, uint32_t prefix, int shift, uint32_t *__restrict__ bins)
{
	__shared__ uint32_t h[kBins];
	for (int i = threadIdx.x; i < kBins; i += blockDim.x) h[i] = 0;
	__syncthreads();
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	const int lane = threadIdx.x & 31;
	// every lane of a warp runs the same number of iterations, so that __match_any_sync sees the whole warp
	const int64_t n_iter = (n + stride - 1) / stride;
	const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t hi_mask = shift + kDigitBits >= 32 ? 0u : ~0u << (shift + kDigitBits);
	for (int64_t it = 0; it < n_iter; ++it) {
		const int64_t i = i0 + it * stride;
		uint32_t d = kBins; // no bin: past the end or outside the prefix
		if (i < n) {
			const uint32_t c = (uint32_t)(pos_off[i + 1] - pos_off[i]);
			if ((c & hi_mask) == (prefix & hi_mask)) d = (c >> shift) & (kBins - 1);
		}
		const unsigned peers = __match_any_sync(0xffffffffu, d);
		if (d < (uint32_t)kBins && lane == __ffs(peers) - 1) atomicAdd(&h[d], (uint32_t)__popc(peers));
	}
	__syncthreads();
	for (int i = threadIdx.x; i < kBins; i += blockDim.x)
		if (h[i]) atomicAdd(&bins[i], h[i]);
}

} // namespace

uint32_t wm_occ_select_dev(const uint64_t *d_pos_off, int64_t n, uint64_t rank, cudaStream_t st)
{
	uint32_t *d_bins = wm_dev_alloc<uint32_t>(kBins);
	uint32_t bins[kBins];
	uint32_t prefix = 0;
	int dev = 0, n_sm = 0;
	WM_CUDA_CHECK(cudaGetDevice(&dev));
	WM_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	const int threads = 512;
	int64_t want = (n + threads - 1) / threads;
	const int blocks = (int)(want < 4 * (int64_t)n_sm ? (want > 0 ? want : 1) : 4 * (int64_t)n_sm);
	for (int shift = 32 - kDigitBits; shift >= 0; shift -= kDigitBits) {
		WM_CUDA_CHECK(cudaMemsetAsync(d_bins, 0, sizeof(bins), st));
		occ_digit_hist<<<blocks, threads, 0, st>>>(d_pos_off, n, prefix, shift, d_bins);
		WM_CUDA_CHECK(cudaGetLastError());
		WM_CUDA_CHECK(cudaMemcpyAsync(bins, d_bins, sizeof(bins), cudaMemcpyDeviceToHost, st));
		WM_CUDA_CHECK(cudaStreamSynchronize(st));
		int d = 0;
		for (; d < kBins; ++d) { // the bucket that holds the rank among the keys still in the prefix
			if (rank < bins[d]) break;
			rank -= bins[d];
		}
		if (d == kBins) { fprintf(stderr, "[ERROR] wm_occ_select_dev: rank outside the counts\n"); exit(1); }
		prefix |= (uint32_t)d << shift;
	}
	cudaFree(d_bins);
	return prefix;
}
