// Index construction on the device (mm_idx_gen / worker_post, reference src/index.c:196-252): the (minimizer, position)
// pairs the sketch kernel produced for the reference sequences are ordered by minimizer hash, positions ascending inside a
// hash -- the order in which mm_idx_get hands out occurrence lists (src/index.c:239) -- and cut into the CSR the mapping
// kernels read: sorted unique hashes `keys`, `pos_off`, `pos`.  Nothing goes through the host.
//
// The pairs arrive in position order (sequences in order, positions ascending), and no two pairs share hash and position,
// so a STABLE sort by hash alone produces exactly the (hash, position) order: an LSD radix sort over the 2k significant
// bits of the hash, 8 bits per pass, ping-pong between two buffers.  One warp owns a tile of WM_IX_TILE consecutive pairs
// in both kernels of a pass; inside a tile the ranks come from __match_any_sync, so equal digits keep their order.
#include "wm_common.cuh"
#include "scan.cuh"
#include "sketch.cuh"
#include "index_dev.cuh"

#define WM_IX_TILE 4096
#define WM_IX_WARPS 4

// the sort key of an element: the x word of a (minimizer, position) pair, or a bare 64-bit key (csrc/topfreq.cu)
__device__ __forceinline__ uint64_t wm_ix_key(const wm128_dev &v) { return v.x; }
__device__ __forceinline__ uint64_t wm_ix_key(const uint64_t &v) { return v; }

template <typename T> __global__ void __launch_bounds__(WM_IX_WARPS * 32)
wm_ix_hist_kernel(const T *__restrict__ a, int64_t n, int shift, int64_t n_tiles, int32_t *__restrict__ hist)
{
	__shared__ int cnt[WM_IX_WARPS][256];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const int64_t tile = (int64_t)blockIdx.x * WM_IX_WARPS + wid;
	for (int d = lane; d < 256; d += 32) cnt[wid][d] = 0;
	__syncwarp();
	if (tile < n_tiles) {
		const int64_t beg = tile * WM_IX_TILE, end = beg + WM_IX_TILE < n ? beg + WM_IX_TILE : n;
		for (int64_t i = beg + lane; i < end; i += 32) atomicAdd(&cnt[wid][(int)(wm_ix_key(a[i]) >> shift & 255)], 1);
		__syncwarp();
		for (int d = lane; d < 256; d += 32) hist[(int64_t)d * n_tiles + tile] = cnt[wid][d]; // digit-major: one scan gives every tile's bases
	}
}

template <typename T> __global__ void __launch_bounds__(WM_IX_WARPS * 32)
wm_ix_scatter_kernel(const T *__restrict__ a, T *__restrict__ b, int64_t n, int shift, int64_t n_tiles, const int64_t *__restrict__ offs)
{
	__shared__ long long base[WM_IX_WARPS][256];
	const unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const int64_t tile = (int64_t)blockIdx.x * WM_IX_WARPS + wid;
	if (tile >= n_tiles) return;
	for (int d = lane; d < 256; d += 32) base[wid][d] = offs[(int64_t)d * n_tiles + tile];
	__syncwarp();
	const int64_t beg = tile * WM_IX_TILE, end = beg + WM_IX_TILE < n ? beg + WM_IX_TILE : n;
	const unsigned lt = (1u << lane) - 1u;
	for (int64_t i0 = beg; i0 < end; i0 += 32) {
		const int64_t i = i0 + lane;
		T v = {};
		int d = -1 - lane; // lanes past the end match nobody
		if (i < end) { v = a[i]; d = (int)(wm_ix_key(v) >> shift & 255); }
		const unsigned m = __match_any_sync(FULL, d);
		long long dst = 0;
		if (i < end) dst = base[wid][d] + __popc(m & lt);
		__syncwarp();
		if (i < end && (m & lt) == 0) base[wid][d] += __popc(m); // the first lane of every digit group advances its counter
		__syncwarp();
		if (i < end) b[dst] = v;
	}
}

__global__ void wm_ix_flag_kernel(const wm128_dev *__restrict__ a, int64_t n, int32_t *__restrict__ flag)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	flag[i] = i == 0 || (a[i].x >> 8) != (a[i - 1].x >> 8);
}

__global__ void wm_ix_csr_kernel(const wm128_dev *__restrict__ a, int64_t n, const int32_t *__restrict__ flag, const int64_t *__restrict__ key_idx,
                                 uint64_t *__restrict__ keys, uint64_t *__restrict__ pos_off, uint64_t *__restrict__ pos)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n) return;
	if (i == n) { pos_off[key_idx[n]] = (uint64_t)n; return; }
	pos[i] = a[i].y;
	if (flag[i]) { const int64_t k = key_idx[i]; keys[k] = a[i].x >> 8; pos_off[k] = (uint64_t)i; }
}

// Stable LSD radix sort of the n elements of a by key bits [bit_lo, bit_hi), 8 bits per pass, ping-pong between a and b.
// Returns the buffer that holds the result.
template <typename T> T *wm_lsd_sort(T *a, T *b, int64_t n, int bit_lo, int bit_hi, cudaStream_t st)
{
	if (n <= 0 || bit_lo >= bit_hi) return a;
	T *bufs[2] = { a, b };
	const int64_t n_tiles = (n + WM_IX_TILE - 1) / WM_IX_TILE;
	int cur = 0;
	int32_t *d_hist = wm_dev_alloc<int32_t>(256 * n_tiles + 1);
	int64_t *d_offs = wm_dev_alloc<int64_t>(256 * n_tiles + 2);
	int64_t *d_tmp = wm_dev_alloc<int64_t>(wm_scan_tmp_elems(256 * n_tiles) + 1);
	const unsigned grid = (unsigned)((n_tiles + WM_IX_WARPS - 1) / WM_IX_WARPS);
	for (int shift = bit_lo; shift < bit_hi; shift += 8) {
		wm_count_launch(); wm_ix_hist_kernel<T><<<grid, WM_IX_WARPS * 32, 0, st>>>(bufs[cur], n, shift, n_tiles, d_hist);
		wm_exclusive_scan(d_hist, 256 * n_tiles, d_offs, d_tmp, st);
		wm_count_launch(); wm_ix_scatter_kernel<T><<<grid, WM_IX_WARPS * 32, 0, st>>>(bufs[cur], bufs[cur ^ 1], n, shift, n_tiles, d_offs);
		WM_CUDA_CHECK(cudaGetLastError());
		cur ^= 1;
	}
	WM_CUDA_CHECK(cudaStreamSynchronize(st));
	cudaFree(d_hist); cudaFree(d_offs); cudaFree(d_tmp);
	return bufs[cur];
}
template uint64_t *wm_lsd_sort<uint64_t>(uint64_t *, uint64_t *, int64_t, int, int, cudaStream_t);

// d_a: n pairs in position order (consumed: used as one of the two sort buffers and freed).  k: the k-mer length (the hash has
// 2k significant bits, src/sketch.c:150).  On return the three CSR arrays are device allocations owned by the caller.
void wm_index_build_dev(wm128_dev *d_a, int64_t n, int k, uint64_t **d_keys_out, uint64_t **d_pos_off_out, uint64_t **d_pos_out, int64_t *n_keys_out, cudaStream_t st)
{
	wm128_dev *bufs[2] = { d_a, wm_dev_alloc<wm128_dev>(n + 1) };
	const int key_bits = 2 * k < 56 ? 2 * k : 56;
	// the hash sits above the 8-bit span in x (src/sketch.c:122)
	const wm128_dev *s = wm_lsd_sort(bufs[0], bufs[1], n, 8, 8 + key_bits, st);
	// CSR: key boundaries -> key index (prefix sum) -> keys / pos_off / pos
	int32_t *d_flag = wm_dev_alloc<int32_t>(n + 1);
	int64_t *d_kidx = wm_dev_alloc<int64_t>(n + 2);
	int64_t *d_tmp2 = wm_dev_alloc<int64_t>(wm_scan_tmp_elems(n) + 1);
	if (n > 0) { wm_count_launch(); wm_ix_flag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s, n, d_flag); }
	wm_exclusive_scan(d_flag, n, d_kidx, d_tmp2, st);
	int64_t n_keys = 0;
	WM_CUDA_CHECK(cudaMemcpyAsync(&n_keys, d_kidx + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
	WM_CUDA_CHECK(cudaStreamSynchronize(st));
	uint64_t *d_keys = wm_dev_alloc<uint64_t>(n_keys + 1), *d_poff = wm_dev_alloc<uint64_t>(n_keys + 2), *d_pos = wm_dev_alloc<uint64_t>(n + 1);
	wm_count_launch(); wm_ix_csr_kernel<<<(unsigned)((n + 1 + 255) / 256), 256, 0, st>>>(s, n, d_flag, d_kidx, d_keys, d_poff, d_pos);
	WM_CUDA_CHECK(cudaGetLastError());
	WM_CUDA_CHECK(cudaStreamSynchronize(st));
	cudaFree(d_flag); cudaFree(d_kidx); cudaFree(d_tmp2);
	cudaFree(bufs[0]); cudaFree(bufs[1]);
	*d_keys_out = d_keys, *d_pos_off_out = d_poff, *d_pos_out = d_pos, *n_keys_out = n_keys;
}
