// Weighted robust-winnowing minimizers on sm_90a: the output of mm_sketch
// (reference src/sketch.c:128-219, weights :70-90, bloom probe ext/bloom/bloom_filter.hpp:303-319,
// :551-565) for a batch of sequences, restructured into three data-parallel passes:
//
//   A  per base: canonical k-mer -> order key (double, murmur64 / 2^64, x^8 when the k-mer is in the
//      down-weight filter) and an "eligible" bit = the key is strictly below the w previous keys.
//   B  the winnowing state machine is history dependent only through ties, so it can be restarted
//      exactly at any eligible position (a strict new minimum is certain there, whatever the
//      history).  One thread per 128-base chunk starts at the first eligible position of its chunk
//      and runs until the first eligible position of a later chunk, flagging emitted minimizers.
//   C  flags -> per-chunk counts -> exclusive scan -> (x,y) records in position order.
//
// For odd k (the defaults 15/19) a k-mer cannot equal its reverse complement, so ring slots and
// bases coincide (src/sketch.c:166 never fires); even k takes a sequential per-sequence kernel.
//
// The sequences are read from the packed pool (pkseq.cuh: 2 bits per base + ambiguity mask).  Pass A stages the packed
// words of its tile with 128-bit loads, takes every k-mer as one unaligned 64-bit window of them (no per-base rebuild),
// and finds the minimum of the w previous keys by doubling (log2 w rounds over shared memory) instead of scanning them.
#include <math.h>
#include <string.h>
#include <vector>
#include "wm_common.cuh"
#include "scan.cuh"
#include "sketch.cuh"
#include "pkseq.cuh"
#include "hpc.cuh"

#define WM_SK_TN 1024      // new positions per tile in pass A
#define WM_SK_THREADS 256
#define WM_SK_CH 128       // chunk size in pass B/C

__device__ __forceinline__ uint64_t wm_murmur64(uint64_t key)
{ // src/sketch.c:43-51
	key ^= key >> 33; key *= 0xff51afd7ed558ccdULL;
	key ^= key >> 33; key *= 0xc4ceb9fe1a85ec53ULL;
	key ^= key >> 33;
	return key;
}
__device__ __forceinline__ uint64_t wm_hash64(uint64_t key, uint64_t mask)
{ // src/sketch.c:53-63
	key = (~key + (key << 21)) & mask;
	key = key ^ key >> 24;
	key = ((key + (key << 3)) + (key << 8)) & mask;
	key = key ^ key >> 14;
	key = ((key + (key << 2)) + (key << 4)) & mask;
	key = key ^ key >> 28;
	key = (key + (key << 31)) & mask;
	return key;
}
__device__ __forceinline__ bool wm_bloom_contains(const wm_bloom_dev &bf, uint64_t key)
{ // bloom_filter.hpp:303-319 with hash_ap on 8 bytes (:556-565) and compute_indices (:461-465)
	const uint32_t i1 = (uint32_t)key, i2 = (uint32_t)(key >> 32);
	for (int i = 0; i < bf.n_salt; ++i) {
		uint32_t h = bf.salt[i];
		h ^= (h << 7) ^ (i1 * (h >> 3)) ^ (~((h << 11) + (i2 ^ (h >> 5))));
		uint64_t bit = (uint64_t)h % bf.bits;
		if (!((bf.table[bit >> 3] >> (bit & 7)) & 1)) return false;
	}
	return true;
}
__device__ __forceinline__ double wm_weight(uint64_t kmer, const wm_bloom_dev &bf)
{ // src/sketch.c:70-90; (double)UINT64_MAX is 2^64, so the division is an exact scaling
	const uint64_t h = wm_murmur64(kmer);
	const double x = __ull2double_rn(h) * 5.421010862427522e-20; // 2^-64
	if (wm_bloom_contains(bf, kmer)) {
		double p2 = __dmul_rn(x, x), p4 = __dmul_rn(p2, p2);
		return -__dmul_rn(p4, p4);
	}
	return -x;
}

// ---- pass A ----
#define WM_SK_NE (WM_SK_TN + 256)   // order keys held per tile: the w previous positions + the tile
#define WM_SK_PKW 96                // packed words staged per tile (64-base aligned start, + the window's look-ahead)
#define WM_SK_SMEM (3 * WM_SK_NE * 8 + WM_SK_PKW * 4 + WM_SK_PKW * 2)

// HPC: the sequence is a compressed slice (symbols), pos maps each symbol to the last base of its run (relative to the
// uncompressed task); a k-mer whose span pos[p] - pos[p - k] reaches 256 is valid but never a candidate: key 3.0.
template <bool HPC>
__global__ void __launch_bounds__(WM_SK_THREADS)
wm_sketch_order_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ tile_off,
                       const int64_t *__restrict__ base_off, int n_tasks, int w, int k, wm_bloom_dev bf,
                       double *__restrict__ ord, uint8_t *__restrict__ elig, const int32_t *__restrict__ pos)
{
	extern __shared__ __align__(16) uint8_t sm_raw[];
	double *s_ord = (double*)sm_raw;                 // position p0 - w + j
	double *s_a = s_ord + WM_SK_NE, *s_b = s_a + WM_SK_NE; // window minima, ping-pong
	uint32_t *s_pk = (uint32_t*)(s_b + WM_SK_NE);    // packed bases from pool base Gw on
	uint32_t *s_nm = s_pk + WM_SK_PKW;
	// which task does this tile belong to?
	int lo = 0, hi = n_tasks;
	const int64_t tile = blockIdx.x;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (tile_off[m] <= tile) lo = m; else hi = m; }
	const wm_sk_task T = tasks[lo];
	const int p0 = (int)(tile - tile_off[lo]) * WM_SK_TN;
	// bases p0 - w - (k - 1) .. p0 + WM_SK_TN - 1 of the sequence, staged from the 64-base boundary below the first one
	const int n_code = WM_SK_TN + w + k - 1;
	const int64_t G0 = T.seq_off + p0 - w - (k - 1);
	const int64_t Gw = (G0 >> 6) << 6; // (floors for a negative G0: the first sequence of the pool)
	const int n_q = ((int)(G0 - Gw) + n_code + 63) / 64 + 1;
	const int64_t q_last = (T.seq_off + T.len) >> 6; // nothing past the sequence is needed
	for (int j = threadIdx.x; j < n_q; j += WM_SK_THREADS) {
		const int64_t q = (Gw >> 6) + j;
		const bool in = q >= 0 && q <= q_last;
		((uint4*)s_pk)[j] = in ? ((const uint4*)seq.pk)[q] : make_uint4(0u, 0u, 0u, 0u);
		((uint2*)s_nm)[j] = in ? ((const uint2*)seq.nm)[q] : make_uint2(~0u, ~0u);
	}
	__syncthreads();
	const uint32_t kmask = (1u << k) - 1u;
	for (int j = threadIdx.x; j < WM_SK_NE; j += WM_SK_THREADS) {
		const int p = p0 - w + j;
		double o = 2.0;
		if (j < WM_SK_TN + w && p >= k - 1 && p < T.len) {
			const int64_t rel = T.seq_off + (p - (k - 1)) - Gw; // first base of the k-mer
			if (!(wm_pk_nwindow(s_nm, rel) & kmask)) {
				uint64_t f, r;
				wm_pk_kmer(wm_pk_window(s_pk, rel), k, &f, &r);
				if (HPC) {
					const int64_t q = T.seq_off + p;
					const int span = pos[q] - (p >= k ? pos[q - k] : -1);
					if (f != r) o = span < 256 ? wm_weight(f < r ? f : r, bf) : 3.0;
				} else if (f != r) o = wm_weight(f < r ? f : r, bf);
			}
		}
		s_ord[j] = o;
	}
	__syncthreads();
	// minimum over [j, j + w): levels of spans 2, 4, .. 2^t <= w, then two overlapping spans of 2^t
	int t = 31 - __clz(w);
	const double *cur = s_ord;
	for (int l = 0; l < t; ++l) {
		double *nxt = (l & 1) ? s_b : s_a;
		const int d = 1 << l;
		for (int j = threadIdx.x; j < WM_SK_NE; j += WM_SK_THREADS) nxt[j] = j + d < WM_SK_NE ? fmin(cur[j], cur[j + d]) : cur[j];
		__syncthreads();
		cur = nxt;
	}
	const int d2 = w - (1 << t);
	const int64_t gb = base_off[lo];
	for (int j = threadIdx.x; j < WM_SK_TN; j += WM_SK_THREADS) {
		const int p = p0 + j;
		if (p >= T.len) break;
		const double o = s_ord[j + w];
		const bool e = o < 2.0 && o < fmin(cur[j], cur[j + d2]);
		ord[gb + p] = o;
		elig[gb + p] = e ? 1 : 0;
	}
}

// ---- pass B ----
// v counts the valid k-mers in a row (l >= k of src/sketch.c): keys below 2.0, and under HPC also the 3.0 of pass A
template <bool HPC>
__global__ void wm_sketch_winnow_kernel(const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ chunk_off,
                                        const int64_t *__restrict__ base_off, int n_tasks, int64_t n_chunks, int w,
                                        const double *__restrict__ ord_all, const uint8_t *__restrict__ elig_all, uint8_t *__restrict__ flag_all)
{
	const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (ch >= n_chunks) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (chunk_off[m] <= ch) lo = m; else hi = m; }
	const int len = tasks[lo].len;
	const int64_t gb = base_off[lo];
	const double *ord = ord_all + gb;
	const uint8_t *elig = elig_all + gb;
	uint8_t *flag = flag_all + gb;
	const int c0 = (int)(ch - chunk_off[lo]) * WM_SK_CH;
	int c1 = c0 + WM_SK_CH; if (c1 > len) c1 = len;
	int min_i = -1, v = 0, i;
	double min_ord = 2.0;
	if (c0 == 0) i = 0;
	else {
		int s = c0;
		while (s < c1 && !elig[s]) ++s;
		if (s >= c1) return; // an earlier thread runs through this chunk
		min_i = s, min_ord = ord[s];
		for (int j = s; j >= 0 && v < w + 1 && (HPC ? ord[j] != 2.0 : ord[j] < 2.0); --j) ++v;
		i = s + 1;
	}
	bool seen = false; // an eligible position was already met in the chunk that contains i
	for (; i < len; ++i) {
		if ((i & (WM_SK_CH - 1)) == 0) seen = false;
		const double o = ord[i];
		v = (HPC ? o != 2.0 : o < 2.0) ? (v < w + 1 ? v + 1 : v) : 0;
		if (o < min_ord) { // a new minimum (src/sketch.c:180-189)
			if (v >= w + 1 && min_i >= 0) flag[min_i] = 1;
			min_i = i, min_ord = o;
		} else if (min_i >= 0 && i - min_i == w) { // the old minimum left the window (:191-205)
			if (v >= w) flag[min_i] = 1;
			int m = -1; double mo = 2.0;
			for (int j = i - w + 1; j <= i; ++j) {
				double oj = ord[j];
				if (mo >= oj) mo = oj, m = j; // ">=": the closest (rightmost) k-mer wins
			}
			if (mo >= 2.0) m = -1, mo = 2.0;
			min_i = m, min_ord = mo;
		}
		if (elig[i]) {
			if (!seen && i >= c1) return; // the thread of that chunk resumes from here
			seen = true;
		}
	}
	if (min_i >= 0) flag[min_i] = 1; // :208
}

// sequential pass for even k (symmetric k-mers make ring slots != bases): one thread per sequence
template <bool HPC>
__global__ void wm_sketch_seq_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ base_off,
                                     int n_tasks, int w, int k, wm_bloom_dev bf, uint8_t *__restrict__ flag_all, double *__restrict__ ring_all,
                                     const int32_t *__restrict__ pos)
{
	const int tid = blockIdx.x * blockDim.x + threadIdx.x;
	if (tid >= n_tasks) return;
	const wm_sk_task T = tasks[tid];
	uint8_t *flag = flag_all + base_off[tid];
	double *buf_ord = ring_all + (size_t)tid * 512; // order keys
	double *buf_pos_ = buf_ord + 256;               // positions, stored as doubles (exact below 2^53)
	const uint64_t shift1 = 2 * (k - 1), mask = (1ULL << 2 * k) - 1;
	uint64_t kmer0 = 0, kmer1 = 0;
	int l = 0, buf_pos = 0, min_pos = 0, min_i = -1;
	double min_ord = 2.0;
	for (int j = 0; j < w; ++j) buf_ord[j] = 2.0, buf_pos_[j] = -1.0;
	for (int i = 0; i < T.len; ++i) {
		const int c = wm_pk_get(seq, T.seq_off + i);
		double o = 2.0; int oi = -1;
		if (c < 4) {
			kmer0 = (kmer0 << 2 | (uint64_t)c) & mask;
			kmer1 = (kmer1 >> 2) | (3ULL ^ (uint64_t)c) << shift1;
			if (kmer0 == kmer1) continue; // src/sketch.c:166
			++l;
			if (l >= k && (!HPC || pos[T.seq_off + i] - (i >= k ? pos[T.seq_off + i - k] : -1) < 256))
				o = wm_weight(kmer0 < kmer1 ? kmer0 : kmer1, bf), oi = i;
		} else l = 0;
		buf_ord[buf_pos] = o, buf_pos_[buf_pos] = (double)oi;
		if (o < min_ord) {
			if (l >= w + k && min_i >= 0) flag[min_i] = 1;
			min_i = oi, min_pos = buf_pos, min_ord = o;
		} else if (buf_pos == min_pos) {
			if (l >= w + k - 1 && min_i >= 0) flag[min_i] = 1;
			min_i = -1, min_ord = 2.0;
			for (int j = buf_pos + 1; j < w; ++j) if (min_ord >= buf_ord[j]) min_i = (int)buf_pos_[j], min_pos = j, min_ord = buf_ord[j];
			for (int j = 0; j <= buf_pos; ++j) if (min_ord >= buf_ord[j]) min_i = (int)buf_pos_[j], min_pos = j, min_ord = buf_ord[j];
		}
		if (++buf_pos == w) buf_pos = 0;
	}
	if (min_i >= 0) flag[min_i] = 1;
}

// ---- pass C ----
__global__ void wm_sketch_count_kernel(const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ chunk_off, const int64_t *__restrict__ base_off,
                                       int n_tasks, int64_t n_chunks, const uint8_t *__restrict__ flag_all, int32_t *__restrict__ cnt)
{
	const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (ch >= n_chunks) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (chunk_off[m] <= ch) lo = m; else hi = m; }
	const int len = tasks[lo].len;
	const uint8_t *flag = flag_all + base_off[lo];
	const int c0 = (int)(ch - chunk_off[lo]) * WM_SK_CH;
	int c1 = c0 + WM_SK_CH; if (c1 > len) c1 = len;
	int n = 0;
	for (int i = c0; i < c1; ++i) n += flag[i];
	cnt[ch] = n;
}

// HPC: positions and spans come from the symbol -> base map
template <bool HPC>
__global__ void wm_sketch_emit_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ chunk_off,
                                      const int64_t *__restrict__ base_off, int n_tasks, int64_t n_chunks, int k,
                                      const uint8_t *__restrict__ flag_all, const int64_t *__restrict__ rank, wm128_dev *__restrict__ out,
                                      int64_t *__restrict__ mz_off, const int32_t *__restrict__ pos)
{
	const int64_t ch = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (ch > n_chunks) return;
	if (ch == n_chunks) { mz_off[n_tasks] = rank[n_chunks]; return; }
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (chunk_off[m] <= ch) lo = m; else hi = m; }
	const wm_sk_task T = tasks[lo];
	const uint8_t *flag = flag_all + base_off[lo];
	const int c0 = (int)(ch - chunk_off[lo]) * WM_SK_CH;
	int c1 = c0 + WM_SK_CH; if (c1 > T.len) c1 = T.len;
	if (c0 == 0) mz_off[lo] = rank[ch];
	// empty sequences own no chunk: give them the offset of the next non-empty one
	if (c0 == 0) for (int t = lo - 1; t >= 0 && tasks[t].len == 0; --t) mz_off[t] = rank[ch];
	int64_t o = rank[ch];
	const uint64_t mask = (1ULL << 2 * k) - 1;
	for (int i = c0; i < c1; ++i)
		if (flag[i]) {
			uint64_t f, r;
			wm_pk_kmer(wm_pk_window(seq.pk, T.seq_off + i - (k - 1)), k, &f, &r);
			const int z = f < r ? 0 : 1; // src/sketch.c:167
			wm128_dev m;
			if (HPC) {
				const int64_t q = T.seq_off + i;
				const int span = pos[q] - (i >= k ? pos[q - k] : -1);
				m.x = wm_hash64(z ? r : f, mask) << 8 | (uint64_t)span;
				m.y = (uint64_t)T.rid << 32 | (uint32_t)pos[q] << 1 | (uint64_t)z;
			} else {
				m.x = wm_hash64(z ? r : f, mask) << 8 | (uint64_t)k;   // :171 (span == k once l >= k)
				m.y = (uint64_t)T.rid << 32 | (uint32_t)i << 1 | (uint64_t)z; // :172
			}
			out[o++] = m;
		}
}

// ---- ASCII -> packed pool ----
__device__ __forceinline__ uint8_t wm_nt4(unsigned c)
{ // seq_nt4_table (src/sketch.c:19-36): ACGT/acgt (and U/u) -> 0..3, everything else 4
	switch (c) {
		case 'A': case 'a': return 0;
		case 'C': case 'c': return 1;
		case 'G': case 'g': return 2;
		case 'T': case 't': case 'U': case 'u': return 3;
		default: return c < 4 ? (uint8_t)c : 4; // the table maps bytes 0..3 to themselves
	}
}

// One thread packs 32 consecutive bases: two 128-bit loads in, 64 + 32 bits out.  `in` is 16-byte aligned.
__global__ void __launch_bounds__(256)
wm_pack_ascii_kernel(const char *__restrict__ in, int64_t n, uint32_t *__restrict__ pk, uint32_t *__restrict__ nm)
{
	__shared__ uint8_t lut[256];
	lut[threadIdx.x] = wm_nt4(threadIdx.x);
	__syncthreads();
	const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x, b0 = g * 32;
	if (b0 >= n) return;
	uint32_t raw[8];
	if (b0 + 32 <= n) {
		const uint4 a = ((const uint4*)in)[2 * g], b = ((const uint4*)in)[2 * g + 1];
		raw[0] = a.x, raw[1] = a.y, raw[2] = a.z, raw[3] = a.w, raw[4] = b.x, raw[5] = b.y, raw[6] = b.z, raw[7] = b.w;
	} else { // the last group of the pool: the bases past the end read as ambiguous
		#pragma unroll
		for (int j = 0; j < 8; ++j) {
			uint32_t v = 0;
			for (int b = 0; b < 4; ++b) { const int64_t i = b0 + 4 * j + b; v |= (uint32_t)(i < n ? (unsigned char)in[i] : 'N') << 8 * b; }
			raw[j] = v;
		}
	}
	uint64_t p; uint32_t m;
	wm_pk_pack32(raw, lut, &p, &m);
	((uint2*)pk)[g] = make_uint2((uint32_t)p, (uint32_t)(p >> 32));
	nm[g] = m;
}

// the same for reads scattered over a device ASCII pool (read i: pool[src_off[i] ..), packed at dst_off[i] of the batch pool)
__global__ void __launch_bounds__(256)
wm_pack_gather_kernel(const char *__restrict__ pool, const int64_t *__restrict__ src_off, const int64_t *__restrict__ dst_off, int n_reads,
                      int64_t n, uint32_t *__restrict__ pk, uint32_t *__restrict__ nm)
{
	__shared__ uint8_t lut[256];
	lut[threadIdx.x] = wm_nt4(threadIdx.x);
	__syncthreads();
	const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x, b0 = g * 32;
	if (b0 >= n) return;
	int lo = 0, hi = n_reads;
	while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (dst_off[m] <= b0) lo = m; else hi = m; }
	uint64_t p = 0; uint32_t m = 0;
	for (int j = 0; j < 32; ++j) {
		const int64_t i = b0 + j;
		uint32_t c = 4;
		if (i < n) {
			while (i >= dst_off[lo + 1]) ++lo;
			c = lut[(unsigned char)pool[src_off[lo] + (i - dst_off[lo])]];
		}
		p |= (uint64_t)(c & 3) << 2 * j;
		m |= (c >> 2) << j;
	}
	((uint2*)pk)[g] = make_uint2((uint32_t)p, (uint32_t)(p >> 32));
	nm[g] = m;
}

// the look-ahead words past the last group (pkseq.cuh) are defined: ambiguous
static void wm_pack_tail(int64_t n, uint32_t *d_pk, uint32_t *d_nm, cudaStream_t st)
{
	const int64_t g = (n + 31) / 32;
	WM_CUDA_CHECK(cudaMemsetAsync(d_pk + 2 * g, 0, sizeof(uint32_t) * WM_PK_SLACK, st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_nm + g, 0xff, sizeof(uint32_t) * WM_PK_SLACK, st));
}

void wm_pack_ascii(const char *d_in, int64_t n, uint32_t *d_pk, uint32_t *d_nm, cudaStream_t st)
{
	wm_pack_tail(n, d_pk, d_nm, st);
	if (n <= 0) return;
	wm_count_launch(); wm_pack_ascii_kernel<<<(unsigned)((n + 32 * 256 - 1) / (32 * 256)), 256, 0, st>>>(d_in, n, d_pk, d_nm);
	WM_CUDA_CHECK(cudaGetLastError());
}

void wm_pack_gather(const char *d_pool, const int64_t *d_src_off, const int64_t *d_dst_off, int n_reads, int64_t n, uint32_t *d_pk, uint32_t *d_nm, cudaStream_t st)
{
	wm_pack_tail(n, d_pk, d_nm, st);
	if (n <= 0) return;
	wm_count_launch(); wm_pack_gather_kernel<<<(unsigned)((n + 32 * 256 - 1) / (32 * 256)), 256, 0, st>>>(d_pool, d_src_off, d_dst_off, n_reads, n, d_pk, d_nm);
	WM_CUDA_CHECK(cudaGetLastError());
}

// ---- host-side launcher on device-resident code arrays ----
// tasks (host copy) describe slices of the packed pool `seq` (offsets in bases).  On return *n_mz is the total number of minimizers,
// ws->mz holds them (device) and ws->mz_off (device, n_tasks+1) their per-task offsets.  HPC: `seq` is the compressed pool and
// `pos` its symbol -> base map (wm_sketch_run_hpc).
template <bool HPC>
static void wm_sketch_passes(wm_sketch_ws *ws, const wm_bloom_dev &bf, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks,
                             int w, int k, const int32_t *pos, int64_t *n_mz, cudaStream_t st)
{
	*n_mz = 0;
	std::vector<int64_t> h_off(3 * (size_t)(n_tasks + 1));
	int64_t *tile_off = h_off.data(), *chunk_off = tile_off + n_tasks + 1, *base_off = chunk_off + n_tasks + 1;
	tile_off[0] = chunk_off[0] = base_off[0] = 0;
	for (int i = 0; i < n_tasks; ++i) {
		int64_t L = h_tasks[i].len > 0 ? h_tasks[i].len : 0;
		tile_off[i + 1] = tile_off[i] + (L + WM_SK_TN - 1) / WM_SK_TN;
		chunk_off[i + 1] = chunk_off[i] + (L + WM_SK_CH - 1) / WM_SK_CH;
		base_off[i + 1] = base_off[i] + L;
	}
	const int64_t n_tiles = tile_off[n_tasks], n_chunks = chunk_off[n_tasks], n_bases = base_off[n_tasks];
	wm_sk_task *d_tasks = (wm_sk_task*)ws->tasks.need(sizeof(wm_sk_task) * (n_tasks + 1));
	int64_t *d_off = (int64_t*)ws->offs.need(sizeof(int64_t) * h_off.size());
	int64_t *d_mz_off = (int64_t*)ws->mz_off.need(sizeof(int64_t) * (n_tasks + 1));
	WM_CUDA_CHECK(wm_memcpy_async(d_tasks, h_tasks, sizeof(wm_sk_task) * n_tasks, cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_off, h_off.data(), sizeof(int64_t) * h_off.size(), cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(cudaMemsetAsync(d_mz_off, 0, sizeof(int64_t) * (n_tasks + 1), st));
	if (n_bases == 0 || n_tasks == 0) { wm_stream_sync(st); return; }
	const int64_t *d_tile_off = d_off, *d_chunk_off = d_off + n_tasks + 1, *d_base_off = d_chunk_off + n_tasks + 1;
	uint8_t *d_flag = (uint8_t*)ws->flag.need(n_bases);
	WM_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, n_bases, st));
	if (k & 1) {
		double *d_ord = (double*)ws->ord.need(sizeof(double) * n_bases);
		uint8_t *d_elig = (uint8_t*)ws->elig.need(n_bases);
		wm_count_launch(); wm_sketch_order_kernel<HPC><<<(unsigned)n_tiles, WM_SK_THREADS, WM_SK_SMEM, st>>>(seq, d_tasks, d_tile_off, d_base_off, n_tasks, w, k, bf, d_ord, d_elig, pos);
		WM_CUDA_CHECK(cudaGetLastError());
		wm_count_launch(); wm_sketch_winnow_kernel<HPC><<<(unsigned)((n_chunks + 127) / 128), 128, 0, st>>>(d_tasks, d_chunk_off, d_base_off, n_tasks, n_chunks, w, d_ord, d_elig, d_flag);
		WM_CUDA_CHECK(cudaGetLastError());
	} else {
		double *d_ring = (double*)ws->ord.need(sizeof(double) * 512 * (size_t)n_tasks);
		wm_count_launch(); wm_sketch_seq_kernel<HPC><<<(n_tasks + 63) / 64, 64, 0, st>>>(seq, d_tasks, d_base_off, n_tasks, w, k, bf, d_flag, d_ring, pos);
		WM_CUDA_CHECK(cudaGetLastError());
	}
	int32_t *d_cnt = (int32_t*)ws->cnt.need(sizeof(int32_t) * (n_chunks + 1));
	int64_t *d_rank = (int64_t*)ws->rank.need(sizeof(int64_t) * (n_chunks + 2));
	int64_t *d_tmp = (int64_t*)ws->scan_tmp.need(sizeof(int64_t) * wm_scan_tmp_elems(n_chunks));
	wm_count_launch(); wm_sketch_count_kernel<<<(unsigned)((n_chunks + 127) / 128), 128, 0, st>>>(d_tasks, d_chunk_off, d_base_off, n_tasks, n_chunks, d_flag, d_cnt);
	WM_CUDA_CHECK(cudaGetLastError());
	wm_exclusive_scan(d_cnt, n_chunks, d_rank, d_tmp, st);
	int64_t total = 0;
	WM_CUDA_CHECK(wm_memcpy_async(&total, d_rank + n_chunks, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	wm128_dev *d_mz = (wm128_dev*)ws->mz.need(sizeof(wm128_dev) * (total + 1));
	// trailing empty sequences: their offset is the total
	{
		std::vector<int64_t> fill(n_tasks + 1, total);
		WM_CUDA_CHECK(wm_memcpy_async(d_mz_off, fill.data(), sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice, st));
	}
	wm_count_launch(); wm_sketch_emit_kernel<HPC><<<(unsigned)((n_chunks + 1 + 127) / 128), 128, 0, st>>>(seq, d_tasks, d_chunk_off, d_base_off, n_tasks, n_chunks, k,
	                                                                                    d_flag, d_rank, d_mz, d_mz_off, pos);
	WM_CUDA_CHECK(cudaGetLastError());
	*n_mz = total;
}

void wm_sketch_run(wm_sketch_ws *ws, const wm_bloom_dev &bf, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks,
                   int w, int k, int64_t *n_mz, cudaStream_t st)
{
	wm_sketch_passes<false>(ws, bf, seq, h_tasks, n_tasks, w, k, 0, n_mz, st);
}

// ---- homopolymer-compressed sketch: a compaction front end, then the passes above on the compressed slices ----
// H1: one thread per 32-base group of a task: the symbol ends of the group (hpc.cuh) and their number
__global__ void wm_hpc_mark_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ grp_off, int n_tasks,
                                   int64_t n_groups, uint32_t *__restrict__ ends, int32_t *__restrict__ cnt)
{
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n_groups) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (grp_off[m] <= g) lo = m; else hi = m; }
	const wm_sk_task T = tasks[lo];
	const int j = (int)(g - grp_off[lo]);
	const int64_t b = T.seq_off + 32 * (int64_t)j;
	uint32_t e = wm_hpc_ends32(wm_pk_window(seq.pk, b), wm_pk_window(seq.pk, b + 1), wm_pk_nwindow(seq.nm, b), wm_pk_nwindow(seq.nm, b + 1));
	e = wm_hpc_clip(e, j, T.len);
	ends[g] = e, cnt[g] = __popc(e);
}

// H3: every symbol's base (relative to its task) at its rank; coff[t] = the first symbol of task t (coff[n_tasks] = total)
__global__ void wm_hpc_scatter_kernel(const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ grp_off, int n_tasks, int64_t n_groups,
                                      const uint32_t *__restrict__ ends, const int64_t *__restrict__ rank, int32_t *__restrict__ pos,
                                      int64_t *__restrict__ coff)
{
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (g > n_groups) return;
	if (g == n_groups) { // the total, also for trailing empty tasks
		coff[n_tasks] = rank[n_groups];
		for (int t = n_tasks - 1; t >= 0 && tasks[t].len <= 0; --t) coff[t] = rank[n_groups];
		return;
	}
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { int m = (lo + hi) >> 1; if (grp_off[m] <= g) lo = m; else hi = m; }
	const int j = (int)(g - grp_off[lo]);
	int64_t o = rank[g];
	if (j == 0) { // empty tasks own no group: give them the offset of the next non-empty one
		coff[lo] = o;
		for (int t = lo - 1; t >= 0 && tasks[t].len <= 0; --t) coff[t] = o;
	}
	for (uint32_t e = ends[g]; e; e &= e - 1) pos[o++] = 32 * j + __ffs(e) - 1;
}

// H4: the compressed pool, one thread per 32 symbols (the gather of wm_pack_gather_kernel, symbol s of task t being base
// pos[s] of the task); past the last symbol the codes read as ambiguous
__global__ void __launch_bounds__(256)
wm_hpc_pack_kernel(const wm_pkseq seq, const wm_sk_task *__restrict__ tasks, const int64_t *__restrict__ coff, int n_tasks,
                   const int32_t *__restrict__ pos, int64_t n, uint32_t *__restrict__ pk, uint32_t *__restrict__ nm)
{
	const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, s0 = g * 32;
	if (s0 >= n) return;
	int lo = 0, hi = n_tasks;
	while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (coff[m] <= s0) lo = m; else hi = m; }
	uint64_t p = 0; uint32_t m = 0;
	for (int j = 0; j < 32; ++j) {
		const int64_t s = s0 + j;
		int c = 4;
		if (s < n) {
			while (s >= coff[lo + 1]) ++lo;
			c = wm_pk_get(seq, tasks[lo].seq_off + pos[s]);
		}
		p |= (uint64_t)(c & 3) << 2 * j;
		m |= (uint32_t)(c >> 2) << j;
	}
	((uint2*)pk)[g] = make_uint2((uint32_t)p, (uint32_t)(p >> 32));
	nm[g] = m;
}

void wm_sketch_run_hpc(wm_sketch_ws *ws, const wm_bloom_dev &bf, const wm_pkseq &seq, const wm_sk_task *h_tasks, int n_tasks,
                       int w, int k, int64_t *n_mz, cudaStream_t st)
{
	*n_mz = 0;
	std::vector<int64_t> grp_off(n_tasks + 1, 0);
	for (int i = 0; i < n_tasks; ++i) grp_off[i + 1] = grp_off[i] + (h_tasks[i].len > 0 ? (h_tasks[i].len + 31) / 32 : 0);
	const int64_t n_groups = grp_off[n_tasks];
	if (n_tasks == 0 || n_groups == 0) { wm_sketch_passes<false>(ws, bf, seq, h_tasks, n_tasks, w, k, 0, n_mz, st); return; }
	wm_sk_task *d_tasks = (wm_sk_task*)ws->hpc_tasks.need(sizeof(wm_sk_task) * n_tasks);
	int64_t *d_goff = (int64_t*)ws->hpc_goff.need(sizeof(int64_t) * (n_tasks + 1));
	int64_t *d_coff = (int64_t*)ws->hpc_coff.need(sizeof(int64_t) * (n_tasks + 1));
	uint32_t *d_ends = (uint32_t*)ws->hpc_ends.need(sizeof(uint32_t) * n_groups);
	int32_t *d_cnt = (int32_t*)ws->cnt.need(sizeof(int32_t) * (n_groups + 1));
	int64_t *d_rank = (int64_t*)ws->rank.need(sizeof(int64_t) * (n_groups + 2));
	int64_t *d_tmp = (int64_t*)ws->scan_tmp.need(sizeof(int64_t) * wm_scan_tmp_elems(n_groups));
	WM_CUDA_CHECK(wm_memcpy_async(d_tasks, h_tasks, sizeof(wm_sk_task) * n_tasks, cudaMemcpyHostToDevice, st));
	WM_CUDA_CHECK(wm_memcpy_async(d_goff, grp_off.data(), sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice, st));
	wm_count_launch(); wm_hpc_mark_kernel<<<(unsigned)((n_groups + 127) / 128), 128, 0, st>>>(seq, d_tasks, d_goff, n_tasks, n_groups, d_ends, d_cnt);
	WM_CUDA_CHECK(cudaGetLastError());
	wm_exclusive_scan(d_cnt, n_groups, d_rank, d_tmp, st);
	int64_t n_sym = 0;
	WM_CUDA_CHECK(wm_memcpy_async(&n_sym, d_rank + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	int32_t *d_pos = (int32_t*)ws->hpc_pos.need(sizeof(int32_t) * (n_sym + 1));
	wm_count_launch(); wm_hpc_scatter_kernel<<<(unsigned)((n_groups + 1 + 127) / 128), 128, 0, st>>>(d_tasks, d_goff, n_tasks, n_groups, d_ends, d_rank, d_pos, d_coff);
	WM_CUDA_CHECK(cudaGetLastError());
	wm_pkseq cs;
	cs.pk = (const uint32_t*)ws->hpc_pk.need(sizeof(uint32_t) * wm_pk_words(n_sym));
	cs.nm = (const uint32_t*)ws->hpc_nm.need(sizeof(uint32_t) * wm_nm_words(n_sym));
	wm_pack_tail(n_sym, (uint32_t*)cs.pk, (uint32_t*)cs.nm, st);
	wm_count_launch(); wm_hpc_pack_kernel<<<(unsigned)((n_sym + 32 * 256 - 1) / (32 * 256)), 256, 0, st>>>(seq, d_tasks, d_coff, n_tasks, d_pos, n_sym,
	                                                                                                   (uint32_t*)cs.pk, (uint32_t*)cs.nm);
	WM_CUDA_CHECK(cudaGetLastError());
	std::vector<int64_t> coff(n_tasks + 1);
	WM_CUDA_CHECK(wm_memcpy_async(coff.data(), d_coff, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyDeviceToHost, st));
	wm_stream_sync(st);
	std::vector<wm_sk_task> ct(n_tasks);
	for (int i = 0; i < n_tasks; ++i) ct[i].seq_off = coff[i], ct[i].len = (int32_t)(coff[i + 1] - coff[i]), ct[i].rid = h_tasks[i].rid;
	wm_sketch_passes<true>(ws, bf, cs, ct.data(), n_tasks, w, k, d_pos, n_mz, st);
}

// one byte per minimizer: its span (x & 0xff)
__global__ void wm_mz_span_kernel(const wm128_dev *__restrict__ mz, int64_t n, uint8_t *__restrict__ span)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) span[i] = (uint8_t)(mz[i].x & 0xff);
}

void wm_mz_spans(const wm128_dev *d_mz, int64_t n, uint8_t *d_span, cudaStream_t st)
{
	if (n <= 0) return;
	wm_count_launch(); wm_mz_span_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_mz, n, d_span);
	WM_CUDA_CHECK(cudaGetLastError());
}

// ---- down-weight filter construction (host; replaces bloom_filter of src/index.c:404-432) ----
struct wm_bloom_s {
	uint64_t bits; uint32_t salt[2]; int n_salt;
	std::vector<uint8_t> table;
};

static inline uint32_t wm_hash_ap8_host(uint64_t key, uint32_t h)
{
	uint32_t i1 = (uint32_t)key, i2 = (uint32_t)(key >> 32);
	h ^= (h << 7) ^ (i1 * (h >> 3)) ^ (~((h << 11) + (i2 ^ (h >> 5))));
	return h;
}

extern "C" wm_bloom_s *wm_bloom_build(const uint64_t *canon_kmers, int64_t n)
{
	wm_bloom_s *b = new wm_bloom_s();
	// bloom_parameters::compute_optimal_parameters (bloom_filter.hpp:108-147) with
	// projected_element_count = max(n,1000), fpp = 0.001, maximum_number_of_hashes = 2 (index.c:411-414)
	const double cnt = (double)(n > 1000 ? n : 1000), p = 0.001;
	double min_m = INFINITY, min_k = 0.0;
	for (double kk = 1.0; kk < 1000.0; kk += 1.0) {
		double m = (-kk * cnt) / log(1.0 - pow(p, 1.0 / kk));
		if (m < min_m) min_m = m, min_k = kk;
	}
	unsigned nh = (unsigned)min_k;
	uint64_t ts = (uint64_t)min_m;
	ts += (ts % 8) != 0 ? 8 - ts % 8 : 0;
	if (nh < 1) nh = 1; else if (nh > 2) nh = 2;
	b->bits = ts, b->n_salt = (int)nh;
	const uint64_t seed = 0xA5A5A5A55A5A5A5AULL * 0xA5A5A5A5ULL + 1; // bloom_filter.hpp:186
	const uint32_t predef[2] = { 0xAAAAAAAAu, 0x55555555u };          // :477
	for (int i = 0; i < b->n_salt; ++i) b->salt[i] = predef[i];
	for (int i = 0; i < b->n_salt; ++i) b->salt[i] = b->salt[i] * b->salt[(i + 3) % b->n_salt] + (uint32_t)seed; // :519-528
	b->table.assign(ts / 8 + 16, 0);
	for (int64_t i = 0; i < n; ++i)
		for (int s = 0; s < b->n_salt; ++s) {
			uint64_t bit = (uint64_t)wm_hash_ap8_host(canon_kmers[i], b->salt[s]) % ts;
			b->table[bit >> 3] |= (uint8_t)(1u << (bit & 7));
		}
	return b;
}
extern "C" uint64_t wm_bloom_bits(const wm_bloom_s *b) { return b->bits; }
extern "C" const uint8_t *wm_bloom_table(const wm_bloom_s *b) { return b->table.data(); }
extern "C" void wm_bloom_destroy(wm_bloom_s *b) { delete b; }

void wm_bloom_params(const wm_bloom_s *b, uint64_t *bits, uint32_t *salt, int *n_salt)
{
	*bits = b->bits; salt[0] = b->salt[0]; salt[1] = b->salt[1]; *n_salt = b->n_salt;
}

// salts depend only on the number of hashes, which is 2 for every table built by the reference
void wm_bloom_dev_from_table(wm_bloom_dev *d, const uint8_t *d_table, uint64_t bits)
{
	const uint64_t seed = 0xA5A5A5A55A5A5A5AULL * 0xA5A5A5A5ULL + 1;
	d->table = d_table; d->bits = bits; d->n_salt = 2;
	d->salt[0] = 0xAAAAAAAAu; d->salt[1] = 0x55555555u;
	for (int i = 0; i < 2; ++i) d->salt[i] = d->salt[i] * d->salt[(i + 3) % 2] + (uint32_t)seed;
}

// ---- C ABI: batched mm_sketch ----
static int wm_sketch_batch_impl(const wm_bloom_s *bloom, int n, const char *seq, const int64_t *off, const uint32_t *rid,
                                int w, int k, int is_hpc, wm128_dev **out, int64_t **out_off)
{
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		fprintf(stderr, "[ERROR] wm_sketch_batch: no CUDA device visible; winnowmap-b200 has no CPU fallback\n");
		exit(1);
	}
	if (!(w > 0 && w < 256 && k > 0 && k <= 28)) { // assert at src/sketch.c:140
		fprintf(stderr, "[ERROR] wm_sketch_batch: invalid (w,k)\n");
		return -1;
	}
	*out = 0; *out_off = (int64_t*)calloc(n + 1, sizeof(int64_t));
	if (n <= 0) return 0;
	const int64_t tot = off[n];
	char *d_ascii = wm_dev_alloc<char>(tot + 1);
	uint32_t *d_pk = wm_dev_alloc<uint32_t>(wm_pk_words(tot)), *d_nm = wm_dev_alloc<uint32_t>(wm_nm_words(tot));
	WM_CUDA_CHECK(cudaMemcpy(d_ascii, seq, tot, cudaMemcpyHostToDevice));
	wm_pack_ascii(d_ascii, tot, d_pk, d_nm, 0);
	wm_pkseq pks; pks.pk = d_pk, pks.nm = d_nm;
	uint8_t *d_table = wm_dev_alloc<uint8_t>(bloom->table.size());
	WM_CUDA_CHECK(cudaMemcpy(d_table, bloom->table.data(), bloom->table.size(), cudaMemcpyHostToDevice));
	wm_bloom_dev bf; wm_bloom_dev_from_table(&bf, d_table, bloom->bits);
	bf.n_salt = bloom->n_salt; bf.salt[0] = bloom->salt[0]; bf.salt[1] = bloom->salt[1];
	std::vector<wm_sk_task> tasks(n);
	for (int i = 0; i < n; ++i) tasks[i].seq_off = off[i], tasks[i].len = (int32_t)(off[i + 1] - off[i]), tasks[i].rid = rid ? rid[i] : 0;
	wm_sketch_ws ws;
	int64_t n_mz = 0;
	if (is_hpc) wm_sketch_run_hpc(&ws, bf, pks, tasks.data(), n, w, k, &n_mz, 0);
	else wm_sketch_run(&ws, bf, pks, tasks.data(), n, w, k, &n_mz, 0);
	WM_CUDA_CHECK(cudaDeviceSynchronize());
	*out = (wm128_dev*)malloc(sizeof(wm128_dev) * (n_mz > 0 ? n_mz : 1));
	if (n_mz > 0) WM_CUDA_CHECK(cudaMemcpy(*out, ws.mz.p, sizeof(wm128_dev) * n_mz, cudaMemcpyDeviceToHost));
	WM_CUDA_CHECK(cudaMemcpy(*out_off, ws.mz_off.p, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost));
	ws.release();
	cudaFree(d_ascii); cudaFree(d_pk); cudaFree(d_nm); cudaFree(d_table);
	return 0;
}

extern "C" int wm_sketch_batch(const wm_bloom_s *bloom, int n, const char *seq, const int64_t *off, const uint32_t *rid,
                               int w, int k, wm128_dev **out, int64_t **out_off)
{
	return wm_sketch_batch_impl(bloom, n, seq, off, rid, w, k, 0, out, out_off);
}

extern "C" int wm_sketch_batch_hpc(const wm_bloom_s *bloom, int n, const char *seq, const int64_t *off, const uint32_t *rid,
                                   int w, int k, wm128_dev **out, int64_t **out_off)
{
	return wm_sketch_batch_impl(bloom, n, seq, off, rid, w, k, 1, out, out_off);
}

// bench: the sketch stage alone on device-resident packed reads, plain or homopolymer-compressed; *ms = CUDA-event time
// of one call, the mean over `reps` calls after one untimed call (workspaces sized)
extern "C" int wm_bench_sketch(const wm_bloom_s *bloom, int n, const char *seq, const int64_t *off, int w, int k, int is_hpc, int reps, double *ms)
{
	if (!(w > 0 && w < 256 && k > 0 && k <= 28) || n <= 0 || reps <= 0) return -1;
	const int64_t tot = off[n];
	char *d_ascii = wm_dev_alloc<char>(tot + 16);
	uint32_t *d_pk = wm_dev_alloc<uint32_t>(wm_pk_words(tot)), *d_nm = wm_dev_alloc<uint32_t>(wm_nm_words(tot));
	WM_CUDA_CHECK(cudaMemcpy(d_ascii, seq, tot, cudaMemcpyHostToDevice));
	wm_pack_ascii(d_ascii, tot, d_pk, d_nm, 0);
	wm_pkseq pks; pks.pk = d_pk, pks.nm = d_nm;
	uint8_t *d_table = wm_dev_alloc<uint8_t>(bloom->table.size());
	WM_CUDA_CHECK(cudaMemcpy(d_table, bloom->table.data(), bloom->table.size(), cudaMemcpyHostToDevice));
	wm_bloom_dev bf; wm_bloom_dev_from_table(&bf, d_table, bloom->bits);
	bf.n_salt = bloom->n_salt; bf.salt[0] = bloom->salt[0]; bf.salt[1] = bloom->salt[1];
	std::vector<wm_sk_task> tasks(n);
	for (int i = 0; i < n; ++i) tasks[i].seq_off = off[i], tasks[i].len = (int32_t)(off[i + 1] - off[i]), tasks[i].rid = 0;
	wm_sketch_ws ws;
	int64_t n_mz = 0;
	cudaEvent_t e0, e1;
	WM_CUDA_CHECK(cudaEventCreate(&e0)); WM_CUDA_CHECK(cudaEventCreate(&e1));
	for (int r = -1; r < reps; ++r) {
		if (r == 0) WM_CUDA_CHECK(cudaEventRecord(e0, 0));
		if (is_hpc) wm_sketch_run_hpc(&ws, bf, pks, tasks.data(), n, w, k, &n_mz, 0);
		else wm_sketch_run(&ws, bf, pks, tasks.data(), n, w, k, &n_mz, 0);
	}
	WM_CUDA_CHECK(cudaEventRecord(e1, 0));
	WM_CUDA_CHECK(cudaEventSynchronize(e1));
	float f = 0.f;
	WM_CUDA_CHECK(cudaEventElapsedTime(&f, e0, e1));
	*ms = f / reps;
	cudaEventDestroy(e0); cudaEventDestroy(e1);
	ws.release();
	cudaFree(d_ascii); cudaFree(d_pk); cudaFree(d_nm); cudaFree(d_table);
	return 0;
}
