/*
 * oracle/wm_oracle_hpc.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement of mm_sketch with is_hpc = 1 (src/sketch.c:128-219, the branch at :146-157), built together with
 * wm_oracle.c into oracle/libwm_oracle_hpc.so.  It is stated the way the CUDA front end computes it, not the way the
 * reference does: the slice is first compressed into symbols (a run of one non-ambiguous code is one symbol at the run's
 * last base, every ambiguous base a symbol of its own), then the plain winnowing walk runs over the symbols, and the
 * span of the k-mer ending at symbol j is pos[j] - pos[j - k] (pos[-1] = -1).  The reference instead keeps the last k run
 * lengths in a tiny queue.  tests/test_hpc_cpu.py pins the two against each other through the digests of the reference's
 * own output.  The product never links, imports or executes this file.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef __cplusplus
extern "C" {
#endif
typedef struct wmo_bloom_s wmo_bloom_t;
uint64_t wmo_hash64(uint64_t key, uint64_t mask);
double wmo_weight(uint64_t kmer, const wmo_bloom_t *bf);
long wmo_hpc_compress(const char *str, int len, uint8_t *code, int32_t *pos);
long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const wmo_bloom_t *bf, uint64_t *out_xy, long max_out);
#ifdef __cplusplus
}
#endif

static int wmo_hpc_nt4(unsigned char c)
{ /* seq_nt4_table, src/sketch.c:19-36 */
	switch (c) {
	case 'A': case 'a': return 0;
	case 'C': case 'c': return 1;
	case 'G': case 'g': return 2;
	case 'T': case 't': case 'U': case 'u': return 3;
	default: return c < 4 ? c : 4;
	}
}

/* The symbols of str[0, len): code[j] and pos[j] (the last base of the symbol); returns their number. */
long wmo_hpc_compress(const char *str, int len, uint8_t *code, int32_t *pos)
{
	long n = 0;
	int i;
	for (i = 0; i < len; ++i) {
		const int c = wmo_hpc_nt4((unsigned char)str[i]);
		if (c < 4)
			while (i + 1 < len && wmo_hpc_nt4((unsigned char)str[i + 1]) == c) ++i;
		code[n] = (uint8_t)c, pos[n] = i, ++n;
	}
	return n;
}

/* returns the number of minimizers; writes up to max_out (x,y) pairs */
long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const wmo_bloom_t *bf, uint64_t *out_xy, long max_out)
{
	const uint64_t shift1 = 2 * (k - 1), mask = (1ULL << 2 * k) - 1;
	uint64_t kmer[2] = {0, 0}, bufx[256], bufy[256], minx = UINT64_MAX, miny = UINT64_MAX;
	double buf_order[256], min_order = 2.0;
	int j, l = 0, buf_pos = 0, min_pos = 0;
	long n = 0, s, n_sym;
	uint8_t *code = (uint8_t*)malloc(len > 0 ? len : 1);
	int32_t *pos = (int32_t*)malloc(sizeof(int32_t) * (len > 0 ? len : 1));
#define WMO_EMIT() do { if (n < max_out) out_xy[2*n] = minx, out_xy[2*n+1] = miny; ++n; } while (0)
	n_sym = wmo_hpc_compress(str, len, code, pos);
	for (j = 0; j < w; ++j) bufx[j] = bufy[j] = UINT64_MAX, buf_order[j] = 2.0;
	for (s = 0; s < n_sym; ++s) {
		const int c = code[s];
		uint64_t ix = UINT64_MAX, iy = UINT64_MAX;
		double io = 2.0;
		if (c < 4) {
			int z;
			kmer[0] = (kmer[0] << 2 | (uint64_t)c) & mask;
			kmer[1] = (kmer[1] >> 2) | (3ULL ^ (uint64_t)c) << shift1;
			if (kmer[0] == kmer[1]) continue; /* symmetric: the symbol still counts in later spans */
			z = kmer[0] < kmer[1] ? 0 : 1;
			++l;
			if (l >= k) {
				const int span = pos[s] - (s >= k ? pos[s - k] : -1);
				if (span < 256) {
					ix = wmo_hash64(kmer[z], mask) << 8 | (uint64_t)span;
					iy = (uint64_t)rid << 32 | (uint32_t)pos[s] << 1 | (uint64_t)z;
					io = wmo_weight(kmer[z], bf);
				}
			}
		} else l = 0;
		bufx[buf_pos] = ix, bufy[buf_pos] = iy, buf_order[buf_pos] = io;
		if (io < min_order) {
			if (l >= w + k && minx != UINT64_MAX) WMO_EMIT();
			minx = ix, miny = iy, min_pos = buf_pos, min_order = io;
		} else if (buf_pos == min_pos) {
			if (l >= w + k - 1 && minx != UINT64_MAX) WMO_EMIT();
			for (j = buf_pos + 1, minx = UINT64_MAX, miny = UINT64_MAX, min_order = 2.0; j < w; ++j)
				if (min_order >= buf_order[j]) minx = bufx[j], miny = bufy[j], min_pos = j, min_order = buf_order[j];
			for (j = 0; j <= buf_pos; ++j)
				if (min_order >= buf_order[j]) minx = bufx[j], miny = bufy[j], min_pos = j, min_order = buf_order[j];
		}
		if (++buf_pos == w) buf_pos = 0;
	}
	if (minx != UINT64_MAX) WMO_EMIT();
#undef WMO_EMIT
	free(code); free(pos);
	return n;
}
