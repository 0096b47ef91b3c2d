// TEST INFRASTRUCTURE: the bit functions of the homopolymer-compression front end (csrc/hpc.cuh) on the host, reading
// the packed pool through the same window functions as the device (csrc/pkseq.cuh, with the funnel shift of
// cuda_emul.h).  tests/test_hpc_cpu.py compares the symbol ends with a byte-per-base restatement.
#include <vector>
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/pkseq.cuh"
#include "../../winnowmap_b200/csrc/hpc.cuh"

static inline uint32_t code_of(char c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': case 'U': case 'u': return 3; default: return 4; }
}

extern "C" long wmt_hpc_ends(const char *pool, long n, const long *off, int n_tasks, int32_t *pos_out)
{ // the pool packed as on the device (bases past n ambiguous), then every task's symbol ends group by group
	const long ng = (n + 31) / 32;
	std::vector<uint32_t> pk(2 * ng + WM_PK_SLACK + 4, 0), nm(ng + WM_PK_SLACK + 4, ~0u);
	for (long g = 0; g < ng; ++g) {
		uint64_t p = 0; uint32_t m = 0;
		for (int j = 0; j < 32; ++j) {
			const uint32_t c = g * 32 + j < n ? code_of(pool[g * 32 + j]) : 4;
			p |= (uint64_t)(c & 3) << 2 * j, m |= (c >> 2) << j;
		}
		pk[2 * g] = (uint32_t)p, pk[2 * g + 1] = (uint32_t)(p >> 32), nm[g] = m;
	}
	long o = 0;
	for (int t = 0; t < n_tasks; ++t) {
		const int len = (int)(off[t + 1] - off[t]);
		for (int g = 0; 32 * g < len; ++g) {
			const int64_t b = off[t] + 32 * g;
			uint32_t e = wm_hpc_ends32(wm_pk_window(pk.data(), b), wm_pk_window(pk.data(), b + 1), wm_pk_nwindow(nm.data(), b), wm_pk_nwindow(nm.data(), b + 1));
			e = wm_hpc_clip(e, g, len);
			for (; e; e &= e - 1) pos_out[o++] = 32 * g + __builtin_ctz(e);
		}
	}
	return o;
}
