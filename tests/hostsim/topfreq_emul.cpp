// TEST INFRASTRUCTURE: the k-mer walk of the -W list counter (csrc/topfreq.cuh) on the host, reading the packed pool through
// the same window functions as the device (csrc/pkseq.cuh, with the funnel shift and bit reversal of cuda_emul.h).
// tests/test_topfreq_cpu.py compares the codes with a byte-per-base restatement.
#include <vector>
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/topfreq.cuh"

static inline uint32_t code_of(char c)
{ // seq_nt4_table as the device packer applies it (csrc/sketch.cu wm_nt4)
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': case 'U': case 'u': return 3; default: return 4; }
}

// the pool packed as on the device (bases past n ambiguous), then every valid k-mer chunk by chunk: its pool position and
// canonical code, in position order; returns how many
extern "C" long wmt_tf_codes(const char *pool, long n, const int64_t *off, int n_tasks, int k, int64_t *pos_out, uint64_t *code_out)
{
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
	for (long c = 0; c < ng; ++c)
		for (uint32_t v = wm_tf_valid32(nm.data(), off, n_tasks, k, 32 * c); v; v &= v - 1) {
			const int64_t p = 32 * c + __builtin_ctz(v);
			uint64_t code;
			if (!wm_tf_kmer(pk.data(), nm.data(), p, k, &code)) return -1; // valid32 passed an ambiguous k-mer
			pos_out[o] = p, code_out[o] = code, ++o;
		}
	return o;
}
