// TEST INFRASTRUCTURE ONLY.  The reference's own mm_chain_dp (src/chain.c:22) with is_cdna = 1, the chaining of spliced mapping,
// behind an extern "C" wrapper shaped like ref_chain_dp of ref_harness.cpp.  Compiled on demand against the reference library that
// oracle/build_ref.sh builds (tests/splice_lib.py), where the reference's sources are present.
#include <stdint.h>
#include <string.h>
#include "minimap.h"
#include "mmpriv.h"
#include "kalloc.h"

extern "C" int ref_chain_dp_cdna(int max_dist_x, int min_dist_x, int max_dist_y, int bw, int max_skip, int max_iter, int min_cnt, int min_sc,
                                 float gap_scale, long n, const uint64_t *a_xy, uint64_t *u_out, uint64_t *b_out, long *n_b)
{ // a_xy is copied (mm_chain_dp frees its input); returns n_u, writes u[] and the compacted anchors
	mm128_t *a = (mm128_t*)kmalloc(0, (n > 0 ? n : 1) * 16);
	memcpy(a, a_xy, n * 16);
	int n_u = 0; uint64_t *u = 0;
	mm128_t *b = mm_chain_dp(max_dist_x, min_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc, gap_scale, 1, 1, n, a, &n_u, &u, 0);
	long nb = 0;
	for (int i = 0; i < n_u; ++i) { u_out[i] = u[i]; nb += (int32_t)u[i]; }
	if (nb) memcpy(b_out, b, nb * 16);
	*n_b = nb;
	kfree(0, b); kfree(0, u);
	return n_u;
}
