// TEST INFRASTRUCTURE ONLY.  The reference's SDUST (sdust(), src/sdust.c:166) and its minimizer squeeze (mm_dust_minier,
// src/map.c:43, a static function: this unit compiles the map.c that build_ref.sh patched into oracle/_ref/build, so that it
// can call it).  Built into oracle/_ref/libref_harness_sdust.so by oracle/build_sdust.sh; nothing in the product path links
// or loads it.
#include "map_patched.c"
#include "sdust.h"

extern "C" {

// the regions of seq[0, len) as start << 32 | end (at most max_out written); returns their number
long ref_sdust(const char *seq, int len, int T, int W, uint64_t *out, long max_out)
{
	int n = 0;
	uint64_t *r = sdust(0, (const uint8_t*)seq, len, T, W, &n);
	memcpy(out, r, sizeof(uint64_t) * (n < max_out ? n : max_out));
	kfree(0, r);
	return n;
}

// mm_dust_minier on n minimizers (x, y pairs) of seq: squeezed in place; returns how many are kept
long ref_dust_minier(uint64_t *xy, long n, const char *seq, int len, int T)
{
	return mm_dust_minier(0, (int)n, (mm128_t*)xy, len, seq, T);
}

} // extern "C"
