// TEST INFRASTRUCTURE ONLY.  The reference's own BED reader and junction annotation (mm_idx_bed_read, mm_idx_bed_junc,
// src/index.c:690-803) on a reference mm_idx_t that holds only sequence names.  Built into oracle/_ref/libref_harness_junc.so by
// oracle/build_junc.sh; nothing in the product path links or loads it.  The interval records are read through the library's
// own declaration of their layout (wm_idx_intv_t, include/winnowmap_b200.h).
#include <string.h>
#include "minimap.h"
#include "kalloc.h"
#include "../include/winnowmap_b200.h"

mm_idx_t *mm_idx_init(int w, int k, int b, int flag); // src/index.c:50 (not in a header)

static mm_idx_t *g_mi = 0;

extern "C" {

// an index whose sequences are `names` (no bases), then mm_idx_bed_read(mi, fn, 1); its return value
int ref_bed_read(int n, const char *const *names, const char *fn)
{
	if (g_mi) mm_idx_destroy(g_mi);
	g_mi = mm_idx_init(10, 15, 14, 0);
	g_mi->n_seq = n;
	g_mi->seq = (mm_idx_seq_t*)kcalloc(g_mi->km, n, sizeof(mm_idx_seq_t));
	for (int i = 0; i < n; ++i) {
		g_mi->seq[i].name = (char*)kmalloc(g_mi->km, strlen(names[i]) + 1);
		strcpy(g_mi->seq[i].name, names[i]);
	}
	return mm_idx_bed_read(g_mi, fn, 1);
}

// the raw 16-byte records of mi->I[rid] (at most cap of them into out); their number
int ref_bed_intervals(int rid, void *out, int cap)
{
	const wm_idx_intv_t *I = (const wm_idx_intv_t*)g_mi->I;
	const int n = I[rid].n;
	memcpy(out, I[rid].a, sizeof(wm_idx_intv1_t) * (n < cap ? n : cap));
	return n;
}

// mm_idx_bed_junc(mi, ctg, st, en, s) on the last index read
int ref_bed_junc(int ctg, int st, int en, uint8_t *s) { return mm_idx_bed_junc(g_mi, ctg, st, en, s); }

} // extern "C"
