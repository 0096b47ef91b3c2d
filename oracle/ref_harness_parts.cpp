// TEST INFRASTRUCTURE ONLY. extern "C" wrappers around the REAL reference's index reader over a FASTA with -I (index parts,
// src/index.c:660-671) and its mm_idx_cal_max_occ (src/index.c:173-194), for tests/test_parts_host.py and
// tools/make_golden.py --parts.  Compiled by tools/make_golden.py (ref_parts_lib) against oracle/_ref/libwinnowmap.a (oracle/build_ref.sh)
// where the reference's sources are present; nothing in the product path links or loads it.
#include <stdint.h>
#include <stdlib.h>
#include "minimap.h"
#include "mmpriv.h"
#include "khash.h"

#define ref_parts_hash(a) ((a)>>1)
#define ref_parts_eq(a, b) ((a)>>1 == (b)>>1)
KHASH_INIT(refparts, uint64_t, uint64_t, 1, ref_parts_hash, ref_parts_eq) // the table type of src/index.c:25-27 under another name (same layout)
typedef struct { // mm_idx_bucket_t, src/index.c:33-38 (opaque in minimap.h)
	mm128_v a;
	int32_t n;
	uint64_t *p;
	void *h;
} ref_parts_bucket_t;

extern "C" {

// the reference's index reader with batch_size = -I; each ref_idx_reader_next is one part (NULL at the end)
void *ref_idx_reader_open(const char *fn, int w, int k, int flag, uint64_t batch_size)
{
	mm_idxopt_t io; mm_mapopt_t mo;
	mm_set_opt(0, &io, &mo);
	io.k = k, io.w = w, io.flag = flag, io.batch_size = batch_size;
	return mm_idx_reader_open(fn, &io, 0);
}
void *ref_idx_reader_next(void *r, const char *kmer_fn) { return mm_idx_reader_read((mm_idx_reader_t*)r, 3, kmer_fn ? kmer_fn : ""); }
void ref_idx_reader_close(void *r) { mm_idx_reader_close((mm_idx_reader_t*)r); }
int ref_idx_part_n_seq(void *mi) { return (int)((mm_idx_t*)mi)->n_seq; }
// the occurrence count of every key (a singleton counts 1), in the bucket walk order of mm_idx_cal_max_occ; returns n
int64_t ref_idx_part_counts(void *mi_, uint32_t *out, int64_t cap)
{
	const mm_idx_t *mi = (const mm_idx_t*)mi_;
	const ref_parts_bucket_t *B = (const ref_parts_bucket_t*)mi->B;
	int64_t n = 0;
	for (uint32_t b = 0; b < 1U << mi->b; ++b) {
		khash_t(refparts) *h = (khash_t(refparts)*)B[b].h;
		if (h == 0) continue;
		for (khint_t x = 0; x < kh_end(h); ++x) {
			if (!kh_exist(h, x)) continue;
			if (n < cap) out[n] = kh_key(h, x) & 1 ? 1 : (uint32_t)kh_val(h, x);
			++n;
		}
	}
	return n;
}
int32_t ref_idx_cal_max_occ(void *mi, float f) { return mm_idx_cal_max_occ((const mm_idx_t*)mi, f); }
void ref_idx_part_free(void *mi) { mm_idx_destroy((mm_idx_t*)mi); }

} // extern "C"
