// TEST INFRASTRUCTURE ONLY.  The reference's own seed collection, collect_seed_hits_heap and collect_seed_hits (src/map.c:156-254,
// static functions: this unit compiles the map.c that build_ref.sh patched into oracle/_ref/build, so that it can call them), on
// an index that the reference's index reader builds from a FASTA file.  Built into oracle/_ref/libref_harness_heap.so by
// oracle/build_heap.sh; nothing in the product path links or loads it.
#include "map_patched.c"

extern "C" {

// mm_idx_reader_open / mm_idx_reader_read (src/index.c:688, :713) on a FASTA file, without a -W list
void *ref_heap_idx(const char *fn, int w, int k)
{
	mm_idxopt_t io; mm_mapopt_t mo;
	mm_set_opt(0, &io, &mo);
	io.k = k, io.w = w;
	mm_idx_reader_t *r = mm_idx_reader_open(fn, &io, 0);
	if (!r) return 0;
	mm_idx_t *mi = mm_idx_reader_read(r, 1, "");
	mm_idx_reader_close(r);
	return mi;
}

void ref_heap_idx_free(void *mi) { mm_idx_destroy((mm_idx_t*)mi); }

// the anchors of one query (n_mv minimizers, x / y pairs) as collect_seed_hits_heap (heap != 0) or collect_seed_hits returns
// them, at most cap written; returns their number.  flag: mm_mapopt_t.flag; qname: 0 for a read without a name.
long ref_heap_seed_hits(void *mi_, int heap, int64_t flag, int max_occ, const char *qname, const uint64_t *mv_xy, long n_mv, int qlen,
                        uint64_t *a_xy, long cap, int *rep_len, uint64_t *mini_pos, int *n_mini_pos)
{
	const mm_idx_t *mi = (const mm_idx_t*)mi_;
	mm_idxopt_t io; mm_mapopt_t opt;
	mm_set_opt(0, &io, &opt);
	opt.flag = flag;
	mm128_v mv;
	mv.n = mv.m = (size_t)n_mv;
	mv.a = (mm128_t*)malloc(sizeof(mm128_t) * (n_mv > 0 ? n_mv : 1));
	memcpy(mv.a, mv_xy, sizeof(mm128_t) * n_mv);
	int64_t n_a = 0;
	uint64_t *mp = 0;
	mm128_t *a = heap ? collect_seed_hits_heap(0, &opt, max_occ, mi, qname, &mv, qlen, &n_a, rep_len, n_mini_pos, &mp)
	                  : collect_seed_hits(0, &opt, max_occ, mi, qname, &mv, qlen, &n_a, rep_len, n_mini_pos, &mp);
	memcpy(a_xy, a, sizeof(mm128_t) * (n_a < cap ? n_a : cap));
	memcpy(mini_pos, mp, sizeof(uint64_t) * *n_mini_pos);
	kfree(0, a); kfree(0, mp); free(mv.a);
	return (long)n_a;
}

} // extern "C"
